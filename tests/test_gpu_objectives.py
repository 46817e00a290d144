"""Per-expert objective kernels (csrc/bcm_nll.cu, csrc/laplace.cu) against the fp64 oracle, on every device variant and
at the size edges (run on an H100: `pytest -m gpu`).  Every case uploads seeded experts, evaluates `eng.bcm_nll` /
`eng.laplace_nll` and compares with `oracle.regression.bcm_objective` / `classification_likelihood_and_gradient`.
Which variant a case reaches follows from `bcm_variant` / `laplace_variant` in test_host_logic.py (the dispatch rule);
`last_bcm_path()` confirms the LU / on-chip split.

Tolerances (written here once):
  TOL_NLL   = 1e-9   objective value, relative (fp64 Cholesky / sweep / LU on the GPU vs the oracle's LU)
  gradient, per component:  |g_i - g0_i| <= RTOL_G |g0_i| + atol_i   with
    atol_i = C_BOUND eps sum_e (n_e + kappa_e) 1/2 sum_ab |dK_i[a,b]| (|alpha_a alpha_b| + |K^-1_ab|)
           (test_host_logic.gradient_atol: rounding of the pair sums, n_e terms per partial sum, and of K^-1 with
            condition number kappa_e; for an ARD beta_k, dK_i = -2 beta_k scale (x_ak - x_bk)^2 k_ab)
  RTOL_G    = 1e-12  (exp() and the final scaling: a few ulp)
  Laplace:  |g_i - g0_i| <= RTOL_LAP |g0_i| + ATOL_LAP sum_e sum_ab |dK_i[a,b]|   (|W_ab| <= 1 at the Laplace mode; the
            Newton loop stops at tol, so both sides carry the same truncated iterate), RTOL_LAP = 1e-9, ATOL_LAP = 1e-11
The old max-norm check (max|g - g0| / max|g0|) cannot see a wrong ARD component when the scale or noise derivative is
O(n) larger; the per-component check can.
"""
import json
import os
import subprocess
import sys

import numpy as np
import pytest

import oracle
import oracle.regression
import spark_gp_b200 as sg
from oracle.classification import classification_likelihood_and_gradient
from spark_gp_b200.hyperopt import group_for_experts, pack_experts
from test_host_logic import MAX_HYPERS, bcm_variant, gradient_atol, laplace_variant

pytestmark = pytest.mark.gpu

TOL_NLL, RTOL_G, RTOL_LAP, ATOL_LAP = 1e-9, 1e-12, 1e-9, 1e-11
FORCE_SMEM = os.environ.get("SGP_BCM_IMPL") == "smem"
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def eng():
    e = sg.ProjectedProcessEngine(0)
    yield e
    e.close()


def rel(a, b):
    return float(np.abs(np.asarray(a) - np.asarray(b)).max() / max(np.abs(np.asarray(b)).max(), 1e-300))


def check_components(g, g0, atol, rtol, what):
    """Per-component check; returns the largest error / allowance."""
    g, g0 = np.asarray(g), np.asarray(g0)
    err = np.abs(g - g0)
    allow = rtol * np.abs(g0) + atol
    ratio = np.where(allow > 0, err / np.where(allow > 0, allow, 1.0), np.where(err > 0, np.inf, 0.0))
    worst = int(np.argmax(ratio))
    assert ratio[worst] <= 1.0, "%s: component %d: |g - g0| = %.3e > %.3e (g0 = %.6e)" % (
        what, worst, err[worst], allow[worst], g0[worst])
    return float(ratio.max())


# ---------------- inputs --------------------------------------------------------------------------------------------
def sizes(n_max, ragged, E):
    """N for `pack_experts` giving exactly n_max points in the largest expert (ragged: half the experts one shorter)."""
    if not ragged:
        return E * n_max, n_max
    n_e = n_max - 1
    N = E * n_e + E // 2
    assert int(np.floor(N / n_e + 0.5)) == E
    return N, n_e


def layout(name, N, d, rng):
    """'standardised': N(0,1) features, ARD betas in [0.3, 3] / sqrt(d) (what L-BFGS visits); 'clustered' (adversarial):
    unit-scale structure inside clusters 300 apart, betas ~1 -- coordinates large against the distances that carry the
    kernel values.  Experts are strided samples of the whole data set, so every expert spans all clusters."""
    if name == "standardised":
        return rng.standard_normal((N, d)), rng.uniform(0.3, 3.0, d) / np.sqrt(d)
    return rng.random((N, d)) + 300.0 * rng.integers(0, 4, (N, 1)), rng.uniform(0.8, 1.2, d)


def kernel_pair(kind, d, beta, rng):
    """(GPU kernel, oracle kernel factory) of one family."""
    b2 = rng.uniform(0.3, 3.0, d) / np.sqrt(d)
    sig = 0.9 * np.sqrt(d)
    fams = {
        "ard": lambda S: 1.3 * S.ARDRBFKernel(beta) + S.const(1e-2) * S.EyeKernel(),
        "ard_noise": lambda S: 1.3 * S.ARDRBFKernel(beta) + S.WhiteNoiseKernel(0.2, 0, 1) + S.const(1e-3) * S.EyeKernel(),
        "rbf": lambda S: S.Scalar(1.5).between(0).and_(30) * S.RBFKernel(sig, 1e-6, 100) + S.WhiteNoiseKernel(0.3, 0, 1)
                         + S.const(1e-3) * S.EyeKernel(),
        "ard2": lambda S: 0.9 * S.ARDRBFKernel(beta) + 0.6 * S.ARDRBFKernel(b2) + S.const(1e-2) * S.EyeKernel(),
        "ard_rbf": lambda S: 1.3 * S.ARDRBFKernel(beta) + 0.5 * S.RBFKernel(sig) + S.const(1e-2) * S.EyeKernel(),
        "three": lambda S: 0.9 * S.ARDRBFKernel(beta) + 0.6 * S.ARDRBFKernel(b2) + 0.4 * S.RBFKernel(sig)
                           + S.const(1e-2) * S.EyeKernel(),
        "four": lambda S: 0.9 * S.ARDRBFKernel(beta) + 0.6 * S.ARDRBFKernel(b2) + 0.4 * S.RBFKernel(sig)
                          + 0.3 * S.RBFKernel(2.0 * sig) + S.WhiteNoiseKernel(0.1, 0, 1) + S.const(1e-3) * S.EyeKernel(),
        "nested": lambda S: S.Scalar(0.7).between(0).and_(10) * (1.5 * S.ARDRBFKernel(beta)
                                                                 + S.Scalar(0.4).between(0).and_(5) * S.RBFKernel(sig))
                            + S.WhiteNoiseKernel(0.2, 0, 1) + S.const(1e-3) * S.EyeKernel(),
    }
    mk = fams[kind]
    return mk(sg), (lambda: mk(oracle))


def oracle_bcm(X, y, n_e, ofac, theta):
    """(nll, gradient, per-component atol) of the oracle, summed over the experts of GPC:26-31."""
    nll0, g0, atol = 0.0, np.zeros(len(theta)), np.zeros(len(theta))
    for ye, ke in oracle.get_expert_labels_and_kernels(X, y, ofac, n_e):
        l, g = oracle.regression.regression_likelihood_and_gradient(ye, ke, theta)
        K, dK = ke.training_kernel_and_derivative()
        nll0 += l; g0 += g; atol += gradient_atol(K, dK, ye)
    return nll0, g0, atol


def n_terms_of(k):
    return sum(1 for t in k.flatten() if t["type"] != sg._native.SGP_TERM_EYE)


def run_bcm_case(eng, kind, n_max, d, ragged=False, lay="standardised", E=6, grouped=False, seed=0):
    rng = np.random.default_rng(seed + 1000 * n_max + 10 * d + len(kind))
    N, n_e = sizes(n_max, ragged, E)
    X, beta = layout(lay, N, d, rng)
    y = np.sin(X.sum(1)) + 0.3 * rng.standard_normal(N)
    k, ofac = kernel_pair(kind, d, beta, rng)
    theta = k.getHyperparameters()
    nll0, g0, atol = oracle_bcm(X, y, n_e, ofac, theta)
    if grouped:
        assert eng.experts_upload_grouped(X, y, n_e) == E
    else:
        eng.experts_upload(*pack_experts(X, y, n_e))
    nll, g = eng.bcm_nll(k)
    variant = bcm_variant(n_max, n_terms_of(k), d, FORCE_SMEM)
    assert eng.last_bcm_path() == (1 if variant == "lu" else 0)
    nll2, g2 = eng.bcm_nll(k)                                     # deterministic reduction: bit-identical
    assert nll2 == nll and np.array_equal(g2, g)
    assert len(g) == len(theta) == k.numberOfHyperparameters()
    assert abs(nll - nll0) <= TOL_NLL * abs(nll0)
    worst = check_components(g, g0, atol, RTOL_G, "%s n_max=%d d=%d %s" % (kind, n_max, d, variant))
    print("bcm %-9s %-12s n_max=%3d d=%2d %-6s %s: dnll=%.1e  grad err/bound=%.2e  old max-norm=%.1e" % (
        kind, lay, n_max, d, "ragged" if ragged else "", variant, abs(nll - nll0) / abs(nll0), worst, rel(g, g0)))
    return g, g0, atol


# ---------------- 1. variant matrix of the BCM objective, one non-Eye term ------------------------------------------------
N_MAX = [1, 2, 16, 63, 64, 65, 96, 97, 112, 113, 127, 128, 129, 168, 169]
RAGGED = {65, 97, 113, 129}                  # the largest expert one past a variant boundary, padded rows in the others


@pytest.mark.parametrize("d", [1, 16, 17, 33])
@pytest.mark.parametrize("n_max", N_MAX)
def test_bcm_one_term_ard_variants(eng, n_max, d):
    run_bcm_case(eng, "ard", n_max, d, ragged=n_max in RAGGED, E=8 if n_max == 1 else 6)


@pytest.mark.parametrize("n_max", [64, 97, 128, 129])
def test_bcm_ard_d64(eng, n_max):
    """64 ARD betas + scale + noise = 66 hyper-parameters: four ARD chunks."""
    run_bcm_case(eng, "ard_noise", n_max, 64, E=4)


@pytest.mark.parametrize("n_max,d", [(2, 1), (64, 3), (65, 5), (112, 17), (128, 8), (128, 93), (128, 100), (168, 2),
                                     (169, 3)])
def test_bcm_one_term_rbf_sigma_and_white_noise(eng, n_max, d):
    """Trainable scale, RBF sigma and WhiteNoise coefficient; (128, 93) is the widest register kernel, (128, 100) must
    fall back to the shared-memory kernel (the register kernel's shared memory would exceed 227 KB)."""
    run_bcm_case(eng, "rbf", n_max, d, ragged=(n_max == 65))


def test_bcm_grouped_upload_ragged(eng):
    """Experts grouped on the device (the fit path), ragged, at a register-kernel boundary."""
    run_bcm_case(eng, "ard", 97, 17, ragged=True, grouped=True)


# ---------------- 2. multi-term kernels: shared-memory kernel and LU path ------------------------------------------------
@pytest.mark.parametrize("kind,n_max,d", [
    ("ard2", 100, 20), ("ard2", 168, 20), ("ard2", 169, 20),        # ARD on two terms, two chunks each
    ("ard2", 110, 16), ("ard2", 111, 16),                           # rows staged / not staged (113 KB)
    ("ard_rbf", 64, 5), ("ard_rbf", 150, 17),
    ("three", 80, 6), ("four", 96, 18), ("four", 169, 4),
    ("nested", 120, 7), ("nested", 33, 17),
])
def test_bcm_multi_term(eng, kind, n_max, d):
    run_bcm_case(eng, kind, n_max, d)


def test_bcm_five_terms_refused(eng):
    rng = np.random.default_rng(1)
    X, y = rng.standard_normal((200, 3)), rng.standard_normal(200)
    eng.experts_upload(*pack_experts(X, y, 50))
    k = sum((0.5 * sg.RBFKernel(1.0 + t) for t in range(5)), sg.const(1e-2) * sg.EyeKernel())
    with pytest.raises(ValueError):
        eng.bcm_nll(k)


# ---------------- 3. per-component gradient check on an adversarial layout ---------------------------------------------
@pytest.mark.parametrize("kind,n_max,d", [("ard", 64, 4), ("ard", 100, 4), ("ard", 128, 17), ("rbf", 100, 4),
                                          ("ard2", 100, 4), ("ard", 169, 4)])
def test_bcm_clustered_layout(eng, kind, n_max, d):
    """Coordinates ~1000 against unit distances: the per-dimension sums must hold the pair-sum rounding bound on every
    variant (an expanded quadratic form of the sums cancels here by ~6 orders of magnitude)."""
    run_bcm_case(eng, kind, n_max, d, lay="clustered")


# ---------------- 4. the two fast kernels on the same inputs ------------------------------------------------------------
DIFF_CASES = [("ard", 16, 1, "standardised"), ("ard", 64, 17, "standardised"), ("ard", 97, 33, "standardised"),
              ("ard", 128, 16, "standardised"), ("rbf", 100, 5, "standardised"), ("ard", 100, 4, "clustered"),
              ("ard", 128, 17, "clustered")]


def _diff_inputs(kind, n_max, d, lay):
    rng = np.random.default_rng(500 + n_max + d)
    X, beta = layout(lay, 6 * n_max, d, rng)
    y = np.sin(X.sum(1)) + 0.3 * rng.standard_normal(len(X))
    k, ofac = kernel_pair(kind, d, beta, rng)
    return X, y, k, ofac


def _diff_eval(eng):
    out = {}
    for case in DIFF_CASES:
        X, y, k, _ = _diff_inputs(*case)
        eng.experts_upload(*pack_experts(X, y, case[1]))
        out[repr(case)] = eng.bcm_nll(k)[1].tolist()
    return out


def test_register_and_shared_memory_kernels_agree(eng, tmp_path):
    """SGP_BCM_IMPL=smem (read once per process) in a subprocess: the shared-memory sweep, which sums pair differences,
    on the inputs the register kernel gets here -- the two agree to the per-component bound of the oracle."""
    here = _diff_eval(eng)
    out = tmp_path / "smem.json"
    env = dict(os.environ, SGP_BCM_IMPL="smem", PYTHONPATH=os.pathsep.join([ROOT, os.path.dirname(__file__)]))
    r = subprocess.run([sys.executable, os.path.abspath(__file__), str(out)], env=env, cwd=ROOT, capture_output=True,
                       text=True, timeout=600)
    assert r.returncode == 0, r.stderr[-3000:]
    there = json.loads(out.read_text())
    for case in DIFF_CASES:
        X, y, k, ofac = _diff_inputs(*case)
        _, g0, atol = oracle_bcm(X, y, case[1], ofac, k.getHyperparameters())
        g_reg, g_smem = np.array(here[repr(case)]), np.array(there[repr(case)])
        worst = check_components(g_smem, g_reg, atol, RTOL_G, "register vs shared-memory kernel %r" % (case,))
        print("register vs smem %r: err/bound=%.2e" % (case, worst))


# ---------------- 5. Laplace objective ----------------------------------------------------------------------------------
def laplace_atol(experts, theta):
    atol = np.zeros(len(theta))
    for _, ke in experts:
        ke.set_hyperparameters(theta)
        _, dK = ke.training_kernel_and_derivative()
        atol += ATOL_LAP * np.array([float(np.abs(d).sum()) for d in dK])
    return atol


def run_laplace_case(eng, kind, n_max, d, E=4, tol=1e-6, seed=3):
    rng = np.random.default_rng(seed + 100 * n_max + d)
    N, n_e = sizes(n_max, False, E)
    X, beta = layout("standardised", N, d, rng)
    y = (np.sin(2 * X[:, 0]) + 0.5 * X.sum(1) / np.sqrt(d) + 0.3 * rng.standard_normal(N) > 0).astype(np.float64)
    k, ofac = kernel_pair(kind, d, beta, rng)
    experts = oracle.get_expert_labels_and_kernels(X, y, ofac, n_e)
    fs = [np.zeros(len(g)) for g in group_for_experts(N, n_e)]
    eng.experts_upload(*pack_experts(X, y, n_e))
    theta0 = k.getHyperparameters()
    worst = 0.0
    for step, theta in enumerate((theta0, theta0 * rng.uniform(0.7, 1.4, len(theta0)))):   # 2nd: warm start
        v0, g0 = 0.0, np.zeros(len(theta))
        for (ye, ke), f in zip(experts, fs):
            v, g = classification_likelihood_and_gradient(ye, f, ke, theta, tol)
            v0 += v; g0 = g0 + g
        v, g = eng.laplace_nll(k.setHyperparameters(theta), tol)
        assert abs(v - v0) <= TOL_NLL * abs(v0)
        worst = max(worst, check_components(g, g0, laplace_atol(experts, theta), RTOL_LAP,
                                            "laplace %s n_max=%d d=%d eval %d" % (kind, n_max, d, step)))
        f_gpu = eng.experts_f(N)                                    # packed expert-major, as uploaded
        f_pack = np.concatenate(fs)
        assert np.abs(f_gpu - f_pack).max() <= 1e-9 * max(1.0, np.abs(f_pack).max())
    print("laplace %-7s n_max=%3d d=%2d (%s): grad err/bound=%.2e" % (kind, n_max, d, laplace_variant(n_max, d), worst))


@pytest.mark.parametrize("kind,n_max,d", [("ard", 1, 3), ("ard", 33, 3), ("ard", 64, 5), ("ard", 100, 20),
                                          ("ard", 117, 3), ("rbf", 100, 4), ("ard_rbf", 64, 6), ("three", 80, 4),
                                          ("nested", 117, 2)])
def test_laplace_variants(eng, kind, n_max, d):
    assert laplace_variant(n_max, d) is not None
    run_laplace_case(eng, kind, n_max, d)


def test_laplace_largest_expert_refused_past_limit(eng):
    assert laplace_variant(118, 1) is None
    rng = np.random.default_rng(9)
    X = rng.standard_normal((4 * 118, 1)); y = (X[:, 0] > 0).astype(np.float64)
    eng.experts_upload(*pack_experts(X, y, 118))
    with pytest.raises(ValueError):
        eng.laplace_nll(1.0 * sg.ARDRBFKernel(np.ones(1)) + sg.const(1e-2) * sg.EyeKernel(), 1e-6)


# ---------------- 6. closed forms and limits -----------------------------------------------------------------------------
def test_bcm_experts_of_one_point(eng):
    """K = scale + s (1 x 1): nll = sum 1/2 y^2 / k + 1/2 log k, d nll / d scale = sum 1/2 (1/k - y^2/k^2), ARD: 0."""
    rng = np.random.default_rng(2)
    X, y = rng.standard_normal((8, 3)), rng.standard_normal(8)
    eng.experts_upload(*pack_experts(X, y, 1))
    k = 1.3 * sg.ARDRBFKernel(np.array([0.5, 1.0, 2.0])) + sg.const(1e-2) * sg.EyeKernel()
    nll, g = eng.bcm_nll(k)
    kk = 1.3 + 1e-2
    assert abs(nll - np.sum(0.5 * y ** 2 / kk + 0.5 * np.log(kk))) <= 1e-14 * abs(nll)
    assert abs(g[0] - np.sum(0.5 * (1.0 / kk - y ** 2 / kk ** 2))) <= 1e-14 * np.sum(0.5 * (1.0 / kk + y ** 2 / kk ** 2))
    assert np.all(g[1:] == 0.0)


def test_bcm_eye_only_kernel(eng):
    """K = s I: nll = 1/2 y'y / s + 1/2 n log s; the WhiteNoise coefficient's derivative is 1/2 sum (1/s - y^2/s^2)."""
    rng = np.random.default_rng(6)
    X, y = rng.standard_normal((600, 2)), rng.standard_normal(600)
    eng.experts_upload(*pack_experts(X, y, 100))
    k = sg.WhiteNoiseKernel(0.7, 0, 10) + sg.const(1e-3) * sg.EyeKernel()
    nll, g = eng.bcm_nll(k)
    s = 0.701
    assert eng.last_bcm_path() == 0
    assert abs(nll - (0.5 * y @ y / s + 0.5 * len(y) * np.log(s))) <= 1e-13 * abs(nll)
    want = 0.5 * np.sum(1.0 / s - y ** 2 / s ** 2)
    assert len(g) == 1 and abs(g[0] - want) <= 1e-13 * np.sum(0.5 * (1.0 / s + y ** 2 / s ** 2))


def test_bcm_hyper_parameter_limit(eng):
    """MAX_HYPERS = 72: scale + 71 ARD betas are evaluated (five ARD chunks, checked on the oracle); one more refused."""
    assert 1 + 71 == MAX_HYPERS
    run_bcm_case(eng, "ard", 40, 71, E=4)
    rng = np.random.default_rng(4)
    X, y = rng.standard_normal((160, 72)), rng.standard_normal(160)
    eng.experts_upload(*pack_experts(X, y, 40))
    with pytest.raises(ValueError):
        eng.bcm_nll(1.3 * sg.ARDRBFKernel(np.full(72, 0.1)) + sg.const(1e-2) * sg.EyeKernel())


if __name__ == "__main__":             # the subprocess of test_register_and_shared_memory_kernels_agree
    e = sg.ProjectedProcessEngine(0)
    with open(sys.argv[1], "w") as fh:
        json.dump(_diff_eval(e), fh)
    e.close()
