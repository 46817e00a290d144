"""Prediction (`sgp_predict`, `sgp_predict_probability` and their device entries, csrc/predict.cu) element by element:
every kernel element, mean, variance and averaged probability within its own rounding bound (oracle/predict_model.py;
tests/test_host_predict_model.py shows the bounds sharp).  Run on an H100: `pytest -m gpu`.

The flat gates of test_gpu_predict.py and test_gpu_probability.py (1e-11 of the summed magnitudes, 3e-14 absolute for
p) are 20 to 10 000 times looser than the rounding of these sums, and say nothing about probabilities below 1e-12 --
the confident negatives whose ranking the binary evaluator and one-vs-rest depend on.  Every case here prints the
largest fraction of the bound used, the rounding counts R_mean and R_var, and the reference's own share of the gate;
it fails above a fraction of 1 or a share of 1/8.  The probability is judged on the device's own (mean, var) with the
library's own rule, so that only the probability kernel's arithmetic is measured.
"""
import os

import numpy as np
import pytest
import torch

import oracle
import spark_gp_b200 as sg
from oracle.predict_model import (LD, SAMPLE_WORK, PredictModel, bound_fraction, fractions, m_padded, probability,
                                  probability_fraction, reference_share, sample_points)
from spark_gp_b200 import _native as N
from spark_gp_b200.regression import ExplicitActiveSetProvider
from test_gpu_predict import install, make_case, points, predict_dev
from test_gpu_probability import prob_dev, same
from test_host_predict_model import far, shifted

pytestmark = pytest.mark.gpu

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
NODES = [1, 2, 100, 256]
KPREDICT_BYTES = 256 << 20                    # kPredictKBytes, sgp_internal.h


@pytest.fixture(scope="module")
def eng():
    e = sg.ProjectedProcessEngine(0)
    yield e
    e.close()


def rule(nodes):
    return sg.ProjectedProcessEngine.gauss_hermite_rule(nodes)


def window_points(m):
    """predict_window_points: the points of one kernel window."""
    return max(128, KPREDICT_BYTES // (m_padded(m) * 8) // 128 * 128)


def windows(n, size):
    return [(w0, min(size, n - w0)) for w0 in range(0, n, size)]


def judge(label, k0, Z, v, M, X, mean, var, rows=None):
    """Mean and variance of the points `rows` of X against the model; returns the model statistics."""
    if rows is None:
        assert len(X) * len(Z) ** 2 <= SAMPLE_WORK                # else the caller passes sample_points
        rows = np.arange(len(X))
    model = PredictModel(k0, Z, v, M)
    st = model.predict(X[rows], with_var=var is not None)
    fm, fv = fractions(st, mean[rows], var[rows] if var is not None else None)
    share = reference_share(st)
    print("%s: mean %.3g var %.3g of the bound, R_mean %d R_var %d, %d of %d points, reference %.1e of the bound" % (
        label, fm, fv, model.R_mean, model.R_var, len(rows), len(X), share))
    assert share < 0.125
    assert fm <= 1.0 and fv <= 1.0
    return st


def judge_p(label, p, mean, var, nodes):
    x, w = rule(nodes)
    prob = probability(mean, var, x, w)
    f = probability_fraction(p, prob)
    share = float(np.max(prob[2] / prob[1])) if len(p) else 0.0
    print("%s: p %.3g of the bound (%d nodes), smallest p %.1e, reference %.1e of the bound" % (
        label, f, nodes, float(np.min(p)) if len(p) else 0.0, share))
    assert share < 0.125
    assert f <= 1.0


# ---------------- element probes: the mean-only call with v = e_j returns column j of K bit for bit -------------------
DBL_MIN = 2.2250738585072014e-308


def probe_columns(eng, c, X, cols, label):
    """Each fma with v_j = 0 and each add of 0 is exact, so the mean of v = e_j is k(x, z_j) itself: the columns `cols`
    of K through the host and device entries from fp64 input and the device entry from fp32 input, each element judged
    against its bound.  Returns the probed columns (fp64 input) as the device computed them."""
    m = c["m"]
    X32 = X.astype(np.float32)
    model = PredictModel(c["k0"], c["Z"], c["v"], c["M"])
    K, a, e = model.elements(X)
    K32, a32, e32 = model.elements(X32.astype(np.float64))
    install(eng, c)
    got, worst = [], 0.0
    for j in cols:
        v = np.zeros(m)
        v[j] = 1.0
        eng.set_magic(v, np.zeros((m, m)))
        hm, _ = eng.predict(X, with_variance=False)
        dm, _ = predict_dev(eng, X, with_var=False)
        fm, _ = predict_dev(eng, X32, with_var=False, f32=True)
        assert same(hm, dm)
        f = max(bound_fraction(hm, K[:, j], a[:, j] + e[:, j]), bound_fraction(fm, K32[:, j], a32[:, j] + e32[:, j]))
        worst = max(worst, f)
        assert f <= 1.0, j
        got.append(hm)
    got = np.stack(got, axis=1)
    print("%s: %d columns, elements %.3g of the bound; %d zeros, %d subnormals" % (
        label, len(cols), worst, int((got == 0).sum()), int(((got > 0) & (got < DBL_MIN)).sum())))
    return got


def probe_set(m, rng):
    """The first and last column of every 64-column tile (so of every 128-column element tile) and 6 random columns."""
    return sorted({j for t0 in range(0, m, 64) for j in (t0, min(t0 + 63, m - 1))} | set(rng.integers(0, m, 6).tolist()))


@pytest.mark.parametrize("m,d,terms", [(257, 65, 2), (256, 32, 4), (129, 5, 1)])
def test_element_probes(eng, m, d, terms):
    """Near and far points: the probed elements reach fp64's subnormal range and 0."""
    c = make_case(m, d, terms, seed=m + d)
    X = np.concatenate([points(c, 90), far(c, 60, m)])
    got = probe_columns(eng, c, X, probe_set(m, np.random.default_rng(m)), "m=%d d=%d terms=%d" % (m, d, terms))
    assert (got == 0).any() and ((got > 0) & (got < DBL_MIN)).any()


# ---------------- mean, variance and p at every tile, group and window edge ---------------------------------------------
NS = [15, 16, 17, 31, 32, 33, 127, 128, 129, 255, 256, 257]


def run_entries(eng, X, nodes, f32=False):
    """(mean, var, p) of the host entries and of the device entries (fp32 or fp64 input); the two agree bit for bit."""
    if f32:
        hm = hv = hp = None
    else:
        hm, hv = eng.predict(X)
        hp, pm, pv = eng.predict_probability(X, nodes, with_mean_var=True)
        assert same(pm, hm) and same(pv, hv)
    dm, dv = predict_dev(eng, X, f32=f32)
    dp, qm, qv = prob_dev(eng, X, nodes, f32=f32)
    assert same(qm, dm) and same(qv, dv)
    if not f32:
        assert same(dm, hm) and same(dv, hv) and same(dp, hp)
    return dm, dv, dp


def check_case(eng, c, X, nodes, label):
    """Installs the case's pair and judges mean, variance and p of every point, from fp64 input through both entries
    and from fp32 input through the device entry; returns the fp64 input's (mean, var, p)."""
    install(eng, c)
    out = None
    for kind, Xi, f32 in (("fp64", X, False), ("fp32", X.astype(np.float32), True)):
        mean, var, p = run_entries(eng, Xi, nodes, f32)
        judge("%s %s" % (label, kind), c["k0"], c["Z"], c["v"], c["M"], Xi.astype(np.float64), mean, var)
        judge_p("   ", p, mean, var, nodes)
        if not f32:
            out = (mean, var, p)
    return out


@pytest.mark.parametrize("n", NS)
def test_edges_within_bound(eng, n):
    """n at the 16-point groups, the 32-point element CTA and the 128-row variance tile; m at 255, 256, 257 (the 64- and
    128-wide tile edges); d at 32, 64, 65 (the 32-dim staging chunk); 1 to 4 terms; every other case with variances
    straddling 0."""
    i = NS.index(n)
    m, d, terms, nodes = (255, 256, 257)[i % 3], (32, 64, 65)[(i // 3) % 3], 1 + i % 4, NODES[i % 4]
    c = make_case(m, d, terms, seed=100 + i)
    X = points(c, n, seed=i)
    if i % 2:
        c = shifted(c, X)
    _, var, _ = check_case(eng, c, X, nodes, "n=%d m=%d d=%d terms=%d" % (n, m, d, terms))
    if i % 2:
        assert (var < 0).any() and (var > 0).any()


@pytest.mark.parametrize("n,m,d", [(1, 1, 1), (1, 65, 5), (40, 1, 3), (200, 129, 100)])
def test_small_and_wide_within_bound(eng, n, m, d):
    """The remaining edges of test_gpu_predict.py: one point, one active point, one dimension, and d = 100."""
    c = make_case(m, d, 1 + d % 4, seed=1000 + n + m + d)
    check_case(eng, c, points(c, n, seed=d), 100, "n=%d m=%d d=%d" % (n, m, d))


def test_asymmetric_matrix_within_bound(eng):
    """The M of test_asymmetric_matrix in test_gpu_predict.py: the packing rounds M_ij + M_ji."""
    c = make_case(300, 6, 2, seed=77)
    E = np.random.default_rng(5).standard_normal(c["M"].shape) * 50.0
    c = dict(c, M=c["M"] + (E - E.T))
    M, Ml = c["M"], c["M"].astype(LD)
    assert (np.triu(M + M.T, 1).astype(LD) != np.triu(Ml + Ml.T, 1)).any()      # pack roundings occur
    check_case(eng, c, points(c, 400), 100, "asymmetric M")


# ---------------- placement: data far from the origin, where only the centre keeps the staging exact -------------------
PLACEMENTS = ["0", "10", "100", "1e3", "-1e3", "1e3_one_dim"]


def placed(where, d=4):
    """The case of test_placement in test_gpu_predict.py: length scales ~ sqrt d, the data `where` of them out."""
    off = np.zeros(d)
    if where == "1e3_one_dim":
        off[0] = 1e3 * np.sqrt(d)
    else:
        off[:] = float(where) * np.sqrt(d)
    return make_case(150, d, 2, seed=21, offset=off)


@pytest.mark.parametrize("where", PLACEMENTS)
def test_placement_within_bound(eng, where):
    """Staged without the centre, the 1e3 placements miss the element bound 286 times over (test_host_predict_model.py);
    here the probed elements, the mean, the variance and p of 300 points, through both entries and both input types."""
    c = placed(where)
    X = points(c, 300)
    probe_columns(eng, c, X, probe_set(c["m"], np.random.default_rng(21)), "placement %s" % where)
    check_case(eng, c, X, 100, "placement %s" % where)


@pytest.mark.parametrize("n,m,d", [(5351, 65, 784), (8193, 4000, 8)])
def test_window_edges_within_bound(eng, n, m, d):
    """The host entry's staging chunk (d = 784: 5349 points) and the kernel window (m = 4000: 8192 points), on sampled
    points including the first and last of every window."""
    c = make_case(m, d, 2, seed=n)
    install(eng, c)
    X = points(c, n)
    mean, var, p = run_entries(eng, X, 100)
    chunk = min(max(4096, (32 << 20) // (d * 8)), window_points(m), n)
    wins = windows(n, chunk) + windows(n, window_points(m))
    rows = sample_points(n, np.random.default_rng(n), wins, 24)
    judge("window n=%d m=%d d=%d" % (n, m, d), c["k0"], c["Z"], c["v"], c["M"], X, mean, var, rows)
    judge_p("   ", p[rows], mean[rows], var[rows], 100)


# ---------------- magic pairs from fits: variances that are small differences of large terms ----------------------------
def test_airfoil_regression_tail(eng):
    """The strict statistics and tail of the airfoil fixture (m = 1000, cond(A) ~ 6e7), then its 150 test points."""
    c = np.load(os.path.join(GOLD, "airfoil_case.npz"))
    kernel = 1 * sg.ARDRBFKernel(5) + sg.const(1) * sg.EyeKernel() + sg.const(float(c["sigma2"])) * sg.EyeKernel()
    kernel.setHyperparameters(c["theta"])
    k0 = (1 * oracle.ARDRBFKernel(5) + oracle.const(1) * oracle.EyeKernel()
          + oracle.const(float(c["sigma2"])) * oracle.EyeKernel())
    k0 = k0.set_hyperparameters(c["theta"]).set_training_vectors(c["Z"])
    eng.set_precision(N.SGP_PREC_F64_STRICT)
    eng.begin(kernel, c["Z"])
    eng.accumulate(c["X"], c["y"])
    eng.finish()
    v, M = eng.magic()
    X = np.ascontiguousarray(c["Xtest"])
    mean, var, p = run_entries(eng, X, 100)
    st = judge("airfoil", k0, c["Z"], v, M, X, mean, var)
    print("   var / selfKernel from %.1e" % float(np.min(st["var"]) / float(k0.self_kernel(None))))
    judge_p("   ", p, mean, var, 100)


def test_mnist68_classifier():
    """The binary classifier of test_gpu_probability.py on mnist 6 vs 8 (d = 784, m = 500).  Its latent means are small,
    so its test probabilities stay between about 0.2 and 0.8, on both sides of 0.5; test_probability_tails covers the
    tails."""
    c = np.load(os.path.join(GOLD, "mnist68_case.npz"))
    n = int(c["n_rows"])
    X = (c["pixels"].astype(np.float64) - c["mean"]) / c["std"]
    Xtr, Xte, ytr = X[:n], X[n:n + 100], c["y01"][:n]
    sigma = float(c["sigma"])
    gp = (sg.GaussianProcessClassifier().setDatasetSizeForExpert(100).setActiveSetSize(500)
          .setKernel(lambda: sg.RBFKernel(sigma)).setTol(1e-3)
          .setActiveSetProvider(ExplicitActiveSetProvider(Xtr[c["active_idx"]])))
    model = gp.fit(Xtr, ytr, hyperparameters=np.array([sigma]))
    rp = model.rawPredictor
    Z = np.asarray(rp.activeSet)
    k0 = (oracle.RBFKernel(sigma) + oracle.const(1e-3) * oracle.EyeKernel())
    k0 = k0.set_hyperparameters(model.hyperparameters).set_training_vectors(Z)
    e = rp._engine
    mean, var = e.predict(Xte)
    judge("mnist68", k0, Z, rp.magicVector, rp.magicMatrix, Xte, mean, var)
    for nodes in NODES:
        p, pm, pv = e.predict_probability(Xte, nodes, with_mean_var=True)
        assert same(pm, mean) and same(pv, var)
        judge_p("   ", p, mean, var, nodes)
        assert p.min() < 0.5 < p.max()


# ---------------- probability tails ----------------------------------------------------------------------------------------
@pytest.mark.parametrize("nodes", NODES)
def test_probability_tails(eng, nodes):
    """Means pushed from -740 to +40 by scaling v, variances from below 0 (clamped) to 1e4 by M = alpha I."""
    c = make_case(130, 4, 2, seed=70)
    X = points(c, 256)
    K0 = c["k0"].cross_kernel(X)
    ksum, k2 = np.median(K0.sum(1)), np.median((K0 * K0).sum(1))
    sk = c["k0"].self_kernel(None)
    worst_low = 1.0
    for target in (-740.0, -400.0, -100.0, -30.0, -5.0, 5.0, 40.0):
        for var_target in (-1.0, 0.0, 1e-2, 1e2, 1e4):
            v = np.full(c["m"], target / ksum)
            M = np.eye(c["m"]) * (var_target - sk) / k2
            install(eng, dict(c, v=v), M=M)
            p, mean, var = eng.predict_probability(X, nodes, with_mean_var=True)
            dp, _, _ = prob_dev(eng, X, nodes)
            assert same(dp, p)
            judge_p("mean ~ %g, var ~ %g" % (target, var_target), p, mean, var, nodes)
            worst_low = min(worst_low, float(p.min()))
    assert worst_low < 1e-300                                  # the left tail reaches fp64's subnormal range and 0


# ---------------- scale ----------------------------------------------------------------------------------------------------
def test_scale_1p3m(eng):
    """The 1.3M-point case of test_gpu_predict.py: 40 kernel windows of 32768 points, judged on sampled points."""
    c = make_case(1000, 16, 1, seed=31)
    install(eng, c)
    n = 1_300_000
    Xd = torch.rand((n, 16), dtype=torch.float64, device="cuda", generator=torch.Generator("cuda").manual_seed(7)) * 2.0
    mean, var = eng.predict_tensor(Xd)
    p, pm, pv = eng.predict_probability_tensor(Xd, nodes=100, with_mean_var=True)
    assert torch.equal(pm, mean) and torch.equal(pv, var)
    rows = sample_points(n, np.random.default_rng(3), windows(n, window_points(1000)), 64)
    idx = torch.from_numpy(rows).cuda()
    X = Xd[idx].cpu().numpy()
    mean, var, p = (t[idx].cpu().numpy() for t in (mean, var, p))
    judge("1.3M points", c["k0"], c["Z"], c["v"], c["M"], X, mean, var)
    judge_p("   ", p, mean, var, 100)
