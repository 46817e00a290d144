"""Host-side mirror of the reference's kernel DSL / Params (no GPU needed): hyperparameter layout,
bounds, flattening into the C-ABI term list -- checked against the oracle's restatement."""
import numpy as np
import pytest

import oracle
import spark_gp_b200 as sg
from spark_gp_b200 import _native as N


def _pairs():
    return [
        (lambda: 1 * sg.ARDRBFKernel(5) + sg.const(1) * sg.EyeKernel(),
         lambda: 1 * oracle.ARDRBFKernel(5) + oracle.const(1) * oracle.EyeKernel()),
        (lambda: sg.Scalar(1.0).between(0).and_(30) * sg.RBFKernel(0.1, 1e-6, 10) + sg.WhiteNoiseKernel(0.5, 0, 1),
         lambda: oracle.Scalar(1.0).between(0).and_(30) * oracle.RBFKernel(0.1, 1e-6, 10) + oracle.WhiteNoiseKernel(0.5, 0, 1)),
        (lambda: sg.RBFKernel(10), lambda: oracle.RBFKernel(10)),
        (lambda: 2.0 * (1.5 * sg.ARDRBFKernel(np.array([0.2, 0.3])) + sg.const(0.5) * sg.EyeKernel()),
         lambda: 2.0 * (1.5 * oracle.ARDRBFKernel(np.array([0.2, 0.3])) + oracle.const(0.5) * oracle.EyeKernel())),
    ]


@pytest.mark.parametrize("idx", range(4))
def test_dsl_matches_oracle(idx):
    mk, mo = _pairs()[idx]
    k, o = mk(), mo()
    assert np.allclose(k.getHyperparameters(), o.get_hyperparameters())
    assert k.numberOfHyperparameters() == o.number_of_hyperparameters()
    for a, b in zip(k.hyperparameterBoundaries(), o.hyperparameter_boundaries()):
        assert np.array_equal(a, b)
    assert np.isclose(k.whiteNoiseVar, o.white_noise_var)
    theta = k.getHyperparameters() * 1.7 + 0.01
    k.setHyperparameters(theta); o.set_hyperparameters(theta)
    assert np.allclose(k.getHyperparameters(), o.get_hyperparameters())
    assert np.isclose(k.whiteNoiseVar, o.white_noise_var)
    assert str(k) == str(o)
    # self kernel = sum of every leaf's scale (each leaf has k(x,x)=1)
    assert np.isclose(sum(t["scale"] for t in k.flatten()), o.self_kernel(np.zeros(5)))


def test_flatten_scales_multiply_through_nesting():
    k = 2.0 * (1.5 * sg.ARDRBFKernel(np.array([0.2, 0.3])) + sg.const(0.5) * sg.EyeKernel())
    t = k.flatten()
    assert [x["type"] for x in t] == [N.SGP_TERM_ARD, N.SGP_TERM_EYE]
    assert np.isclose(t[0]["scale"], 3.0) and np.isclose(t[1]["scale"], 1.0)
    assert np.allclose(k.getHyperparameters(), [2.0, 1.5, 0.2, 0.3])


def test_params_defaults_and_getkernel():
    gp = sg.GaussianProcessRegression()
    assert (gp._datasetSizeForExpert, gp._activeSetSize, gp._sigma2, gp._maxIter, gp._tol) == (100, 100, 1e-3, 100, 1e-6)
    k = gp.setSigma2(1e-4).setKernel(lambda: 1 * sg.ARDRBFKernel(5) + sg.const(1) * sg.EyeKernel()).getKernel()
    assert np.isclose(k.whiteNoiseVar, 1.0001)            # GPC:18 appends sigma2.const * Eye
    assert len(k.getHyperparameters()) == 6
    with pytest.raises(ValueError):
        sg.Scalar(-1.0) * sg.RBFKernel()
    with pytest.raises(ValueError):
        sg.Scalar(1.0, 2.0, 1.0)


# ---- hyper-parameter descriptors (what sgp_bcm_nll consumes) vs the oracle's trainingKernelAndDerivative ------------
def _dense_from_descriptors(k, X):
    """K and dK/dtheta_i rebuilt in numpy from (flatten(), hyper_descriptors()) exactly as csrc/bcm_nll.cu does."""
    terms = k.flatten()
    n, d = X.shape
    kt, sq = [], []
    for t in terms:
        if t["type"] == N.SGP_TERM_EYE:
            kt.append(np.eye(n)); sq.append(np.zeros((n, n))); continue
        beta = t["beta"] if t["type"] == N.SGP_TERM_ARD else np.full(d, 1.0 / (np.sqrt(2.0) * t["sigma"]))
        diff = X[:, None, :] - X[None, :, :]
        kt.append(np.exp(-((diff * beta) ** 2).sum(2))); sq.append((diff ** 2).sum(2))
    K = sum(t["scale"] * m for t, m in zip(terms, kt))
    dK = []
    for h in k.hyper_descriptors():
        if h["kind"] == N.SGP_HYPER_SCALE:
            dK.append(sum(c * kt[t] for t, c in h["coef"].items()))
        elif h["kind"] == N.SGP_HYPER_ARD_BETA:
            t, kk = h["term"], h["dim"]
            dx2 = (X[:, None, kk] - X[None, :, kk]) ** 2
            dK.append(terms[t]["scale"] * (-2.0 * h["value"] * dx2) * kt[t])
        else:
            t = h["term"]
            dK.append(terms[t]["scale"] * sq[t] * kt[t] / h["value"] ** 3)
    return K, dK


@pytest.mark.parametrize("idx", range(5))
def test_hyper_descriptors_match_oracle_derivatives(idx):
    pairs = _pairs() + [
        (lambda: 0.7 * (1.5 * sg.ARDRBFKernel(np.full(5, 0.9)) + 0.5 * sg.RBFKernel(2.0)) + sg.WhiteNoiseKernel(0.4, 0, 1) + sg.const(0.2) * sg.EyeKernel(),
         lambda: 0.7 * (1.5 * oracle.ARDRBFKernel(np.full(5, 0.9)) + 0.5 * oracle.RBFKernel(2.0)) + oracle.WhiteNoiseKernel(0.4, 0, 1) + oracle.const(0.2) * oracle.EyeKernel())]
    mk, mo = pairs[idx]
    k, o = mk(), mo()
    d = 2 if idx == 3 else 5
    X = np.random.default_rng(idx).random((9, d))
    K, dK = _dense_from_descriptors(k, X)
    K0, dK0 = o.set_training_vectors(X).training_kernel_and_derivative()
    assert len(dK) == len(dK0) == k.numberOfHyperparameters()
    assert np.allclose(K, K0, rtol=1e-13, atol=1e-15)
    for a, b in zip(dK, dK0):
        assert np.allclose(a, b, rtol=1e-12, atol=1e-14)


@pytest.mark.parametrize("idx", range(5))
def test_descriptor_gradient_from_pair_sums(idx):
    """csrc/expert_common.cuh: sum_ab dK_i[a,b] W_ab for a symmetric W from ONE lower-triangle sweep of pair sums
    (S_t, Q_t, D_tk per non-Eye term, trW) -- the algebra both objective kernels use -- vs the oracle's dense dK_i."""
    pairs = _pairs() + [
        (lambda: 0.7 * (1.5 * sg.ARDRBFKernel(np.full(5, 0.9)) + 0.5 * sg.RBFKernel(2.0)) + sg.WhiteNoiseKernel(0.4, 0, 1) + sg.const(0.2) * sg.EyeKernel(),
         lambda: 0.7 * (1.5 * oracle.ARDRBFKernel(np.full(5, 0.9)) + 0.5 * oracle.RBFKernel(2.0)) + oracle.WhiteNoiseKernel(0.4, 0, 1) + oracle.const(0.2) * oracle.EyeKernel())]
    mk, mo = pairs[idx]
    k, o = mk(), mo()
    d = 2 if idx == 3 else 5
    rng = np.random.default_rng(10 + idx)
    n = 11
    X = rng.random((n, d))
    A = rng.standard_normal((n, n)); W = A + A.T
    _, dK0 = o.set_training_vectors(X).training_kernel_and_derivative()
    terms = k.flatten()
    tri = [(a, b) for a in range(n) for b in range(a + 1)]
    w2 = {(a, b): (1.0 if a == b else 2.0) * W[a, b] for a, b in tri}
    S, Q, D = {}, {}, {}
    for t, term in enumerate(terms):
        if term["type"] == N.SGP_TERM_EYE:
            continue
        beta = term["beta"] if term["type"] == N.SGP_TERM_ARD else np.full(d, 1.0 / (np.sqrt(2.0) * term["sigma"]))
        S[t], Q[t], D[t] = 0.0, 0.0, np.zeros(d)
        for a, b in tri:
            dx = X[a] - X[b]
            kw = np.exp(-((dx * beta) ** 2).sum()) * w2[(a, b)]
            S[t] += kw; Q[t] += (dx ** 2).sum() * kw; D[t] += dx ** 2 * kw
    trW = np.trace(W)
    hd = k.hyper_descriptors()
    assert len(hd) == len(dK0)
    for h, dk in zip(hd, dK0):
        if h["kind"] == N.SGP_HYPER_SCALE:
            g = sum(c * (trW if terms[t]["type"] == N.SGP_TERM_EYE else S[t]) for t, c in h["coef"].items())
        elif h["kind"] == N.SGP_HYPER_ARD_BETA:
            g = terms[h["term"]]["scale"] * (-2.0 * h["value"]) * D[h["term"]][h["dim"]]
        else:
            g = terms[h["term"]]["scale"] * Q[h["term"]] / h["value"] ** 3
        g0 = float((dk * W).sum())
        assert abs(g - g0) <= 1e-12 * max(1.0, abs(g0))


def test_expert_packing_matches_reference_grouping():
    from spark_gp_b200.hyperopt import group_for_experts, pack_experts
    for n, ne in ((1503, 100), (150, 100), (1000, 100), (999, 37)):
        g1, g0 = group_for_experts(n, ne), oracle.group_for_experts(n, ne)
        assert len(g1) == len(g0) and all(np.array_equal(a, b) for a, b in zip(g1, g0))
    X = np.arange(30.0).reshape(15, 2); y = np.arange(15.0)
    Xp, yp, off = pack_experts(X, y, 5)                     # E = 3 experts: points i % 3
    assert list(off) == [0, 5, 10, 15]
    assert np.array_equal(yp[:5], [0, 3, 6, 9, 12]) and np.array_equal(Xp[5], X[1])
    with pytest.raises(ZeroDivisionError):
        group_for_experts(40, 100)


def test_greedy_provider_selection_matches_scalar_fold():
    """GreedilyOptimizingActiveSetProvider.select_index (vectorised) vs the oracle's transcription of the reference's
    per-expert foldLeft + filter(!isNaN) + max (ActiveSetProvider.scala:108-135)."""
    from oracle.active_set import _fold_expert
    rng = np.random.default_rng(2)
    for trial in range(200):
        n = int(rng.integers(5, 90)); E = int(rng.integers(1, 9))
        delta = np.round(rng.standard_normal(n), 1)                 # coarse values: plenty of ties
        if trial % 3 == 0:
            delta[rng.integers(n)] = np.nan
        best = None
        for e in range(E):
            md, mi = _fold_expert(delta[e::E])
            if np.isnan(md) or mi < 0:
                continue
            if best is None or not (best[0] >= md):
                best = (md, mi * E + e)
        if best is None:
            with pytest.raises(ValueError):
                sg.GreedilyOptimizingActiveSetProvider.select_index(delta, E)
        else:
            assert sg.GreedilyOptimizingActiveSetProvider.select_index(delta, E) == best[1]


def test_classification_model_surface_matches_reference_semantics():
    """predictRaw / probability / prediction of GaussianProcessClassificationModel (GPCls:136-162 + Spark's
    raw2prediction) through a stub predictor, against the oracle's restatement."""
    from oracle.classification import classification_model_outputs
    from spark_gp_b200.classification import GaussianProcessClassificationModel

    class _Engine:
        def __init__(self, f): self.f = f
        def predict(self, X, with_variance=True): return self.f[:len(X)], None

    class _Raw:
        def __init__(self, f): self._engine = _Engine(f)

    f = np.array([-3.0, -0.2, 0.0, 0.4, 5.0])
    model = GaussianProcessClassificationModel(_Raw(f), np.zeros(1))
    raw0, prob0, pred0 = classification_model_outputs(f)
    X = np.zeros((len(f), 2))
    assert np.array_equal(model.predictRaw(X), raw0)
    assert np.allclose(model.predictProbability(X), prob0, rtol=0, atol=1e-16)
    assert np.array_equal(model.predict(X), pred0)
    assert list(pred0) == [0.0, 0.0, 0.0, 1.0, 1.0]                      # f == 0: argmax takes the first maximum
    assert prob0[3, 0] > 0.5 and pred0[3] == 1.0                        # the quirk: P(class 0) = sigmoid(f) > 1/2, label 1


def test_kmeans_active_set_provider():
    """ActiveSetProvider.scala:22-46: centroids of K-means on the features (host-side library call, as in the reference)."""
    rng = np.random.default_rng(0)
    centres = rng.random((5, 3)) * 10
    X = np.concatenate([c + 0.05 * rng.standard_normal((40, 3)) for c in centres])
    prov = sg.KMeansActiveSetProvider(maxIter=20)
    A = prov(5, X, None, None, None, 13)
    assert A.shape == (5, 3) and A.dtype == np.float64 and A.flags["C_CONTIGUOUS"]
    assert np.array_equal(A, prov(5, X, None, None, None, 13))                    # same seed, same centroids
    d = np.linalg.norm(A[:, None, :] - centres[None, :, :], axis=2)
    assert np.all(d.min(axis=0) < 0.05)                                           # every true centre is recovered
    assert sg.KMeansActiveSetProvider().maxIter == 20                             # the reference's default


def test_scale_matches_oracle():
    X = np.random.default_rng(1).random((50, 4)) * [1.0, 10.0, 0.0, 3.0] + [0.0, 5.0, 2.0, -1.0]   # column 2 is constant
    got, want = sg.scale(X), oracle.scale(X)
    assert np.array_equal(got, want)
    assert np.allclose(got.mean(0), 0.0, atol=1e-14) and np.allclose(got[:, [0, 1, 3]].std(0), 1.0) and np.all(got[:, 2] == 0.0)


def test_greedy_rank1_update_identities():
    """The algebra of csrc/greedy.cu restated in NumPy and checked against the reference's per-round quantities
    (oracle.active_set: inv(K_mm), inv(s2 K_mm + G), magic vector; p_i, q_i, mu_i of ASP:109-113): adding one active point
    borders K_mm and A = s2 K_mm + G, so
        p_i' = p_i + (u~.k_i - k*_i)^2 / s~,   q_i' = q_i + (u.k_i - k*_i)^2 / s,   mu_i' = mu_i + a (u.k_i - k*_i)
    with u~ = inv(K_mm) c, s~ = kii - c.u~, u = inv(A) w, w = s2 c + K_mn k*, s = s2 kii + k*.k* - w.u, a = (u.b - k*.y) / s."""
    rng = np.random.default_rng(9)
    n, d, rounds = 400, 3, 12
    X = rng.random((n, d)); y = np.sin(3 * X.sum(1)) + 0.1 * rng.standard_normal(n)
    beta = np.full(d, 2.5)
    kern = lambda: 1.2 * oracle.ARDRBFKernel(beta) + oracle.const(0.3) * oracle.EyeKernel()
    k0 = kern()
    s2 = k0.white_noise_var
    kii = 1.2 + 0.3                                               # trainingKernelDiag: every leaf has k(x, x) = 1
    picks = rng.permutation(n)[:rounds]
    Kt = np.zeros((0, n)); Kinv = np.zeros((0, 0)); Ainv = np.zeros((0, 0)); b = np.zeros(0); mv = np.zeros(0)
    p = np.zeros(n); q = np.zeros(n); mu = np.zeros(n)
    for r, idx in enumerate(picks):
        kstar = kern().set_training_vectors(X[[idx]]).cross_kernel(X)[:, 0]      # k(x_i, x_idx) for every point i
        m = len(Kt)
        c = Kt[:, idx] if m else np.zeros(0)
        g = Kt @ kstar if m else np.zeros(0)
        gamma, bnew = kstar @ kstar, kstar @ y
        ut = Kinv @ c if m else np.zeros(0)
        w = s2 * c + g
        u = Ainv @ w if m else np.zeros(0)
        s1 = kii - c @ ut
        s = s2 * kii + gamma - w @ u
        a = ((u @ b) - bnew) / s
        t1 = Kt.T @ ut if m else np.zeros(n)
        t2 = Kt.T @ u if m else np.zeros(n)
        p += (t1 - kstar) ** 2 / s1; q += (t2 - kstar) ** 2 / s; mu += a * (t2 - kstar)
        # bordered inverses
        def border(inv, v, sc):
            out = np.zeros((m + 1, m + 1))
            out[:m, :m] = inv + np.outer(v, v) / sc
            out[:m, m] = out[m, :m] = -v / sc
            out[m, m] = 1.0 / sc
            return out
        Kinv, Ainv = border(Kinv, ut, s1), border(Ainv, u, s)
        mv = np.concatenate([mv + u * a, [-a]]); b = np.concatenate([b, [bnew]])
        Kt = np.vstack([Kt, kstar])
        # the reference's quantities for this active set, from scratch
        active = X[picks[:r + 1]]
        inst = kern().set_training_vectors(active)
        kmm = inst.training_kernel()
        cross = inst.cross_kernel(X).T                            # m x n (crossKernel: rows = test vectors, Kernel.scala:69-74)
        G = cross @ cross.T
        A = s2 * kmm + G
        assert np.allclose(Kinv, np.linalg.inv(kmm), rtol=1e-8, atol=1e-10)
        assert np.allclose(Ainv, np.linalg.inv(A), rtol=1e-7, atol=1e-12)
        assert np.allclose(mv, np.linalg.solve(A, cross @ y), rtol=1e-7, atol=1e-12)
        assert np.allclose(p, np.einsum("ji,jk,ki->i", cross, np.linalg.inv(kmm), cross), rtol=1e-8, atol=1e-12)
        assert np.allclose(q, np.einsum("ji,jk,ki->i", cross, np.linalg.inv(A), cross), rtol=1e-7, atol=1e-12)
        assert np.allclose(mu, cross.T @ np.linalg.solve(A, cross @ y), rtol=1e-7, atol=1e-12)


# ---- which device kernel evaluates a per-expert objective (tests/test_gpu_objectives.py is built on this rule) -------
# The rule is plan_objective (csrc/bcm_nll.cu); sgp_bcm_nll and sgp_laplace_nll launch what it returns.  BCM: experts
# whose shared-memory Cholesky does not fit (bcm_nll_smem_bytes > 227 KB) take the global-memory LU path; one non-Eye
# term and n_max <= 128 run the register kernel (template shape by 16-row blocks) unless its shared memory exceeds
# 227 KB; otherwise the shared-memory kernel runs, and stages the expert's rows when two CTAs per SM still fit (113 KB
# each).  Laplace: refused when laplace_smem_bytes > 227 KB, rows staged when they fit beside it.  A Cholesky pivot <= 0
# also sends sgp_bcm_nll to the LU path (not modelled: SPD inputs only), whose kernel stages the rows up to 200 KB.
K_MAX_TERMS, DCH = 4, 16
EX_SUMS = 2 * K_MAX_TERMS + 1 + DCH
SMEM_MAX, SMEM_STAGE_BCM, SMEM_STAGE_LU = 227 * 1024, 113 * 1024, 200 * 1024
BCM_REG_SHAPES = ((4, (2, 4)), (6, (3, 6)), (7, (4, 7)), (8, (4, 8)))     # (16-row blocks <=, (RBR, RBC))
MAX_HYPERS = 72


def bcm_nll_smem_bytes(n):
    return 8 * (n * (n + 1) + 3 * n + 8 + EX_SUMS)


def bcm_nll_reg_smem_bytes(rbr, rbc, d):
    nr, npad = 32 * rbr, 16 * rbc
    return 8 * (5 * nr + 16 + EX_SUMS + nr * (d | 1) + nr * npad)


def laplace_smem_bytes(n):
    return 8 * (2 * n * (n + 1) + 12 * n + 8 + EX_SUMS)


def bcm_variant(n_max, n_terms, d, force_smem=False):
    """'reg<RBR,RBC>', 'smem-staged', 'smem-global' or 'lu': the kernel sgp_bcm_nll runs for an SPD objective.
    force_smem: SGP_BCM_IMPL=smem (read once per process)."""
    if bcm_nll_smem_bytes(n_max) > SMEM_MAX:
        return "lu"
    if n_terms == 1 and n_max <= 128 and not force_smem:
        rb = (n_max + 15) // 16
        rbr, rbc = next(shape for lim, shape in BCM_REG_SHAPES if rb <= lim)
        if bcm_nll_reg_smem_bytes(rbr, rbc, d) <= SMEM_MAX:
            return "reg<%d,%d>" % (rbr, rbc)
    staged = bcm_nll_smem_bytes(n_max) + 8 * n_max * (d | 1) <= SMEM_STAGE_BCM
    return "smem-staged" if staged else "smem-global"


def laplace_variant(n_max, d):
    """None when sgp_laplace_nll refuses the expert size, else 'staged' / 'global'."""
    if laplace_smem_bytes(n_max) > SMEM_MAX:
        return None
    return "staged" if laplace_smem_bytes(n_max) + 8 * n_max * (d | 1) <= SMEM_MAX else "global"


def test_objective_dispatch_thresholds():
    # register kernel: one term, shape by n_max; the largest shape falls back above d = 93 (RBF: 2 hyper-parameters)
    assert [bcm_variant(n, 1, 4) for n in (1, 64, 65, 96, 97, 112, 113, 128)] == [
        "reg<2,4>", "reg<2,4>", "reg<3,6>", "reg<3,6>", "reg<4,7>", "reg<4,7>", "reg<4,8>", "reg<4,8>"]
    assert bcm_variant(128, 1, 93) == "reg<4,8>" and bcm_variant(128, 1, 94) == "smem-global"
    assert bcm_variant(128, 1, 100) == "smem-global"
    assert bcm_variant(128, 1, 64) == "reg<4,8>"             # 64 ARD betas + scale + noise = 66 hyper-parameters
    # shared-memory kernel: 129..168 points or >= 2 terms; staging limit 113 KB (n_max 110 / 111 at d = 16; never
    # above 117 points)
    assert bcm_variant(129, 1, 4) == "smem-global" and bcm_variant(168, 1, 4) == "smem-global"
    assert max(n for n in range(1, 200) if bcm_variant(n, 2, 1) == "smem-staged") == 117
    assert bcm_variant(104, 2, 4) == "smem-staged" and bcm_variant(100, 1, 4, force_smem=True) == "smem-staged"
    assert bcm_variant(110, 2, 16) == "smem-staged" and bcm_variant(111, 2, 16) == "smem-global"
    assert bcm_variant(168, 2, 1) == "smem-global"
    # LU path from 169 points on, whatever the kernel
    assert bcm_variant(168, 4, 20) != "lu" and bcm_variant(169, 1, 1) == "lu" and bcm_variant(406, 2, 5) == "lu"
    assert max(n for n in range(1, 400) if bcm_nll_smem_bytes(n) <= SMEM_MAX) == 168
    # Laplace: largest expert 117, rows not staged there; the error message's "~115" is the staged size at small d
    assert max(n for n in range(1, 400) if laplace_variant(n, 1) is not None) == 117
    assert laplace_variant(118, 1) is None and laplace_variant(117, 1) == "global"
    assert laplace_variant(100, 20) == "staged" and laplace_variant(115, 1) == "staged"
    # hyper-parameter limit: 71 ARD betas + scale fit, 72 + scale do not; d = 71 fits every register shape
    assert 1 + 71 == MAX_HYPERS and bcm_variant(64, 1, 71) == "reg<2,4>"


def test_objective_mirror_constants_match_source():
    """The limits and shapes the objective-dispatch mirrors above transcribe, read from the sources."""
    import os
    import re
    csrc = os.path.join(os.path.dirname(os.path.abspath(__file__)), "..", "spark_gp_b200", "csrc")
    read = lambda f: open(os.path.join(csrc, f)).read()
    bcm, internal = read("bcm_nll.cu"), read("sgp_internal.h")
    kib = lambda src, name: int(re.search(r"constexpr size_t %s = (\d+) \* 1024;" % name, src).group(1)) * 1024
    assert kib(internal, "kSmemOptInMax") == SMEM_MAX
    assert kib(bcm, "kStageTwoCtas") == SMEM_STAGE_BCM
    assert kib(bcm, "kStageGeneral") == SMEM_STAGE_LU
    assert int(re.search(r"constexpr int kMaxHypers = (\d+);", internal).group(1)) == MAX_HYPERS
    table = re.search(r"const RegShape kRegShapes\[\] = \{(.*?)\};", bcm, re.S).group(1)
    shapes = re.findall(r"\{(\d+), (\d+), (\d+), bcm_nll_reg_kernel<(\d+), (\d+)>\}", table)
    assert [(int(b), (int(r), int(c))) for b, r, c, _, _ in shapes] == list(BCM_REG_SHAPES)
    assert all((r, c) == (tr, tc) for _, r, c, tr, tc in shapes)       # each row names the template it launches
    assert 16 * BCM_REG_SHAPES[-1][0] == 128                            # the register kernel's largest expert


# ---- per-component error bound of the objective gradient (test_gpu_objectives.py asserts it on the GPU) --------------
# g_i = -1/2 sum_ab dK_i[a,b] W_ab,  W = alpha alpha' - K^-1.  Rounding of the pair sums (direct form, n terms per
# partial sum) and of K^-1 (condition number kappa) give, per expert,
#   |dg_i| <= C_BOUND eps (n + kappa) * 1/2 sum_ab |dK_i[a,b]| (|alpha_a alpha_b| + |K^-1_ab|)
# summed over experts.  For an ARD beta_k, dK_i = -2 beta_k scale (x_ak - x_bk)^2 k_ab.  The expanded form
# 2 (sum_a x_ak^2 m_a - x_k' M x_k) has a rounding error of ~n eps 2|beta_k| scale sum_ab |x_ak| |M_ab| |x_bk| instead,
# which exceeds this bound as soon as |x_k| is large against the distances that carry the kernel values.
EPS = float(np.finfo(np.float64).eps)
C_BOUND = 4.0


def gradient_atol(K, dK, y):
    """Absolute error bound of every gradient component of one expert (see above)."""
    Kinv = np.linalg.inv(K)
    alpha = Kinv @ y
    absW = np.abs(np.outer(alpha, alpha)) + np.abs(Kinv)
    scale = C_BOUND * EPS * (len(y) + np.linalg.cond(K))
    return np.array([scale * 0.5 * float((np.abs(d) * absW).sum()) for d in dK])


def _layout(name, n, d, rng):
    """'standardised': N(0,1) features, beta in [0.3, 3] / sqrt(d) (what L-BFGS visits); 'clustered': unit-scale
    structure inside clusters 300 apart, beta = 1 -- coordinates large against the distances inside a cluster."""
    if name == "standardised":
        return rng.standard_normal((n, d)), rng.uniform(0.3, 3.0, d) / np.sqrt(d)
    X = rng.random((n, d)) + 300.0 * rng.integers(0, 4, (n, 1))
    return X, np.ones(d)


@pytest.mark.parametrize("layout", ["standardised", "clustered"])
def test_gradient_error_bound_vs_extended_precision(layout):
    """The per-component bound holds for the direct pair-sum gradient in fp64 against an extended-precision reference
    (long double kernel, inverse refined by one Newton step in long double); the expanded quadratic form breaks it on
    the clustered layout."""
    rng = np.random.default_rng(7)
    n, d, scale, noise = 100, 4, 1.3, 1e-2
    X, beta = _layout(layout, n, d, rng)
    y = rng.standard_normal(n)
    diff = X[:, None, :] - X[None, :, :]
    k = np.exp(-((diff * beta) ** 2).sum(2))
    K = scale * k + noise * np.eye(n)
    dK = [k] + [scale * (-2.0 * beta[j]) * diff[:, :, j] ** 2 * k for j in range(d)]
    atol = gradient_atol(K, dK, y)
    Kinv = np.linalg.inv(K)
    W = np.outer(Kinv @ y, Kinv @ y) - Kinv
    g = np.array([-0.5 * float((dk * W).sum()) for dk in dK])
    # reference: everything in long double
    L = np.longdouble
    Xl, bl = X.astype(L), beta.astype(L)
    dl = Xl[:, None, :] - Xl[None, :, :]
    kl = np.exp(-((dl * bl) ** 2).sum(2))
    Kl = L(scale) * kl + L(noise) * np.eye(n, dtype=L)
    Xi = Kinv.astype(L)
    Xi = Xi + Xi @ (np.eye(n, dtype=L) - Kl @ Xi)
    al = Xi @ y.astype(L)
    Wl = np.outer(al, al) - Xi
    dKl = [kl] + [L(scale) * (L(-2.0) * bl[j]) * dl[:, :, j] ** 2 * kl for j in range(d)]
    g_ref = np.array([float(L(-0.5) * (dk * Wl).sum()) for dk in dKl])
    err = np.abs(g - g_ref)
    assert np.all(err <= atol), (err / atol).max()
    # the expanded form of the ARD sums (rows translated by the first row, as the register kernel's build does)
    M = k * W
    Xt = X - X[0]
    g_exp = np.array([-0.5 * scale * (-2.0 * beta[j]) * 2.0 * ((Xt[:, j] ** 2) @ M.sum(1) - Xt[:, j] @ M @ Xt[:, j])
                      for j in range(d)])
    ratio = np.abs(g_exp - g_ref[1:]) / atol[1:]
    print("%s: direct form max err/bound %.1e, expanded form %.1e" % (layout, (err / atol).max(), ratio.max()))
    if layout == "clustered":
        assert ratio.max() > 10.0


def test_bcm_register_kernel_identities():
    """Two identities of `bcm_nll_reg_kernel` (csrc/bcm_nll.cu), in NumPy: (1) n sweeps of Goodnight's sweep operator
    turn an SPD matrix into minus its inverse, the pivots are the Schur complements (all positive) and their logs sum to
    log|det|; (2) the per-dimension gradient sums equal the quadratic forms
    sum_ab (x_ak - x_bk)^2 M_ab = 2 (sum_a x_ak^2 m_a - x_k' M x_k) with m = M 1, for any symmetric M -- in exact
    arithmetic; the kernel sums the pair differences, because the expanded form cancels (test_gradient_error_bound_...)."""
    rng = np.random.default_rng(4)
    n, d = 37, 5
    X = rng.standard_normal((n, d))
    K = np.exp(-0.5 * ((X[:, None, :] - X[None, :, :]) ** 2).sum(-1)) + 0.1 * np.eye(n)
    A = K.copy()
    logdet = 0.0
    for k in range(n):
        piv = A[k, k]
        assert piv > 0
        logdet += np.log(piv)
        col = A[:, k].copy()
        A -= np.outer(col, col) / piv                      # rank-1 update everywhere ...
        A[:, k] = col / piv; A[k, :] = col / piv            # ... then the pivot column / row
        A[k, k] = -1.0 / piv
    assert np.allclose(-A, np.linalg.inv(K), rtol=1e-9, atol=1e-10)
    assert abs(logdet - np.linalg.slogdet(K)[1]) < 1e-9
    W = rng.standard_normal((n, n)); M = K * (W + W.T)      # any symmetric pair weight
    m1 = M.sum(1)
    for k in range(d):
        direct = (((X[:, None, k] - X[None, :, k]) ** 2) * M).sum()
        assert abs(direct - 2.0 * ((X[:, k] ** 2) @ m1 - X[:, k] @ M @ X[:, k])) < 1e-9 * max(1.0, abs(direct))


# ---- launch geometry of the int8 Gram (tests/test_gpu_entry_points.py picks its shapes with these mirrors) -----------
# i8_slices transcribes csrc/gram_i8_wgmma.cu: a launch over n_units 64-point units runs nt(nt+1) CTAs per point slice
# (two half tiles per tile of the upper block triangle) and takes the slice count <= 16 that minimises waves x units per
# slice.  host_chunks transcribes the chunk plan of sgp_stats_accumulate (csrc/api.cu): ~16 MB of X per chunk, at least
# 65536 points, equal chunks in multiples of 64 points, and a first chunk of a quarter of the others.  The device entry
# (sgp_stats_accumulate_device) makes one launch over the whole shard.  Inside a slice, the kernel folds its int32
# accumulators into the fp64 partial tile every FLUSH_UNITS units: the first fold stores, later folds add.
UNIT_POINTS, FLUSH_UNITS, SLICES_MAX, TILE = 64, 400, 16, 128
H100_SXM_SMS = 132


def i8_slices(m_pad, num_sms, n_units):
    nt = m_pad // TILE
    ctas = nt * (nt + 1)
    best, best_cost = 1, None
    for s in range(1, min(SLICES_MAX, n_units) + 1):
        cost = -(-ctas * s // num_sms) * -(-n_units // s)
        if best_cost is None or cost < best_cost:
            best, best_cost = s, cost
    return best


def host_chunks(n, d, x_is_f32):
    """Point counts of the launches sgp_stats_accumulate makes for one call of n points."""
    row = d * (4 if x_is_f32 else 8)
    chunk = max((16 << 20) // row, 65536)
    nchunks = -(-n // chunk)
    chunk = min((-(-n // nchunks) + 63) // 64 * 64, n)
    first = chunk
    if n > chunk:
        first = min(max((chunk // 4 + 63) // 64 * 64, 65536), chunk)
        rest = n - first
        nchunks = -(-rest // chunk)
        chunk = max((-(-rest // nchunks) + 63) // 64 * 64, first)
    sizes, p0, step = [], 0, first
    while p0 < n:
        sizes.append(min(step, n - p0))
        p0 += step
        step = chunk
    return sizes


def units_per_slice(n, m, d, x_is_f32=True, device=False, num_sms=H100_SXM_SMS):
    """Units the first (fullest) point slice of every int8 launch of one accumulate call runs through."""
    m_pad = -(-m // TILE) * TILE
    out = []
    for cn in ([n] if device else host_chunks(n, d, x_is_f32)):
        nu = -(-cn // UNIT_POINTS)
        out.append(-(-nu // i8_slices(m_pad, num_sms, nu)))
    return out


def points_for_units(m, target, num_sms, jag=0):
    """A device-entry point count n whose fullest slice runs exactly `target` units (n = units * 64 - jag)."""
    m_pad = -(-m // TILE) * TILE
    for nu in range(target, SLICES_MAX * target + 1):
        s = i8_slices(m_pad, num_sms, nu)
        if -(-nu // s) == target:
            return nu * UNIT_POINTS - jag
    raise ValueError("no point count gives %d units per slice" % target)


# (n, m, d, fp32, device entry) -> units per slice of the fullest launch, on 132 SMs
UNITS_TABLE = [
    ((1_000_000, 1000, 16, True, False), 332),   # test_full_size_config2_properties (AUTO, host entry)
    ((1_600_000, 128, 8, True, False), 367),     # test_auto_budget_checked_over_whole_window
    ((300_000, 1000, 16, True, False), 167),     # test_i8_headline_path_vs_oracle
    ((300_000, 512, 16, True, False), 141),      # __graft_entry__.smoke
    ((20480, 2000, 32, True, False), 20),        # test_i8_config_shapes_vs_oracle
    ((8192, 4000, 8, True, False), 128),
    ((120_000, 500, 8, True, False), 145),       # test_auto_routes_multi_term_kernels_to_direct_mode
    ((1_000_000, 1000, 16, True, True), 1421),   # bench.py configs1, device entry: three folds that add
    ((1_250_000, 2000, 32, True, True), 1221),   # bench.py configs3, device entry
    ((399 * 64, 1300, 16, True, True), 399),     # fold boundaries: m_pad = 1408 is one slice on 132 SMs
    ((400 * 64 - 17, 1300, 16, True, True), 400),
    ((401 * 64, 1300, 16, True, True), 401),
    ((800 * 64, 1300, 16, True, True), 800),
    ((801 * 64 - 5, 1300, 16, True, True), 801),
    ((1201 * 64, 1300, 16, True, True), 1201),
    ((1_300_000, 1300, 2, True, False), 20313),  # d <= 2: one 1.3M-point chunk through the host entry
    ((6400 * 64, 4, 4, True, True), 400),        # one tile, 16 slices
    ((16 * 1201 * 64, 4, 4, True, True), 1201),
]


@pytest.mark.parametrize("args,want", UNITS_TABLE)
def test_int8_units_per_slice_table(args, want):
    assert max(units_per_slice(*args)) == want


def test_int8_launch_geometry_rules():
    # every int8 test that compares values before tests/test_gpu_entry_points.py stayed below the first fold that adds
    assert max(want for (n, m, d, f32, dev), want in UNITS_TABLE[:7]) < FLUSH_UNITS
    # m_pad in (1280, 1408]: 11 tiles, 132 CTAs per slice -- one slice on an H100 SXM, so units per slice = ceil(n / 64)
    for m in (1281, 1300, 1408):
        assert all(i8_slices(-(-m // TILE) * TILE, H100_SXM_SMS, nu) == 1 for nu in (1, 399, 400, 401, 5000))
    # ... but not on a 114-SM part: the shape picker reads the SM count instead of assuming it
    assert i8_slices(1408, 114, 4000) != 1
    for sms in (114, 132):
        for target in (399, 400, 401, 800, 801, 1201):
            n = points_for_units(1300, target, sms)
            assert units_per_slice(n, 1300, 16, device=True, num_sms=sms) == [target]
    # host chunk plan: covers the call, multiples of 64 except the last, first chunk the smallest
    for n, d, f32 in ((1_000_000, 16, True), (1_250_000, 32, True), (70001, 3, False), (65536, 8, True), (65537, 8, True),
                      (10_000_000, 4, False), (1_300_000, 2, True)):
        sizes = host_chunks(n, d, f32)
        assert sum(sizes) == n and all(s % 64 == 0 for s in sizes[:-1]) and sizes[0] == min(sizes[:-1] or sizes)


def test_int8_mirror_constants_match_source():
    """The constants the mirrors and the fixed-point emulation below transcribe, read from the kernel source."""
    import os
    import re
    src = open(os.path.join(os.path.dirname(os.path.abspath(__file__)), "..", "spark_gp_b200", "csrc",
                            "gram_i8_wgmma.cu")).read()
    assert re.search(r"constexpr int FLUSH_UNITS = (\d+);", src).group(1) == str(FLUSH_UNITS)
    assert re.search(r"constexpr int UP = (\d+);", src).group(1) == str(UNIT_POINTS)
    assert re.search(r"for \(int s = 1; s <= (\d+) && s <= n_units; \+\+s\)", src).group(1) == str(SLICES_MAX)
    assert float(re.search(r"constexpr float C0 = ([0-9.]+)f;", src).group(1)) == float(FIXED_C0)
    m = re.search(r"constexpr float MAGIC = ([0-9.]+)f \+ ([0-9.]+)f;", src)
    assert float(m.group(1)) + float(m.group(2)) == float(FIXED_MAGIC)


# ---- the fixed-point encoding of the int8 Gram (fixed_word in csrc/gram_i8_wgmma.cu), emulated exactly ----------------
# fixed_word(kappa) = bits(fmaf(kappa, C0, MAGIC)) << 1.  kappa * C0 is exact in fp64 (24 + 23 bits); below 2^24 the fp32
# result has ulp 1, so fmaf = MAGIC + rint(kappa * C0) (round half to even, like the FMA's single rounding); from 2^24 on
# the ulp is 2.  The bytes of the word are (2 s0 + 128, s1 + 128, s2); the planes are P0 = 2 s0, P1 = s1 (both signed)
# and P2 = s2 (unsigned), the base-256 digits of 2u with u = s2 2^15 + s1 2^7 + s0.
FIXED_C0 = np.float32(8355000.0)
FIXED_MAGIC = np.float32(8388608.0 + 16448.0)


def fixed_word(kappa):
    p = np.asarray(kappa, dtype=np.float32).astype(np.float64) * np.float64(FIXED_C0)
    below = np.float64(FIXED_MAGIC) + np.rint(p)
    above = 2.0 * np.rint((np.float64(FIXED_MAGIC) + p) / 2.0)
    f = np.where(below < 2.0 ** 24, below, above).astype(np.float32)
    return (f.view(np.uint32).astype(np.uint64) << np.uint64(1)) & np.uint64(0xFFFFFFFF)


def digit_planes(word):
    b = [((word >> np.uint64(8 * i)) & np.uint64(0xFF)).astype(np.int64) for i in range(3)]
    return b[0] - 128, b[1] - 128, b[2]                       # P0 (x ^ 0x80 as int8), P1, P2


def test_fixed_point_digits_exact_in_range():
    kappa = np.unique(np.concatenate([np.linspace(0.0, 1.0 + 2e-3, 2_000_001, dtype=np.float32),
                                      np.float32(1.0) + np.arange(-4096, 4097, dtype=np.float32) * np.float32(2 ** -23),
                                      np.float32(2.0) ** -np.arange(0, 150, dtype=np.float32)]))
    kappa = kappa[kappa <= np.float32(1.0 + 2e-3)]
    P0, P1, P2 = digit_planes(fixed_word(kappa))
    u = np.rint(kappa.astype(np.float64) * np.float64(FIXED_C0)).astype(np.int64)
    assert np.array_equal(P2 * 2 ** 16 + P1 * 2 ** 8 + P0, 2 * u)           # u comes back exactly from the planes
    assert np.all(P0 % 2 == 0)
    assert P0.min() >= -128 and P0.max() <= 126                             # s0 in [-64, 63]
    assert P1.min() >= -128 and P1.max() <= 127                             # s1 in [-128, 127]
    assert P2.min() >= 0 and P2.max() <= 255                                # s2 in [0, 255]: the unsigned operand
    assert P2.max() == 255 and P1.min() == -128 and P0.max() == 126          # the ranges are used to their ends


def test_fixed_point_accumulator_bounds():
    """Per-point products of the three int32 accumulators, and the fold interval that keeps them exact."""
    per_fold = FLUSH_UNITS * UNIT_POINTS                                    # 25600 points between folds
    # box bounds over the digit ranges: P2'P2, P2'P1 + P1'P2, P2'P0 + P0'P2 + P1'P1
    b4, b3, b2 = 255 * 255, 2 * 255 * 128, 2 * 255 * 128 + 128 * 128
    assert (b4, b3, b2) == (65025, 65280, 81664)
    assert max(b4, b3, b2) * per_fold < 2 ** 31 - 1                         # 2.09e9: a 2.6 % margin
    assert b2 * (per_fold + UNIT_POINTS) < 2 ** 31 - 1 < b2 * 2 * per_fold    # one more unit fits, a doubled interval not
    # the digit patterns that reach the bounds on a diagonal element (the same kappa on both sides)
    u_worst = 255 * 2 ** 15 - 128 * 2 ** 7 + 63                             # s2 = 255, s1 = -128, s0 = 63
    for u, want in ((u_worst, (65025, -65280, 80644)), (int(FIXED_C0), None)):
        kappa = np.float32(u / float(FIXED_C0))
        P0, P1, P2 = (int(v) for v in digit_planes(fixed_word(kappa)))
        assert P2 * 2 ** 16 + P1 * 2 ** 8 + P0 == 2 * u
        acc = (P2 * P2, 2 * P2 * P1, 2 * P2 * P0 + P1 * P1)
        assert all(abs(a) * per_fold < 2 ** 31 for a in acc)
        if want:
            assert acc == want


def test_fixed_point_breaks_just_above_margin():
    """u + 0x4040 must stay below 2^23: the encoding holds up to kappa = 8372160 / C0 = 1 + 2.05e-3 and breaks above --
    an element there reads back as a different, much smaller value.  The GPU tests check that the kernel's kappa stays
    below 1 + 2e-3 at every norm the operand gate admits (test_gpu_entry_points.py::test_kappa_margin_...)."""
    kappa = np.float32(1.0) + np.arange(0, 40000, dtype=np.float32) * np.float32(2 ** -23)
    P0, P1, P2 = digit_planes(fixed_word(kappa))
    u = np.rint(kappa.astype(np.float64) * np.float64(FIXED_C0)).astype(np.int64)
    ok = P2 * 2 ** 16 + P1 * 2 ** 8 + P0 == 2 * u
    first_bad = kappa[np.argmin(ok)]
    assert np.all(ok[kappa < first_bad]) and not np.any(ok[kappa >= first_bad])
    assert 1.0 + 2e-3 < first_bad <= 1.0 + 2.06e-3
    assert abs(float(first_bad) - 8372160.0 / float(FIXED_C0)) < 2 ** -22
    back = (P2 * 2 ** 16 + P1 * 2 ** 8 + P0) / 2.0 / float(FIXED_C0)
    assert np.all(back[~ok] < 0.5)                                          # silently O(1) wrong


# ---- the fp64 DMMA statistics kernel (kmn_gram_f64_kernel, csrc/gram_f64.cu) and the int8 direct-mode gate ----------
# launch_stats_f64 (csrc/api.cu) runs one of four loop variants of the kernel and splits the points into slices:
#   SGP_PREC_F64 (and AUTO's fp64 path): fp32 elements on a 128 x 64 staircase of tiles (two CTAs per SM), the
#     pipelined loop for one non-Eye term with dpad <= DC, else the generic loop (z reloaded per term and per DC-dim
#     chunk, the terms summed into the panel);
#   SGP_PREC_F64_STRICT: fp64 elements on the 128 x 128 triangle, z resident for one term with dpad <= DC, else chunked.
# Slices: num_sms // (tiles of the 128 x 128 triangle), at least 1 and at most one per 16-point block; every slice
# takes ceil(blocks / slices) blocks, so the last slices can be empty.  tests/test_gpu_gram_variants.py builds its
# cases from these mirrors.  sgp_stats_begin admits the int8 direct-distance mode for n_terms * dpad <= 72.
F64_PB, F64_DC, DIRECT_WIDTH = 16, 32, 72


def dpad4(d):
    return (d + 3) // 4 * 4


def f64_variant(precision, n_terms, d):
    """'pipelined' / 'generic' (fp32 elements) or 'resident' / 'chunked' (SGP_PREC_F64_STRICT) for n_terms non-Eye terms."""
    one = n_terms == 1 and dpad4(d) <= F64_DC
    if precision == N.SGP_PREC_F64_STRICT:
        return "resident" if one else "chunked"
    return "pipelined" if one else "generic"


def f64_slices(m, n, num_sms):
    """16-point blocks of every point slice of one fp64-kernel launch over n points (len = the slice count)."""
    nt1 = -(-m // TILE)
    blocks = -(-n // F64_PB)
    slices = min(max(num_sms // (nt1 * (nt1 + 1) // 2), 1), blocks)
    bps = -(-blocks // slices)
    return [max(0, min(bps * (s + 1), blocks) - bps * s) for s in range(slices)]


def direct_ok(n_terms, d):
    return 1 <= n_terms and n_terms * dpad4(d) <= DIRECT_WIDTH


def test_f64_mirror_constants_match_source():
    """The constants and rules the fp64-kernel mirrors transcribe, read from the sources."""
    import os
    import re
    csrc = os.path.join(os.path.dirname(os.path.abspath(__file__)), "..", "spark_gp_b200", "csrc")
    read = lambda f: open(os.path.join(csrc, f)).read()
    gram, api, internal = read("gram_f64.cu"), read("api.cu"), read("sgp_internal.h")
    assert re.search(r"constexpr int PB = (\d+);", gram).group(1) == str(F64_PB)
    assert re.search(r"constexpr int DC = (\d+);", gram).group(1) == str(F64_DC)
    assert re.search(r"constexpr int kTile = (\d+);", internal).group(1) == str(TILE)
    assert re.search(r"i8_direct_ok = kf\.n_terms >= 1 && kf\.n_terms \* dpad <= (\d+);", api).group(1) == str(DIRECT_WIDTH)
    assert "const bool z_resident = (p.n_terms == 1 && p.dpad <= DC);" in gram
    assert "int n_slices = c->num_sms / ntiles;" in api and "const int ntiles = nt1 * (nt1 + 1) / 2;" in api
    assert "const long long bps = (total_blocks + p.n_slices - 1) / p.n_slices;" in gram
    assert "const int dpad = (d + 3) & ~3;" in api


def test_f64_dispatch_and_slices():
    assert [f64_variant(N.SGP_PREC_F64, 1, d) for d in (1, 32, 33)] == ["pipelined", "pipelined", "generic"]
    assert [f64_variant(N.SGP_PREC_F64, t, 4) for t in (1, 2, 4)] == ["pipelined", "generic", "generic"]
    assert [f64_variant(N.SGP_PREC_F64_STRICT, t, d) for t, d in ((1, 29), (1, 31), (1, 33), (2, 1))] == [
        "resident", "resident", "chunked", "chunked"]
    assert [direct_ok(t, d) for t, d in ((1, 72), (1, 69), (1, 73), (2, 36), (2, 33), (2, 37), (3, 24), (3, 21),
                                         (3, 25), (4, 16), (4, 13), (4, 17), (0, 4))] == [
        True, True, False, True, True, False, True, True, False, True, True, False, False]
    for sms in (114, 132):
        # m <= 128: one tile, one slice per SM
        assert f64_slices(128, 16 * sms - 1, sms) == [1] * sms
        assert f64_slices(1, 16 * sms + 1, sms) == [2] * (sms // 2) + [1] + [0] * (sms - sms // 2 - 1)
        s = f64_slices(64, 16 * (sms + 1), sms)
        assert len(s) == sms and sum(s) == sms + 1 and s.count(0) == sms - (sms + 1 + 1) // 2   # trailing slices empty
        assert f64_slices(65, 15, sms) == [1] and f64_slices(128, 33, sms) == [1, 1, 1]
        # m >= 2049 (on these SM counts): more tiles than SMs, one slice
        assert -(-2049 // TILE) * (-(-2049 // TILE) + 1) // 2 > sms and f64_slices(2049, 10 ** 6, sms) == [62500]
    for m, n, sms in ((1000, 77777, 132), (129, 5, 132), (257, 16 * 44 + 3, 132), (4000, 1, 114)):
        s = f64_slices(m, n, sms)
        assert sum(s) == -(-n // F64_PB) and s == sorted(s, reverse=True)


# The CTA's tile decode (kmn_gram_f64_kernel): blockIdx.x -> (ti, tj) from an fp32 sqrtf estimate corrected by two
# while loops; TN = 128 covers the lower block triangle tj <= ti, TN = 64 the staircase tj <= 2 ti + 1 of 64-column tiles.
def tile_decode(t, tn):
    f = np.float32
    if tn == 128:
        ti = int((np.sqrt(f(8.0) * f(t) + f(1.0)) - f(1.0)) * f(0.5))
        est = ti
        while (ti + 1) * (ti + 2) // 2 <= t:
            ti += 1
        while ti * (ti + 1) // 2 > t:
            ti -= 1
        return ti, t - ti * (ti + 1) // 2, ti - est
    ti = int((np.sqrt(f(4.0) * f(t) + f(1.0)) - f(1.0)) * f(0.5))
    est = ti
    while (ti + 1) * (ti + 2) <= t:
        ti += 1
    while ti * (ti + 1) > t:
        ti -= 1
    return ti, t - ti * (ti + 1), ti - est


@pytest.mark.parametrize("tn", [128, 64])
def test_f64_tile_decode_covers_every_tile_once(tn):
    fixes = 0
    for nt1 in range(1, 65):
        count = nt1 * (nt1 + 1) // 2 if tn == 128 else nt1 * (nt1 + 1)
        tiles = [tile_decode(t, tn) for t in range(count)]
        want = {(i, j) for i in range(nt1) for j in range(i + 1 if tn == 128 else 2 * i + 2)}
        got = [(i, j) for i, j, _ in tiles]
        assert len(set(got)) == len(got) == count and set(got) == want
        fixes = max(fixes, max(abs(c) for _, _, c in tiles))
    assert fixes <= 1                       # the fp32 estimate is off by at most one row tile up to 64 row tiles
    if tn == 64:
        # diagonal block: tiles 2 ti (b_I, joff 0) and 2 ti + 1 (joff 64) read the J columns from the I panel; at
        # m = 64 / 192 the second one lies wholly past m, at m = 65 / 193 partly
        for m in (64, 65, 192, 193):
            ti = (m - 1) // TILE
            lo = (2 * ti + 1) * 64
            assert (lo >= m) == (m % TILE == 64)


# ---- why the fp64 kernel centres its operands ------------------------------------------------------------------------
# The fp32-element variants stage x~ = (x - c) beta sqrt(log2 e) and z~ = (Z beta - c beta) sqrt(log2 e), each rounded
# to fp32, then form d = x~ - z~ and q = sum d^2 in fp32 and K = 2^-q.  Without the centre c, the staged coordinates
# carry a rounding of 2^-24 |x| beta -- the distance from the origin in length scales -- into every element; centred,
# the rounding follows the spread of the data.  f64_centre transcribes the centre of stats_scales (csrc/api.cu): the
# active-set mean rounded to a whole multiple of the active set's standard deviation, 0 for data centred already.
def f64_centre(Z):
    mean = Z.sum(0) / len(Z)
    sd = np.sqrt(((Z - mean) ** 2).sum(0) / len(Z))
    return np.where(sd > 0, np.rint(mean / np.where(sd > 0, sd, 1.0)) * sd, mean)


def test_f64_centre_rule():
    rng = np.random.default_rng(5)
    Z = rng.standard_normal((300, 6)) * [1.0, 2.0, 0.1, 5.0, 1.0, 1.0] + [0.1, -0.5, 0.0, 2.0, 1e3, -1e3]
    Z[:, 5] = -1e3                                              # constant column: the mean itself
    c, mean = f64_centre(Z), Z.mean(0)
    sd = Z.std(0)
    assert np.all(np.abs(c - mean) <= 0.5 * sd + 1e-9 * np.abs(mean))
    assert np.all(c[:3] == 0.0) and c[5] == -1e3                # standardised columns keep the uncentred arithmetic
    assert abs(c[4] - 1e3) <= 0.5                               # an offset of 1e3 is removed to within half a deviation
def f32_elements(X, Z, beta, centre):
    P = np.sqrt(np.log2(np.e))
    xs = ((X - centre) * beta * P).astype(np.float32)
    zs = (-(P * (Z * beta - centre * beta))).astype(np.float32)
    q = np.zeros((len(X), len(Z)), dtype=np.float32)
    for k in range(X.shape[1]):
        dk = xs[:, None, k] + zs[None, :, k]
        q += dk * dk
    return np.exp2(-q.astype(np.float64))


def test_f64_kernel_centring_emulated():
    rng = np.random.default_rng(3)
    n, d, m = 6000, 5, 200
    beta = np.ones(d)
    errs = {}
    for off in (0.0, 100.0, 1000.0):
        X = rng.random((n, d)) * 3 + off
        Z = X[:m]
        diff = X[:, None, :] - Z[None, :, :]
        K0 = np.exp(-((diff * beta) ** 2).sum(-1))
        G0 = K0.T @ K0
        for name, c in (("uncentred", np.zeros(d)), ("centred", f64_centre(Z))):
            K = f32_elements(X, Z, beta, c)
            errs[(off, name)] = float(np.abs(K.T @ K - G0).max() / np.abs(G0).max())
    print(", ".join("%g %s: dG=%.1e" % (o, nm, e) for (o, nm), e in errs.items()))
    assert all(errs[(off, "centred")] < 1e-7 for off in (0.0, 100.0, 1000.0))
    assert errs[(1000.0, "uncentred")] > 1e-5 and errs[(100.0, "uncentred")] > 1e-6
