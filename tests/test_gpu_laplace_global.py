"""The Laplace objective for experts of any size (run on an H100: `pytest -m gpu`).

`sgp_laplace_nll_any_size` / `sgp_laplace_nll_classes_any_size` run `laplace_kernel` while the largest expert fits on
chip (117 points) and `laplace_global_kernel` (csrc/laplace_global.cu: matrices in global memory, persistent grid,
blocked Cholesky on fp64 tensor cores) above.  Gates are those of the on-chip Laplace tests (test_gpu_objectives.py,
written there once): value relative TOL_NLL = 1e-9; gradient per component RTOL_LAP |g0| + laplace_atol (ATOL_LAP
sum_ab |dK|); latent modes 1e-9 max(1, |f|).  Estimator gates: test_gpu_one_vs_rest.py's TOL_PRED = 1e-5 on raw
predictions.  Bit identity is asserted wherever two paths run the same arithmetic.
"""
import os

import numpy as np
import pytest

import oracle
import spark_gp_b200 as sg
from oracle.classification import classification_likelihood_and_gradient
from oracle.one_vs_rest import one_vs_rest_fixed_theta
from oracle.ppa import projected_process
from spark_gp_b200 import _native as N
from spark_gp_b200.hyperopt import group_for_experts, pack_experts
from spark_gp_b200.regression import ExplicitActiveSetProvider
from test_gpu_objectives import RTOL_LAP, TOL_NLL, check_components, kernel_pair, laplace_atol, layout

pytestmark = pytest.mark.gpu

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
TOL_PRED = 1e-5


@pytest.fixture(scope="module")
def engs():
    a, b = sg.ProjectedProcessEngine(0), sg.ProjectedProcessEngine(0)
    yield a, b
    a.close()
    b.close()


def bits(a):
    return np.ascontiguousarray(a, dtype=np.float64).view(np.int64)


def labels(X, rng):
    d = X.shape[1]
    return (np.sin(2 * X[:, 0]) + 0.5 * X.sum(1) / np.sqrt(d) + 0.3 * rng.standard_normal(len(X)) > 0).astype(np.float64)


def run_sizes_case(eng, kind, sizes, d, seed=3, tol=1e-6, path=1):
    """Experts of the given sizes, packed back to back; two evaluations (the second warm-starts) against the oracle."""
    rng = np.random.default_rng(seed + 7 * len(sizes) + max(sizes) + d)
    off = np.concatenate([[0], np.cumsum(sizes)]).astype(np.int64)
    X, beta = layout("standardised", int(off[-1]), d, rng)
    y = labels(X, rng)
    k, ofac = kernel_pair(kind, d, beta, rng)
    experts = [(y[a:b], ofac().set_training_vectors(X[a:b])) for a, b in zip(off[:-1], off[1:])]
    fs = [np.zeros(s) for s in sizes]
    eng.experts_upload(X, y, off)
    theta0 = k.getHyperparameters()
    worst = 0.0
    for step, theta in enumerate((theta0, theta0 * rng.uniform(0.7, 1.4, len(theta0)))):
        v0, g0 = 0.0, np.zeros(len(theta))
        for (ye, ke), f in zip(experts, fs):
            v, g = classification_likelihood_and_gradient(ye, f, ke, theta, tol)
            v0 += v; g0 = g0 + g
        v, g = eng.laplace_nll_any_size(k.setHyperparameters(theta), tol)
        assert eng.last_laplace_path() == path
        assert abs(v - v0) <= TOL_NLL * abs(v0), (v, v0)
        worst = max(worst, check_components(g, g0, laplace_atol(experts, theta), RTOL_LAP,
                                            "%s sizes=%s d=%d eval %d" % (kind, sizes[:4], d, step)))
        f_gpu, f_ref = eng.experts_f(int(off[-1])), np.concatenate(fs)
        assert np.abs(f_gpu - f_ref).max() <= 1e-9 * max(1.0, np.abs(f_ref).max())
    print("laplace any-size %-7s n_max=%4d E=%3d d=%3d: grad err/bound=%.2e" % (kind, max(sizes), len(sizes), d, worst))


# ---------------- 1. against the oracle -----------------------------------------------------------------------------
@pytest.mark.parametrize("n_max,E", [(118, 3), (128, 3), (129, 3), (200, 3), (500, 2), (1000, 2), (2000, 1)])
def test_global_sizes_vs_oracle(engs, n_max, E):
    run_sizes_case(engs[0], "ard", [n_max] * E, 3)


def test_global_ragged_experts_vs_oracle(engs):
    """Experts of 1, 63, 64, 65 and 129 points beside a large one: partial tiles and single-point experts."""
    run_sizes_case(engs[0], "ard", [1, 63, 64, 65, 129, 300], 3)


@pytest.mark.parametrize("kind,n_max,d", [("rbf", 200, 1), ("ard2", 150, 20), ("nested", 160, 3), ("rbf", 300, 784)])
def test_global_kernels_and_widths_vs_oracle(engs, kind, n_max, d):
    run_sizes_case(engs[0], kind, [n_max, n_max - 7], d)


def test_global_many_experts_loop_over_the_grid(engs):
    """300 experts: more work items than resident CTAs, so every CTA runs several."""
    run_sizes_case(engs[0], "ard", [120 + (e % 9) for e in range(300)], 2)


# ---------------- 2. the boundary -------------------------------------------------------------------------------------
def test_boundary_117_on_chip_and_118_global(engs):
    eng, ref = engs
    rng = np.random.default_rng(17)
    X = rng.standard_normal((3 * 117, 2)); y = labels(X, rng)
    k = 1.2 * sg.ARDRBFKernel(np.array([0.7, 1.1])) + sg.const(1e-2) * sg.EyeKernel()
    eng.experts_upload(*pack_experts(X, y, 117))
    ref.experts_upload(*pack_experts(X, y, 117))
    for _ in range(2):                                      # the second call warm-starts on both
        v, g = eng.laplace_nll_any_size(k, 1e-6)
        assert eng.last_laplace_path() == 0
        v0, g0 = ref.laplace_nll(k, 1e-6)
        assert bits(v) == bits(v0) and np.array_equal(bits(g), bits(g0))
        assert np.array_equal(bits(eng.experts_f(len(X))), bits(ref.experts_f(len(X))))
    X = rng.standard_normal((3 * 118, 2)); y = labels(X, rng)
    eng.experts_upload(*pack_experts(X, y, 118))
    eng.laplace_nll_any_size(k, 1e-6)
    assert eng.last_laplace_path() == 1
    with pytest.raises(ValueError, match="too large"):    # the on-chip form still refuses
        eng.laplace_nll(k, 1e-6)


# ---------------- 3. determinism --------------------------------------------------------------------------------------
def test_expert_bits_do_not_depend_on_the_launch(engs):
    """One expert's modes are the same bits alone and among 299 others (larger n_max, many CTAs), and two fresh contexts
    return the same bits."""
    eng, _ = engs
    rng = np.random.default_rng(23)
    d = 3
    X = rng.standard_normal((150, d)); y = labels(X, rng)
    k = 1.1 * sg.ARDRBFKernel(np.array([0.6, 0.9, 1.2])) + sg.const(1e-2) * sg.EyeKernel()
    eng.experts_upload(X, y, np.array([0, 150]))
    eng.laplace_nll_any_size(k, 1e-6)
    alone = eng.experts_f(150)
    sizes = [130 + (e % 70) for e in range(300)]
    sizes[137] = 150
    off = np.concatenate([[0], np.cumsum(sizes)]).astype(np.int64)
    Xa = rng.standard_normal((int(off[-1]), d)); ya = labels(Xa, rng)
    Xa[off[137]:off[138]] = X; ya[off[137]:off[138]] = y
    eng.experts_upload(Xa, ya, off)
    v1, g1 = eng.laplace_nll_any_size(k, 1e-6)
    assert eng.last_laplace_path() == 1
    among = eng.experts_f(int(off[-1]))
    assert np.array_equal(bits(among[off[137]:off[138]]), bits(alone))
    f1 = among
    for _ in range(2):
        fresh = sg.ProjectedProcessEngine(0)
        try:
            fresh.experts_upload(Xa, ya, off)
            v2, g2 = fresh.laplace_nll_any_size(k, 1e-6)
            assert bits(v2) == bits(v1) and np.array_equal(bits(g2), bits(g1))
            assert np.array_equal(bits(fresh.experts_f(int(off[-1]))), bits(f1))
        finally:
            fresh.close()


# ---------------- 4. the classes form on the global path --------------------------------------------------------------
def class_data(N, d, C, seed, missing=None):
    rng = np.random.default_rng(seed)
    X = rng.standard_normal((N, d))
    s = np.sin(2 * X[:, 0]) + X[:, -1] + 0.3 * rng.standard_normal(N)
    y = np.digitize(s, np.quantile(s, np.linspace(0, 1, C + 1)[1:-1])).astype(np.float64)
    if missing is not None:
        y[y == missing] = (missing + 1) % C
    return X, y


@pytest.mark.parametrize("C,n_e,E,missing", [(2, 150, 3, None), (3, 200, 2, None), (10, 130, 3, 4)])
def test_classes_global_match_binary_uploads_bitwise(engs, C, n_e, E, missing):
    eng, ref = engs
    d, tol = 3, 1e-6
    N = n_e * E
    X, y = class_data(N, d, C, seed=C * 10 + n_e, missing=missing)
    mk = lambda c, step: (1.2 * (1 + 0.07 * c) * (1 + 0.15 * step)) * sg.ARDRBFKernel(np.linspace(0.6, 1.1, d)) \
        + sg.const(1e-2) * sg.EyeKernel()
    eng.experts_upload(*pack_experts(X, y, n_e))
    calls = [list(range(C)), list(range(C))[::-1], [C - 1, 0] if C > 2 else [1]]
    steps = np.zeros(C, dtype=int)
    got = {c: [] for c in range(C)}
    for call in calls:
        if call is calls[-1]:
            before = {c: eng.experts_f_class(c, N) for c in range(C)}
        vals, grads = eng.laplace_nll_classes_any_size(C, call, [mk(c, steps[c]) for c in call], tol)
        assert eng.last_laplace_path() == 1
        for i, c in enumerate(call):
            got[c].append((vals[i], grads[i], eng.experts_f_class(c, N)))
            steps[c] += 1
    for c in range(C):
        if c not in calls[-1]:
            assert np.array_equal(bits(eng.experts_f_class(c, N)), bits(before[c]))
    for c in range(C):
        ref.experts_upload(*pack_experts(X, (y == c).astype(np.float64), n_e))
        for step, (v, g, f) in enumerate(got[c]):
            v0, g0 = ref.laplace_nll_any_size(mk(c, step), tol)
            assert ref.last_laplace_path() == 1
            assert bits(v) == bits(v0), (c, step)
            assert np.array_equal(bits(g), bits(g0)), (c, step)
            assert np.array_equal(bits(f), bits(ref.experts_f(N))), (c, step)


def test_classes_global_refusals(engs):
    eng, _ = engs
    mk = lambda: sg.RBFKernel(1.3) + sg.const(1e-2) * sg.EyeKernel()
    X, y = class_data(3 * 130, 2, 3, seed=5)
    eng.experts_upload(*pack_experts(X, y, 130))
    with pytest.raises(ValueError, match="too large"):
        eng.laplace_nll_classes(3, [0], [mk()], 1e-6)
    for n_classes, classes in ((3, [3]), (3, [-1]), (3, [0, 0]), (2, [0, 1, 2]), (0, [0])):
        with pytest.raises(ValueError):
            eng.laplace_nll_classes_any_size(n_classes, classes, [mk()] * len(classes), 1e-6)
    eng.laplace_nll_classes_any_size(3, [1], [mk()], 1e-6)
    assert eng.last_laplace_path() == 1
    assert np.all(eng.experts_f_class(0, len(X)) == 0.0)


# ---------------- 5. refusal ------------------------------------------------------------------------------------------
def test_expert_too_large_for_device_memory(engs):
    """One expert of 75 000 points needs 8 ld (2 ld + 44) = 90 GB of workspace: SGP_E_NOMEM before any launch, and the
    context stays usable."""
    eng, _ = engs
    rng = np.random.default_rng(8)
    n = 75000
    X = rng.standard_normal((n, 1)); y = (X[:, 0] > 0).astype(np.float64)
    eng.experts_upload(X, y, np.array([0, n]))
    launches = eng.launch_count()
    with pytest.raises(sg.SgpError, match="error %d" % N.SGP_E_NOMEM):
        eng.laplace_nll_any_size(sg.RBFKernel(1.0) + sg.const(1e-2) * sg.EyeKernel(), 1e-6)
    assert eng.launch_count() == launches
    run_sizes_case(eng, "ard", [200, 200], 2)


# ---------------- 6. estimators ---------------------------------------------------------------------------------------
def test_classifier_mnist68_experts_of_500():
    """GaussianProcessClassifier with datasetSizeForExpert(500) on the mnist68 rows (three experts of 500),
    RBFKernel(10), tol 1e-3, fixed theta, explicit active set: modes and raw predictions against the oracle."""
    c = np.load(os.path.join(GOLD, "mnist68_case.npz"))
    n = int(c["n_rows"])
    X = (c["pixels"].astype(np.float64) - c["mean"]) / c["std"]
    Xtr, Xte, ytr = X[:n], X[n:n + 100], c["y01"][:n]
    sigma, sigma2, tol = float(c["sigma"]), float(c["sigma2"]), 1e-3
    Z = Xtr[c["active_idx"]]
    gp = (sg.GaussianProcessClassifier().setDatasetSizeForExpert(500).setActiveSetSize(500).setSigma2(sigma2)
          .setKernel(lambda: sg.RBFKernel(sigma)).setTol(tol).setActiveSetProvider(ExplicitActiveSetProvider(Z)))
    model = gp.fit(Xtr, ytr, hyperparameters=np.array([sigma]))
    factory = oracle.get_kernel(lambda: oracle.RBFKernel(sigma), sigma2)
    theta = np.array([sigma])
    experts = oracle.get_expert_labels_and_kernels(Xtr, ytr, factory, 500)
    assert len(experts) == 3
    f_all, fk = np.zeros(n), []
    for (ye, ke), idx in zip(experts, group_for_experts(n, 500)):
        f = np.zeros(len(ye))
        classification_likelihood_and_gradient(ye, f, ke, theta, tol)
        f_all[idx] = f
        fk.append((f, ke))
    assert np.abs(gp.last_latent - f_all).max() <= 1e-9 * max(1.0, np.abs(f_all).max())
    pred, _, _ = projected_process(fk, Z, factory, theta)
    want = pred.predict_many(Xte)[0]
    raw = model.predictRaw(Xte)
    assert np.abs(raw[:, 1] - want).max() <= TOL_PRED * max(1.0, np.abs(want).max())


def iris_gp(active=None):
    gp = sg.GaussianProcessClassifier().setDatasetSizeForExpert(150).setActiveSetSize(30)
    return gp.setActiveSetProvider(ExplicitActiveSetProvider(active)) if active is not None else gp


def test_one_vs_rest_iris_single_expert_of_150():
    c = np.load(os.path.join(GOLD, "iris_case.npz"))
    X, y = c["X"], c["y"]
    Xte = X[c["test_idx"]]
    ovr = sg.OneVsRest().setClassifier(iris_gp())
    model = ovr.fit(X, y)
    raw = model.predictRaw(Xte)
    for k in range(3):                                     # optimisation on: each class equals its binary fit
        gp = iris_gp()
        bm = gp.fit(X, (y == k).astype(np.float64))
        assert np.array_equal(bits(model.models[k].hyperparameters), bits(bm.hyperparameters)), k
        assert np.array_equal(bits(ovr.last_latent[k]), bits(gp.last_latent)), k
        assert np.array_equal(bits(raw[:, k]), bits(bm.predictRaw(Xte)[:, 1])), k
    Z = X[c["train_idx"]][c["active_idx"]]
    ovr = sg.OneVsRest().setClassifier(iris_gp(Z))
    model = ovr.fit(X, y, hyperparameters=c["thetas"])
    factory = oracle.get_kernel(lambda: oracle.RBFKernel(1.0), float(c["sigma2"]))
    per_class = one_vs_rest_fixed_theta(X, y, 3, factory, c["thetas"], Z, 150, float(c["tol"]))
    want = np.stack([p.predict_many(Xte)[0] for _, p in per_class], axis=1)
    raw = model.predictRaw(Xte)
    assert np.abs(raw - want).max() <= TOL_PRED * max(1.0, np.abs(want).max())
