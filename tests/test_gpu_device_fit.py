"""Fitting from device-resident data (run on an H100: `pytest -m gpu`).

Every estimator and model selector takes X (and y) as CUDA tensors: the grouped and fold uploads read them in place, the
latent modes are ungrouped on the device, the K-means and greedy providers read them in place.  On the same data (the
tensor's dtype equal to the array's) the device path must give the host path's results bit for bit: the uploads' expert
sets (checked through every objective), the modes, the providers' outputs, and each estimator's theta, objective record,
active set and latent modes; G and b agree to 1e-12 relative.  X itself never crosses PCIe.
"""
import os

import numpy as np
import pytest

import oracle
import spark_gp_b200 as sg
from oracle.cpu_baseline import stats_parallel
from spark_gp_b200 import _native as N
from spark_gp_b200.hyperopt import group_for_experts
from spark_gp_b200.regression import GreedilyOptimizingActiveSetProvider, KMeansActiveSetProvider, \
    RandomActiveSetProvider

torch = pytest.importorskip("torch")
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
    if isinstance(a, torch.Tensor):
        a = a.cpu().numpy()
    return np.ascontiguousarray(a, dtype=np.float64).view(np.int64)


def cuda(a):
    return torch.as_tensor(np.ascontiguousarray(a), device="cuda:0")


def rel(a, b):
    return float(np.abs(np.asarray(a) - np.asarray(b)).max() / np.abs(np.asarray(b)).max())


def data(n, d, dtype, seed, classes=2):
    rng = np.random.default_rng(seed)
    X = rng.standard_normal((n, d)).astype(dtype)
    s = np.sin(2 * X[:, 0]) + X[:, -1] + 0.3 * rng.standard_normal(n)
    y = np.digitize(s, np.quantile(s, np.linspace(0, 1, classes + 1)[1:-1])).astype(np.float64)
    return X, y


def mk(d):
    return 1.2 * sg.ARDRBFKernel(np.linspace(0.6, 1.1, d)) + sg.const(1e-2) * sg.EyeKernel()


# ---------------- 1. uploads: the device forms give the host forms' expert sets --------------------------------------
UPLOADS = [  # (n, n_e, dtype): n % E != 0 on chip, E = 1, n just above n_e / 2, global-memory Laplace experts
    (437, 40, np.float64),
    (437, 40, np.float32),
    (90, 100, np.float32),
    (51, 100, np.float64),
    (620, 150, np.float32),
]


def objectives(eng, d, n):
    """Every objective over the current upload, and the modes each leaves: (values, gradients, modes) in call order."""
    out = []
    k = mk(d)
    out.append(eng.bcm_nll(k) + (None,))
    for step in range(2):
        v, g = eng.laplace_nll_any_size(mk(d).setHyperparameters(k.getHyperparameters() * (1 + 0.1 * step)), 1e-6)
        out.append((v, g, eng.experts_f(n)))
    v, g = eng.laplace_nll_classes_any_size(2, [1, 0], [mk(d), mk(d)], 1e-6)
    out.append((v, g, np.stack([eng.experts_f_class(c, n) for c in range(2)])))
    v, g = eng.laplace_nll_slots_any_size(3, [2, 0], [1, 0], [mk(d), mk(d)], 1e-6)
    out.append((v, g, np.stack([eng.experts_f_slot(s, n) for s in (0, 2)])))
    return out, eng.last_laplace_path()


@pytest.mark.parametrize("n,n_e,dtype", UPLOADS)
def test_grouped_upload_device_equals_host(engs, n, n_e, dtype):
    host, dev = engs
    d = 3
    X, y = data(n, d, dtype, seed=n + n_e)
    E = host.experts_upload_grouped(X, y, n_e)
    assert dev.experts_upload_grouped(cuda(X), cuda(y), n_e) == E
    a, path_a = objectives(host, d, n)
    b, path_b = objectives(dev, d, n)
    assert path_a == path_b == (1 if n_e > 117 else 0)
    for (va, ga, fa), (vb, gb, fb) in zip(a, b):
        assert np.array_equal(bits(va), bits(vb)) and np.array_equal(bits(ga), bits(gb))
        if fa is not None:
            assert np.array_equal(bits(fa), bits(fb))
    # the on-chip entry where the experts fit
    if n_e <= 117:
        host.experts_upload_grouped(X, y, n_e)
        dev.experts_upload_grouped(cuda(X), cuda(y), n_e)
        va, ga = host.laplace_nll(mk(d), 1e-6)
        vb, gb = dev.laplace_nll(mk(d), 1e-6)
        assert bits(va) == bits(vb) and np.array_equal(bits(ga), bits(gb))
        assert np.array_equal(bits(host.experts_f(n)), bits(dev.experts_f(n)))


@pytest.mark.parametrize("dtype", [np.float64, np.float32])
def test_fold_upload_device_equals_host(engs, dtype):
    host, dev = engs
    n, d, K, n_e = 700, 3, 4, 60
    X, y = data(n, d, dtype, seed=7)
    fold_of = np.random.default_rng(1).integers(0, K, n)
    ea = host.experts_upload_folds(X, y, fold_of, K, n_e)
    eb = dev.experts_upload_folds(cuda(X), cuda(y), fold_of, K, n_e)
    assert np.array_equal(ea, eb)
    kernels = [mk(d).setHyperparameters(mk(d).getHyperparameters() * (1 + 0.05 * s)) for s in range(K)]
    va, ga = host.bcm_nll_folds(list(range(K)), kernels)
    vb, gb = dev.bcm_nll_folds(list(range(K)), kernels)
    assert np.array_equal(bits(va), bits(vb)) and np.array_equal(bits(ga), bits(gb))


def raw_rc(eng, fn, *args):
    return fn(eng._h, *args)


def test_upload_refusals_launch_nothing(engs):
    eng, _ = engs
    lib = eng._lib
    X, y = data(40, 2, np.float64, seed=3)
    dX, dy = cuda(X), cuda(y)
    vp = lambda t: N.C.c_void_p(t.data_ptr()) if isinstance(t, torch.Tensor) else N.ptr(t)
    fold2 = np.zeros(40, dtype=np.int32); fold2[:20] = 1
    cases = [  # (device call, host call or None, expected code)
        ((lib.sgp_experts_upload_grouped_device, vp(dX), 0, vp(dy), 40, 2, 100),
         (lib.sgp_experts_upload_grouped, N.ptr(X), 0, N.ptr(y), 40, 2, 100), N.SGP_E_BADARG),       # E == 0
        ((lib.sgp_experts_upload_grouped_device, vp(dX), 0, vp(dy), 0, 2, 10),
         (lib.sgp_experts_upload_grouped, N.ptr(X), 0, N.ptr(y), 0, 2, 10), N.SGP_E_BADARG),         # n <= 0
        ((lib.sgp_experts_upload_grouped_device, vp(dX), 0, vp(dy), -3, 2, 10),
         (lib.sgp_experts_upload_grouped, N.ptr(X), 0, N.ptr(y), -3, 2, 10), N.SGP_E_BADARG),
        ((lib.sgp_experts_upload_grouped_device, None, 0, vp(dy), 40, 2, 10),
         (lib.sgp_experts_upload_grouped, None, 0, N.ptr(y), 40, 2, 10), N.SGP_E_BADARG),            # null
        ((lib.sgp_experts_upload_grouped_device, N.ptr(X), 0, vp(dy), 40, 2, 10), None, N.SGP_E_BADARG),  # host X
        ((lib.sgp_experts_upload_grouped_device, vp(dX), 0, N.ptr(y), 40, 2, 10), None, N.SGP_E_BADARG),  # host y
        ((lib.sgp_experts_upload_folds_device, vp(dX), 0, vp(dy), 40, 2, N.ptr(fold2), 2, 100),
         (lib.sgp_experts_upload_folds, N.ptr(X), 0, N.ptr(y), 40, 2, N.ptr(fold2), 2, 100), N.SGP_E_BADARG),  # empty set
        ((lib.sgp_experts_upload_folds_device, vp(dX), 0, vp(dy), 0, 2, N.ptr(fold2), 2, 10),
         (lib.sgp_experts_upload_folds, N.ptr(X), 0, N.ptr(y), 0, 2, N.ptr(fold2), 2, 10), N.SGP_E_BADARG),
        ((lib.sgp_experts_upload_folds_device, N.ptr(X), 0, vp(dy), 40, 2, N.ptr(fold2), 2, 10), None, N.SGP_E_BADARG),
        ((lib.sgp_experts_upload_folds_device, vp(dX), 0, None, 40, 2, N.ptr(fold2), 2, 10), None, N.SGP_E_BADARG),
    ]
    torch.cuda.synchronize()
    for dcall, hcall, code in cases:
        l0 = eng.launch_count()
        assert raw_rc(eng, *dcall) == code
        if hcall is not None:
            assert raw_rc(eng, *hcall) == code
        assert eng.launch_count() == l0


# ---------------- 2. the modes in row order -------------------------------------------------------------------------
@pytest.mark.parametrize("n,n_e", [(437, 40), (620, 150)])
def test_modes_rows_equal_host_reorder(engs, n, n_e):
    eng, _ = engs
    d = 3
    X, y = data(n, d, np.float64, seed=n)
    order = np.concatenate(group_for_experts(n, n_e))
    eng.experts_upload_grouped(cuda(X), cuda(y), n_e)
    eng.laplace_nll_any_size(mk(d), 1e-6)
    eng.laplace_nll_classes_any_size(2, [0, 1], [mk(d), mk(d)], 1e-6)
    eng.laplace_nll_slots_any_size(3, [1, 2], [1, 0], [mk(d), mk(d)], 1e-6)
    for store, index, packed in [(N.SGP_MODES_BINARY, 0, eng.experts_f(n)),
                                 (N.SGP_MODES_CLASS, 1, eng.experts_f_class(1, n)),
                                 (N.SGP_MODES_SLOT, 2, eng.experts_f_slot(2, n))]:
        latent = np.empty(n)
        latent[order] = packed
        got = eng.experts_modes_rows(store, index, n)
        assert got.is_cuda and got.dtype == torch.float64
        assert np.array_equal(bits(got), bits(latent)), store


def test_modes_rows_refusals(engs):
    eng, _ = engs
    lib = eng._lib
    n, d = 120, 2
    X, y = data(n, d, np.float64, seed=5)
    out = torch.empty(n, dtype=torch.float64, device="cuda:0")
    host_out = np.empty(n)
    eng.experts_upload_grouped(cuda(X), cuda(y), 40)

    def rc(store, index, ptr):
        l0 = eng.launch_count()
        r = lib.sgp_experts_get_f_rows_device(eng._h, store, index, ptr)
        assert eng.launch_count() == l0
        return r
    dptr = N.C.c_void_p(out.data_ptr())
    # no class / slot modes since the upload: the host getters' SGP_E_STATE
    assert rc(N.SGP_MODES_CLASS, 0, dptr) == lib.sgp_experts_get_f_class(eng._h, 0, N.ptr(host_out)) == N.SGP_E_STATE
    assert rc(N.SGP_MODES_SLOT, 0, dptr) == lib.sgp_experts_get_f_slot(eng._h, 0, N.ptr(host_out)) == N.SGP_E_STATE
    eng.laplace_nll_classes_any_size(2, [0, 1], [mk(d), mk(d)], 1e-6)
    eng.laplace_nll_slots_any_size(2, [0, 1], [1, 0], [mk(d), mk(d)], 1e-6)
    assert rc(N.SGP_MODES_CLASS, 2, dptr) == lib.sgp_experts_get_f_class(eng._h, 2, N.ptr(host_out)) == N.SGP_E_BADARG
    assert rc(N.SGP_MODES_SLOT, -1, dptr) == lib.sgp_experts_get_f_slot(eng._h, -1, N.ptr(host_out)) == N.SGP_E_BADARG
    assert rc(N.SGP_MODES_BINARY, 0, None) == lib.sgp_experts_get_f(eng._h, None) == N.SGP_E_STATE
    assert rc(7, 0, dptr) == N.SGP_E_BADARG                                   # unknown store
    assert rc(N.SGP_MODES_BINARY, 0, N.ptr(host_out)) == N.SGP_E_BADARG       # host pointer
    eng.experts_upload_folds(cuda(X), cuda(y), np.arange(n) % 2, 2, 40)        # no row order after a fold upload
    assert rc(N.SGP_MODES_BINARY, 0, dptr) == N.SGP_E_STATE


# ---------------- 3. providers ---------------------------------------------------------------------------------------
@pytest.mark.parametrize("dtype", [np.float32, np.float64])
def test_kmeans_device_equals_host(engs, dtype):
    eng, _ = engs
    rng = np.random.default_rng(11)
    X = (rng.standard_normal((5000, 6)) + 3 * rng.integers(0, 4, (5000, 1))).astype(dtype)
    a = eng.kmeans(X, 40, max_iter=20, seed=9)
    b = eng.kmeans(cuda(X), 40, max_iter=20, seed=9)
    assert np.array_equal(bits(a[0]), bits(b[0]))
    assert np.array_equal(a[1], b[1]) and a[2] == b[2] and bits(a[3]) == bits(b[3])
    lib, l0 = eng._lib, eng.launch_count()
    c, k_out, it, cost = np.empty((40, 6)), N.C.c_int32(), N.C.c_int32(), N.C.c_double()
    assert lib.sgp_kmeans_device(eng._h, N.ptr(X), int(dtype == np.float32), 5000, 6, 40, 20, 1e-4, 9, None, N.ptr(c),
                                 N.C.byref(k_out), None, N.C.byref(it), N.C.byref(cost)) == N.SGP_E_BADARG
    assert eng.launch_count() == l0


def test_greedy_device_equals_host(engs):
    eng, _ = engs
    n, d = 900, 3
    X, _ = data(n, d, np.float64, seed=21)
    y = np.sin(X.sum(1))
    k = mk(d)
    a = eng.greedy_active_set(k, X, y, 9, 5, 30)
    b = eng.greedy_active_set(k, cuda(X), cuda(y), 9, 5, 30)
    assert np.array_equal(a, b)
    desc, keep = sg.engine._make_desc(k, d)
    idx, l0 = np.empty(30, dtype=np.int64), eng.launch_count()
    assert eng._lib.sgp_greedy_active_set_device(eng._h, N.C.byref(desc), N.ptr(X), N.C.c_void_p(cuda(y).data_ptr()), n,
                                                 d, 9, 5, 30, N.ptr(idx)) == N.SGP_E_BADARG
    assert eng.launch_count() == l0


def test_providers_device_equal_host():
    n, d = 1200, 3
    X, _ = data(n, d, np.float32, seed=4)
    y = np.sin(X.astype(np.float64).sum(1))
    gp = sg.GaussianProcessRegression().setKernel(lambda: 1.0 * sg.RBFKernel(1.0)).setDatasetSizeForExpert(100)
    theta = gp.getKernel().getHyperparameters()
    for provider in (RandomActiveSetProvider, KMeansActiveSetProvider(on_gpu=True),
                     GreedilyOptimizingActiveSetProvider(first_index=3)):
        a = provider(40, X, y, gp.getKernel, theta, 5, gp=gp)
        b = provider(40, cuda(X), cuda(y), gp.getKernel, theta, 5, gp=gp)
        assert isinstance(b, np.ndarray) and np.array_equal(bits(a), bits(b)), provider


# ---------------- 4. estimators ----------------------------------------------------------------------------------------
def airfoil():
    c = np.load(os.path.join(GOLD, "airfoil_case.npz"))
    return c, c["X"], c["y"]


def mnist68():
    c = np.load(os.path.join(GOLD, "mnist68_case.npz"))
    n = int(c["n_rows"])
    X = (c["pixels"].astype(np.float64) - c["mean"]) / c["std"]
    return c, X[:n], c["y01"][:n], X[n:n + 100]


def iris():
    c = np.load(os.path.join(GOLD, "iris_case.npz"))
    return c["X"], c["y"]


def airfoil_gp():
    c, _, _ = airfoil()
    return (sg.GaussianProcessRegression().setKernel(lambda: 1 * sg.ARDRBFKernel(5) + sg.const(1) * sg.EyeKernel())
            .setSigma2(float(c["sigma2"])).setDatasetSizeForExpert(100).setActiveSetSize(150).setMaxIter(10))


def mnist_gp():
    return (sg.GaussianProcessClassifier().setDatasetSizeForExpert(100).setActiveSetSize(100)
            .setKernel(lambda: sg.RBFKernel(10.0)).setTol(1e-3).setMaxIter(3))


def iris_ovr():
    return sg.OneVsRest().setClassifier(sg.GaussianProcessClassifier().setDatasetSizeForExpert(20).setActiveSetSize(30)
                                        .setMaxIter(10))


def oracle_posterior(X, f, Z, kernel_o, theta, n_e, Xt):
    G0, b0, _ = stats_parallel(np.asarray(X, dtype=np.float64), f, Z, kernel_o, theta, n_e)
    k0 = kernel_o().set_hyperparameters(theta).set_training_vectors(Z)
    mv0, mm0 = oracle.get_magic_vector(k0, G0, b0)
    return oracle.GaussianProjectedProcessRawPredictor(mv0, mm0, k0).predict_many(Xt)


def same_objective(a, b):
    assert a.keys() == b.keys()
    for k in a:
        assert np.array_equal(bits(a[k]), bits(b[k])) if isinstance(a[k], float) else a[k] == b[k], k


@pytest.mark.parametrize("dtype", [np.float64, np.float32])
def test_regression_fit_device_equals_host(dtype):
    c, X, y = airfoil()
    X = X.astype(dtype)
    ga, gb = airfoil_gp(), airfoil_gp()
    ma = ga.fit(X, y)
    mb = gb.fit(cuda(X), cuda(y))
    assert np.array_equal(bits(ma.hyperparameters), bits(mb.hyperparameters))
    same_objective(ga.last_objective, gb.last_objective)
    Z = ma.rawPredictor.activeSet
    assert np.array_equal(bits(Z), bits(mb.rawPredictor.activeSet))
    assert rel(gb.last_stats[0], ga.last_stats[0]) < 1e-12 and rel(gb.last_stats[1], ga.last_stats[1]) < 1e-12
    mean, var = mb.rawPredictor.predict(c["Xtest"])
    s2 = float(c["sigma2"])
    ko = lambda: 1 * oracle.ARDRBFKernel(5) + oracle.const(1) * oracle.EyeKernel() + oracle.const(s2) * oracle.EyeKernel()
    m0, v0 = oracle_posterior(X, y, Z, ko, mb.hyperparameters, 100, c["Xtest"])
    assert rel(mean, m0) < TOL_PRED and np.abs(var / v0 - 1).max() < TOL_PRED


def test_classifier_fit_device_equals_host():
    c, X, y, Xte = mnist68()
    ga, gb = mnist_gp(), mnist_gp()
    ma = ga.fit(X, y)
    mb = gb.fit(cuda(X), cuda(y))
    assert np.array_equal(bits(ma.hyperparameters), bits(mb.hyperparameters))
    same_objective(ga.last_objective, gb.last_objective)
    assert gb.last_latent.is_cuda and gb.last_latent.dtype == torch.float64
    assert np.array_equal(bits(ga.last_latent), bits(gb.last_latent))
    Z = ma.rawPredictor.activeSet
    assert np.array_equal(bits(Z), bits(mb.rawPredictor.activeSet))
    assert rel(gb.last_stats[0], ga.last_stats[0]) < 1e-12 and rel(gb.last_stats[1], ga.last_stats[1]) < 1e-12
    mean, var = mb.rawPredictor.predict(Xte)
    ko = lambda: oracle.RBFKernel(10.0) + oracle.const(1e-3) * oracle.EyeKernel()
    m0, v0 = oracle_posterior(X, ga.last_latent, Z, ko, mb.hyperparameters, 100, Xte)
    assert rel(mean, m0) < TOL_PRED and np.abs(var / v0 - 1).max() < TOL_PRED


def test_one_vs_rest_fit_device_equals_host():
    X, y = iris()
    oa, ob = iris_ovr(), iris_ovr()
    ma = oa.fit(X, y)
    mb = ob.fit(cuda(X), cuda(y))
    assert np.array_equal(bits(ma.hyperparameters), bits(mb.hyperparameters))
    assert oa.last_objective["rounds"] == ob.last_objective["rounds"]
    assert oa.last_objective["launches"] == ob.last_objective["launches"]
    for ra, rb in zip(oa.last_objective["classes"], ob.last_objective["classes"]):
        same_objective(ra, rb)
    assert ob.last_latent.is_cuda and np.array_equal(bits(oa.last_latent), bits(ob.last_latent))
    for a, b in zip(ma.models, mb.models):
        assert np.array_equal(bits(a.rawPredictor.activeSet), bits(b.rawPredictor.activeSet))
        assert np.array_equal(bits(a.rawPredictor.magicVector), bits(b.rawPredictor.magicVector))
    assert np.array_equal(bits(ma.predictRaw(X)), bits(mb.predictRaw(X)))


# ---------------- 5. model selectors -----------------------------------------------------------------------------------
def synthetics():
    rng = np.random.default_rng(13)
    X = np.linspace(0, 1, 2000)[:, None]
    y = np.sin(X[:, 0]) + np.sqrt(0.01) * rng.standard_normal(2000)
    return X, y


def synthetics_cv(provider):
    gp = (sg.GaussianProcessRegression()
          .setKernel(lambda: 1 * sg.RBFKernel(0.1, 1e-6, 10) + sg.WhiteNoiseKernel(0.5, 0, 1))
          .setDatasetSizeForExpert(100).setActiveSetProvider(provider).setActiveSetSize(100).setSeed(13).setMaxIter(10))
    maps = sg.ParamGridBuilder().addGrid("sigma2", [1e-3, 1e-2]).build()
    return sg.CrossValidator().setEstimator(gp).setEstimatorParamMaps(maps).setNumFolds(3).setSeed(13)


def mnist_tvs():
    maps = sg.ParamGridBuilder().addGrid("kernel", [(lambda s: lambda: sg.RBFKernel(s))(s) for s in (9.0, 10.0)]).build()
    return (sg.TrainValidationSplit().setEstimator(mnist_gp()).setEvaluator(sg.MulticlassClassificationEvaluator("accuracy"))
            .setEstimatorParamMaps(maps).setTrainRatio(0.8).setSeed(3))


def iris_tvs():
    maps = sg.ParamGridBuilder().addGrid("sigma2", [1e-3, 1e-1]).build()
    return (sg.TrainValidationSplit().setEstimator(iris_ovr()).setEvaluator(sg.MulticlassClassificationEvaluator())
            .setEstimatorParamMaps(maps).setTrainRatio(0.8).setSeed(5))


def test_cross_validator_device_equals_host():
    X, y = synthetics()
    ca, cb = synthetics_cv(KMeansActiveSetProvider(on_gpu=True)), synthetics_cv(KMeansActiveSetProvider(on_gpu=True))
    ma = ca.fit(X, y)
    mb = cb.fit(cuda(X), cuda(y))
    assert ma.bestIndex == mb.bestIndex and np.array_equal(bits(ma.avgMetrics), bits(mb.avgMetrics))
    for key, fa in ca.last_folds.items():
        fb = cb.last_folds[key]
        for name in ("theta", "magicVector", "prediction"):
            assert np.array_equal(bits(fa[name]), bits(fb[name])), (key, name)
    assert np.array_equal(bits(ma.bestModel.hyperparameters), bits(mb.bestModel.hyperparameters))


@pytest.mark.parametrize("case", ["mnist68", "iris"])
def test_train_validation_split_device_equals_host(case):
    if case == "mnist68":
        _, X, y, _ = mnist68()
        ta, tb = mnist_tvs(), mnist_tvs()
    else:
        X, y = iris()
        ta, tb = iris_tvs(), iris_tvs()
    ma = ta.fit(X, y)
    mb = tb.fit(cuda(X), cuda(y))
    assert ma.bestIndex == mb.bestIndex and np.array_equal(bits(ma.validationMetrics), bits(mb.validationMetrics))
    for pa, pb in zip(ta.last_predictions, tb.last_predictions):
        assert np.array_equal(bits(pa), bits(pb))
    for ga, gb in zip(ma.last_objective["groups"], mb.last_objective["groups"]):
        for sa, sb in zip(ga["slots"], gb["slots"]):
            assert np.array_equal(bits(sa["theta"]), bits(sb["theta"]))
    assert np.array_equal(bits(ma.bestModel.hyperparameters), bits(mb.bestModel.hyperparameters))


# ---------------- 6. X stays on the device -------------------------------------------------------------------------------
@pytest.fixture
def host_copies(monkeypatch):
    """Records the shape of every tensor copied to the host through Tensor.cpu, Tensor.numpy and Tensor.__array__."""
    seen = []
    for name in ("cpu", "numpy", "__array__"):
        orig = getattr(torch.Tensor, name)

        def wrapped(self, *a, _orig=orig, **k):
            seen.append(tuple(self.shape))
            return _orig(self, *a, **k)
        monkeypatch.setattr(torch.Tensor, name, wrapped)
    return seen


def fit_airfoil(X, y):
    airfoil_gp().fit(X, y)


def fit_mnist(X, y):
    mnist_gp().fit(X, y)


def fit_iris(X, y):
    iris_ovr().fit(X, y)


def cv_synthetics(X, y):
    synthetics_cv(RandomActiveSetProvider).fit(X, y)


def tvs_mnist(X, y):
    mnist_tvs().fit(X, y)


@pytest.mark.parametrize("fit,load", [(fit_airfoil, lambda: airfoil()[1:]), (fit_mnist, lambda: mnist68()[1:3]),
                                      (fit_iris, iris), (cv_synthetics, synthetics), (tvs_mnist, lambda: mnist68()[1:3])])
def test_x_never_copied_to_host(host_copies, fit, load):
    X, y = load()
    dX, dy = cuda(X), cuda(y)
    host_copies.clear()
    fit(dX, dy)
    n = len(X)
    assert not [s for s in host_copies if s and s[0] >= n], host_copies


# ---------------- 7. errors before anything runs ----------------------------------------------------------------------
def test_fit_argument_errors():
    X, y = iris()
    dX, dy = cuda(X), cuda(y)
    estimators = [lambda dev=0: sg.GaussianProcessRegression(device=dev),
                  lambda dev=0: sg.GaussianProcessClassifier(device=dev),
                  lambda dev=0: sg.OneVsRest().setClassifier(sg.GaussianProcessClassifier(device=dev))]
    for make in estimators:
        with pytest.raises(ValueError):
            make(1).fit(dX, dy)                                 # the tensor is on another device than the estimator
        with pytest.raises(ValueError):
            make().fit(dX, dy[:-1])                             # y of the wrong length
        with pytest.raises(ValueError):
            make().fit(dX, y[:-1])
        with pytest.raises(ValueError):
            make().fit(dX, torch.as_tensor(y))                  # y on another device than X
    for sel in (sg.CrossValidator().setEstimator(sg.GaussianProcessRegression()),
                sg.TrainValidationSplit().setEstimator(sg.GaussianProcessRegression())
                .setEvaluator(sg.RegressionEvaluator())):
        with pytest.raises(ValueError):
            sel.fit(dX, dy[:-1])
        with pytest.raises(ValueError):
            sel.fit(dX, torch.as_tensor(y))
    with pytest.raises(RuntimeError, match="Only 0 and 1 labels"):
        sg.GaussianProcessClassifier().fit(dX, dy)              # iris labels 0, 1, 2
    with pytest.raises(ValueError, match="non-negative integers"):
        sg.OneVsRest().setClassifier(sg.GaussianProcessClassifier()).fit(dX, dy + 0.5)
    with pytest.raises(RuntimeError, match="Only 0 and 1 labels"):
        (sg.TrainValidationSplit().setEstimator(sg.GaussianProcessClassifier())
         .setEvaluator(sg.MulticlassClassificationEvaluator()).fit(dX, dy))
