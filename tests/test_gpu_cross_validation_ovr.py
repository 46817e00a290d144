"""CrossValidator over one-vs-rest on the GPU (run on an H100: `pytest -m gpu`).

`sgp_laplace_nll_fold_slots_any_size` evaluates the binary Laplace objective of several (training set, class, mode slot)
slots of one fold upload in one launch per kernel family.  Slot i's value, gradient and modes must equal, bit for bit,
what `sgp_laplace_nll_any_size` returns on a grouped upload of (X[fold != k], y[fold != k] == c) after the same sequence
of evaluations of its mode slot, whichever other slots are in the call, on the on-chip kernel, on the global-memory
kernel and in a call whose sets straddle the 117-point edge.  `CrossValidator.fit` over `OneVsRest` must then give every
(map, fold) exactly the class hyper-parameters and validation predictions of the independent
`OneVsRest().setClassifier(gp.copy(map)).fit(X[train], y[train])`.
Tolerances against the fp64 oracle are test_gpu_one_vs_rest.py's: predictions 1e-5, magic vectors 1e-3 relative.
"""
import os

import numpy as np
import pytest

import oracle
import spark_gp_b200 as sg
from oracle import cross_validation as ocv
from oracle import cross_validation_ovr as ocv_ovr
from spark_gp_b200 import _native as N
from spark_gp_b200.hyperopt import group_for_experts
from spark_gp_b200.regression import ExplicitActiveSetProvider
from spark_gp_b200.tuning import best_index
from spark_gp_b200.utils import kfold_assignment

pytestmark = pytest.mark.gpu

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
TOL_PRED, TOL_MAGIC = 1e-5, 1e-3


@pytest.fixture(scope="module")
def engs():
    a, b = sg.ProjectedProcessEngine(0), sg.ProjectedProcessEngine(0)
    yield a, b
    a.close()
    b.close()


def bits(a):
    if type(a).__module__.startswith("torch"):
        a = a.cpu().numpy()
    return np.ascontiguousarray(a, dtype=np.float64).view(np.int64)


def mk_ard(d):
    return 1.2 * sg.ARDRBFKernel(np.linspace(0.6, 1.1, d)) + sg.const(1e-2) * sg.EyeKernel()


def mk_rbf(d):
    return 1.0 * sg.RBFKernel(1.3) + sg.const(1e-2) * sg.EyeKernel()


def class_data(n, d, C, seed):
    rng = np.random.default_rng(seed)
    X = rng.standard_normal((n, d))
    s = np.sin(2 * X[:, 0]) + X[:, -1] + 0.3 * rng.standard_normal(n)
    y = np.digitize(s, np.quantile(s, np.linspace(0, 1, C + 1)[1:-1])).astype(np.float64)
    return X, y


def theta_of(mk, d, m, step):
    return mk(d).getHyperparameters() * (1.0 + 0.05 * m) * (1.0 + 0.12 * step)


def fold_call(eng, mk, d, n_mode, listed, steps, tol=1e-6):
    """One fold-slots call over listed [(mode slot, set, class)], each mode slot at its own theta for its next step."""
    kernels = [mk(d).setHyperparameters(theta_of(mk, d, m, steps[m])) for m, _, _ in listed]
    return eng.laplace_nll_fold_slots_any_size(n_mode, [m for m, _, _ in listed], [k for _, k, _ in listed],
                                               [c for _, _, c in listed], kernels, tol)


def straddle_folds(seed):
    """Two folds whose training sets have largest experts of 117 (set 0: 234 rows) and 118 points (set 1: 236 rows)."""
    fold = np.array([0] * 236 + [1] * 234, dtype=np.int32)
    return np.random.default_rng(seed).permutation(fold)


# ---------------- 1. fold slots against independent grouped uploads, bit for bit --------------------------------------
CASES = [  # (kernel, K, n, n_e, expected Laplace path); the sets are ragged (folds of unequal size)
    ("ard", 2, 330, 40, 0),
    ("rbf", 10, 450, 40, 0),
    ("ard", 3, 470, 150, 1),
    ("rbf", 2, 470, 117, 1),                      # straddles: set 0 on chip (117 points), set 1 global memory (118)
]


@pytest.mark.parametrize("kind,K,n,n_e,path", CASES)
def test_fold_slots_match_independent_uploads_bitwise(engs, kind, K, n, n_e, path):
    eng, ref = engs
    mk = {"ard": mk_ard, "rbf": mk_rbf}[kind]
    d, C = 3, 3
    X, y = class_data(n, d, C, seed=K * 100 + n_e)
    fold = straddle_folds(n_e) if n_e == 117 else kfold_assignment(n, K, n_e)
    if n_e == 117:
        nk = n - np.bincount(fold, minlength=K)
        assert [-(-int(m) // int(np.floor(m / n_e + 0.5))) for m in nk] == [117, 118]
    assert np.all(np.bincount(fold, minlength=K) > 0)
    eng.experts_upload_folds(X, y, fold, K, n_e)
    sets = [k for k in range(K)][:4]
    slot_of = [(k, c) for k in sets for c in range(C)] + [(sets[0], 1), (sets[-1], 1)]   # a set under several slots
    n_mode = len(slot_of) + 1                     # mode slot n_mode - 1 is never listed
    calls = [
        [(m, *slot_of[m]) for m in range(len(slot_of))],                       # every slot
        [(m, *slot_of[m]) for m in range(len(slot_of))][::3][::-1],            # a permuted subset, warm-started
        [(m, *slot_of[m]) for m in range(len(slot_of))][::-1],                 # every slot reversed
    ]
    steps = np.zeros(n_mode, dtype=int)
    nk = n - np.bincount(fold, minlength=K)
    got = {m: [] for m in range(len(slot_of))}
    for call in calls:
        vals, grads = fold_call(eng, mk, d, n_mode, call, steps)
        assert eng.last_laplace_path() == path
        for i, (m, k, _) in enumerate(call):
            got[m].append((vals[i], grads[i], eng.experts_f_fold_slot(k, m, nk[k])))
            steps[m] += 1
    for k in sets:
        assert np.all(eng.experts_f_fold_slot(k, n_mode - 1, nk[k]) == 0.0)
    for m, (k, c) in enumerate(slot_of):
        tr = fold != k
        ref.experts_upload_grouped(X[tr], (y[tr] == c).astype(np.float64), n_e)
        for step, (v, g, f) in enumerate(got[m]):
            v0, g0 = ref.laplace_nll_any_size(mk(d).setHyperparameters(theta_of(mk, d, m, step)), 1e-6)
            assert bits(v) == bits(v0), (m, step, v, v0)
            assert np.array_equal(bits(g), bits(g0)), (m, step)
            assert np.array_equal(bits(f), bits(ref.experts_f(nk[k]))), (m, step)


# ---------------- 2. the store: isolation and resets ----------------------------------------------------------------
def test_fold_store_isolation_and_resets(engs):
    eng, _ = engs
    d, C, K, n = 2, 3, 3, 300
    X, y = class_data(n, d, C, seed=5)
    fold = kfold_assignment(n, K, 5)
    nk = n - np.bincount(fold, minlength=K)
    eng.experts_upload_folds(X, y, fold, K, 40)
    with pytest.raises(sg.TrainingVectorsNotInitializedException):
        eng.experts_f_fold_slot(0, 0, nk[0])      # no fold slot modes since the upload
    k0 = mk_rbf(d)
    v_fresh, g_fresh = eng.laplace_nll_fold_slots_any_size(4, [2], [1], [1], [k0], 1e-6)
    f_fresh = eng.experts_f_fold_slot(1, 2, nk[1])
    assert np.any(f_fresh != 0.0) and np.all(eng.experts_f_fold_slot(1, 0, nk[1]) == 0.0)
    n_all = int(nk.sum())                         # the rows of every set, as the classes and slots entries see them
    for rnd in range(2):
        fold_modes = [eng.experts_f_fold_slot(k, m, nk[k]) for k in range(K) for m in range(4)]
        eng.bcm_nll_folds([0, 1, 2], [mk_rbf(d)] * 3)
        eng.laplace_nll_classes_any_size(C, range(C), [mk_rbf(d).setHyperparameters(theta_of(mk_rbf, d, c, rnd))
                                                       for c in range(C)], 1e-6)
        eng.laplace_nll_slots_any_size(3, [0, 2], [1, 2], [mk_rbf(d)] * 2, 1e-6)
        assert [bits(eng.experts_f_fold_slot(k, m, nk[k])).tolist() for k in range(K) for m in range(4)] == \
            [bits(f).tolist() for f in fold_modes]
        fc = [eng.experts_f_class(c, n_all) for c in range(C)]
        fs = [eng.experts_f_slot(m, n_all) for m in range(3)]
        eng.laplace_nll_fold_slots_any_size(4, [0, 3], [0, 2], [2, 0], [mk_rbf(d)] * 2, 1e-6)
        for c in range(C):
            assert np.array_equal(bits(eng.experts_f_class(c, n_all)), bits(fc[c]))
        for m in range(3):
            assert np.array_equal(bits(eng.experts_f_slot(m, n_all)), bits(fs[m]))
    # another n_mode_slots: every mode slot restarts at zero
    v, g = eng.laplace_nll_fold_slots_any_size(5, [2], [1], [1], [k0], 1e-6)
    assert bits(v[0]) == bits(v_fresh[0]) and np.array_equal(bits(g), bits(g_fresh))
    assert np.array_equal(bits(eng.experts_f_fold_slot(1, 2, nk[1])), bits(f_fresh))
    # any upload zeroes the store: a fold upload, and a grouped upload (which also leaves no fold sets)
    eng.experts_upload_folds(X, y, fold, K, 40)
    with pytest.raises(sg.TrainingVectorsNotInitializedException):
        eng.experts_f_fold_slot(1, 2, nk[1])
    v, g = eng.laplace_nll_fold_slots_any_size(5, [2], [1], [1], [k0], 1e-6)
    assert bits(v[0]) == bits(v_fresh[0]) and np.array_equal(bits(eng.experts_f_fold_slot(1, 2, nk[1])), bits(f_fresh))
    eng.experts_upload_grouped(X, y, 40)
    with pytest.raises(sg.TrainingVectorsNotInitializedException):
        eng.experts_f_fold_slot(1, 2, nk[1])


# ---------------- 3. every refusal, with its code and no launch -----------------------------------------------------
def test_fold_slots_refusals(engs):
    eng, _ = engs
    d, K, n = 2, 3, 300
    fresh = sg.ProjectedProcessEngine(0)
    fresh._experts_d = d
    with pytest.raises(sg.TrainingVectorsNotInitializedException):
        fresh.laplace_nll_fold_slots_any_size(2, [0], [0], [1], [mk_rbf(d)], 1e-6)
    X, y = class_data(n, d, 3, seed=9)
    fresh.experts_upload_grouped(X, y, 100)       # an upload, but not a fold upload
    with pytest.raises(sg.TrainingVectorsNotInitializedException):
        fresh.laplace_nll_fold_slots_any_size(2, [0], [0], [1], [mk_rbf(d)], 1e-6)
    fresh.close()
    fold = kfold_assignment(n, K, 9)
    nk = n - np.bincount(fold, minlength=K)
    eng.experts_upload_folds(X, y, fold, K, 100)
    with pytest.raises(sg.TrainingVectorsNotInitializedException):
        eng.experts_f_fold_slot(0, 0, nk[0])
    eng.laplace_nll_fold_slots_any_size(4, [0, 1, 3], [0, 1, 2], [0, 1, 1], [mk_rbf(d)] * 3, 1e-6)
    snap = [eng.experts_f_fold_slot(k, m, nk[k]) for k in range(K) for m in range(4)]

    def untouched():
        assert [bits(eng.experts_f_fold_slot(k, m, nk[k])).tolist() for k in range(K) for m in range(4)] == \
            [bits(f).tolist() for f in snap]

    bad = [
        (4, [0, 0], [0, 1], [1, 1]),              # repeated mode slot
        (4, [4], [0], [1]),                       # mode slot out of range
        (4, [-1], [0], [1]),
        (4, [0], [0], [-1]),                      # negative class
        (4, [0], [3], [1]),                       # set outside [0, n_folds)
        (4, [0], [-1], [1]),
        (1, [0, 1], [0, 0], [1, 1]),              # n_eval > n_mode_slots
        (0, [0], [0], [1]),
    ]
    for n_mode, modes, sets, classes in bad:
        launches = eng.launch_count()
        with pytest.raises(ValueError):
            eng.laplace_nll_fold_slots_any_size(n_mode, modes, sets, classes, [mk_rbf(d)] * len(modes), 1e-6)
        assert eng.launch_count() == launches
        untouched()
    launches = eng.launch_count()
    with pytest.raises(ValueError, match="same kernel structure"):
        eng.laplace_nll_fold_slots_any_size(4, [0, 1], [0, 1], [1, 1],
                                            [mk_rbf(d), sg.RBFKernel(1.3) + sg.RBFKernel(2.0)], 1e-6)
    assert eng.launch_count() == launches
    untouched()
    vals = np.zeros(1)
    z = np.zeros(1, np.int32)
    rc = eng._lib.sgp_laplace_nll_fold_slots_any_size(eng._h, 70000, N.ptr(z), N.ptr(z), N.ptr(z), 65536, None, None, 0,
                                                      1e-6, N.ptr(vals), None)
    assert rc == N.SGP_E_BADARG
    for tol in (1.0, 1.5, np.inf):
        launches = eng.launch_count()
        with pytest.raises(sg.MatrixSingularException, match="no Newton iteration runs"):
            eng.laplace_nll_fold_slots_any_size(4, [0, 1], [0, 1], [0, 1], [mk_rbf(d)] * 2, tol)
        assert eng.launch_count() == launches
        untouched()
    for set_, m in ((3, 0), (0, 4), (-1, 0)):
        with pytest.raises(ValueError):
            eng.experts_f_fold_slot(set_, m, 10)
    launches = eng.launch_count()
    with pytest.raises(sg.SgpError, match="error %d" % N.SGP_E_NOMEM):
        eng.laplace_nll_fold_slots_any_size(2 ** 31 - 1, [0], [0], [1], [mk_rbf(d)], 1e-6)
    assert eng.launch_count() == launches
    untouched()
    t = mk_ard(d).getHyperparameters()
    nan = mk_ard(d).setHyperparameters(np.concatenate([t[:1], np.full(d, np.nan)]))
    with pytest.raises(sg.NotPositiveDefiniteException, match="mode slot 3:"):
        eng.laplace_nll_fold_slots_any_size(4, [0, 3, 1], [0, 1, 2], [1, 1, 1], [mk_ard(d), nan, nan], 1e-6)
    # an expert above the global kernel's limit: one set of 46 337 points per expert
    rng = np.random.default_rng(2)
    big = 2 * 46337
    Xb = rng.standard_normal((big, 1))
    eng.experts_upload_folds(Xb, (Xb[:, 0] > 0).astype(np.float64), np.repeat([0, 1], big // 2).astype(np.int32), 2,
                             46337)
    launches = eng.launch_count()
    with pytest.raises(ValueError, match="46336"):
        eng.laplace_nll_fold_slots_any_size(1, [0], [0], [1], [mk_rbf(1)], 1e-6)
    assert eng.launch_count() == launches


# ---------------- 4. getters ---------------------------------------------------------------------------------------
def test_fold_getters_row_order(engs):
    import torch
    eng, ref = engs
    d, K, n, n_e = 3, 4, 400, 30
    X, y = class_data(n, d, 3, seed=12)
    fold = kfold_assignment(n, K, 12)
    nk = n - np.bincount(fold, minlength=K)
    gp = (sg.GaussianProcessClassifier().setDatasetSizeForExpert(n_e).setSigma2(1e-2).setTol(1e-6).setActiveSetSize(10)
          .setKernel(lambda: 1.2 * sg.ARDRBFKernel(np.linspace(0.6, 1.1, d))))
    mk = lambda _: gp.getKernel()
    eng.experts_upload_folds(X, y, fold, K, n_e)
    listed = [(m, k, m % 3) for m, k in enumerate(range(K))]
    fold_call(eng, mk, d, K, listed, np.zeros(K, dtype=int))
    for m, k, c in listed:
        tr = fold != k
        gp.fit(X[tr], (y[tr] == c).astype(np.float64), hyperparameters=theta_of(mk, d, m, 0))
        rows = eng.experts_f_fold_slot_rows(k, m, nk[k])
        assert rows.is_cuda and rows.dtype == torch.float64
        assert np.array_equal(bits(rows), bits(gp.last_latent)), (m, k)
        packed = eng.experts_f_fold_slot(k, m, nk[k])
        host = np.empty(nk[k])
        host[np.concatenate(group_for_experts(nk[k], n_e))] = packed
        assert np.array_equal(bits(host), bits(gp.last_latent)), (m, k)
    f = torch.empty(n, dtype=torch.float64, device="cuda:0")
    rc = eng._lib.sgp_experts_get_f_rows_device(eng._h, N.SGP_MODES_BINARY, 0, N.C.c_void_p(f.data_ptr()))
    assert rc == N.SGP_E_STATE                    # a fold upload has no single row order


# ---------------- 5. Iris as the reference writes it ---------------------------------------------------------------
def iris():
    c = np.load(os.path.join(GOLD, "iris_case.npz"))
    return c, c["X"], c["y"]


def iris_ovr(**extra):
    gp = sg.GaussianProcessClassifier().setDatasetSizeForExpert(20).setActiveSetSize(30)
    for name, v in extra.items():
        gp = gp.copy({name: v})
    return sg.OneVsRest().setClassifier(gp)


def check_folds_against_independent(cv, model, ovr, maps, X, y, fold_of, K):
    for p, m in enumerate(maps):
        for k in range(K):
            tr = fold_of != k
            ind = ovr.copy(m).fit(X[tr], y[tr])
            out = cv.last_folds[p, k]
            assert np.array_equal(bits(out["theta"]), bits(ind.hyperparameters)), (p, k)
            for c in range(ind.numClasses):
                assert np.array_equal(bits(out["magicVector"][c]), bits(ind.models[c].rawPredictor.magicVector)), (p, k)
            assert np.array_equal(bits(out["prediction"]), bits(ind.predict(X[~tr]))), (p, k)
            del ind
    ev = cv._evaluator
    metrics = model.last_objective["fold_metrics"]
    for p in range(len(maps)):
        for k in range(K):
            assert metrics[p, k] == ev.evaluate(y[fold_of == k], cv.last_folds[p, k]["prediction"])
        assert model.avgMetrics[p] == sum(metrics[p, k] for k in range(K)) / K
    assert model.bestIndex == best_index(model.avgMetrics, ev.isLargerBetter())


def test_cv_iris_equals_independent_fits():
    c, X, y = iris()
    K = 10
    ovr = iris_ovr()
    maps = sg.ParamGridBuilder().addGrid("sigma2", [1e-3, 1e-1]).build()
    cv = (sg.CrossValidator().setEstimator(ovr).setEvaluator(sg.MulticlassClassificationEvaluator("accuracy"))
          .setEstimatorParamMaps(maps).setNumFolds(K).setSeed(1))
    model = cv.fit(X, y)
    fold_of = kfold_assignment(len(X), K, 1)
    check_folds_against_independent(cv, model, ovr, maps, X, y, fold_of, K)
    best = ovr.copy(maps[model.bestIndex]).fit(X, y)
    for k in range(3):
        assert np.array_equal(bits(model.bestModel.models[k].rawPredictor.magicVector),
                              bits(best.models[k].rawPredictor.magicVector))
    assert np.array_equal(model.predict(X), best.predict(X))
    (group,) = model.last_objective["groups"]
    assert group["calls"] == group["rounds"] + 1
    assert group["rounds"] == max(s["evaluations"] for s in group["slots"])
    assert len(group["slots"]) == len(maps) * K * 3
    assert min(model.avgMetrics) > 0.8


# ---------------- 6. fixed theta against the oracle ----------------------------------------------------------------
def test_cv_fixed_theta_vs_oracle():
    c, X, y = iris()
    K = 3
    fold_of = kfold_assignment(len(X), K, 2)
    Z = X[c["active_idx"]]
    sigma2 = 1e-3
    ovr = iris_ovr(maxIter=0, sigma2=sigma2, activeSetProvider=ExplicitActiveSetProvider(Z))
    cv = (sg.CrossValidator().setEstimator(ovr).setEvaluator(sg.MulticlassClassificationEvaluator("accuracy"))
          .setNumFolds(K))
    model = cv.fit(X, y, folds=fold_of)
    (group,) = model.last_objective["groups"]
    assert group["rounds"] == 0 and group["calls"] == 1
    gp = ovr.getClassifier()
    factory = oracle.get_kernel(lambda: oracle.RBFKernel(1.0), sigma2)       # the default kernel, RBFKernel()
    for k in range(K):
        theta = cv.last_folds[0, k]["theta"]
        Ck, classes, raw, pred = ocv_ovr.fold_one_vs_rest_fixed_theta(X, y, fold_of, k, factory, theta, Z, 20, gp._tol)
        assert theta.shape[0] == Ck
        for cc, (_, mv) in enumerate(classes):
            got = cv.last_folds[0, k]["magicVector"][cc]
            assert np.abs(got - mv).max() / np.abs(mv).max() < TOL_MAGIC, (k, cc)
        top2 = np.sort(raw, axis=1)[:, -2:]
        clear = top2[:, 1] - top2[:, 0] > TOL_PRED * max(1.0, np.abs(raw).max())
        assert np.array_equal(cv.last_folds[0, k]["prediction"][clear], pred[clear]), k


# ---------------- 7. a training set without the top class ----------------------------------------------------------
def test_cv_missing_class_matches_independent_fits():
    c, X, y = iris()
    K = 3
    fold_of = kfold_assignment(len(X), K, 3)
    fold_of[y == 2] = 0                           # fold 0 holds every row of class 2: its training set lacks it
    ovr = iris_ovr(maxIter=3)
    cv = sg.CrossValidator().setEstimator(ovr).setEvaluator(sg.MulticlassClassificationEvaluator()).setNumFolds(K)
    model = cv.fit(X, y, folds=fold_of)
    assert cv.last_folds[0, 0]["theta"].shape[0] == 2 and cv.last_folds[0, 1]["theta"].shape[0] == 3
    check_folds_against_independent(cv, model, ovr, [{}], X, y, fold_of, K)


# ---------------- 8. a grid over two kernel structures -------------------------------------------------------------
def test_cv_two_kernel_structures(monkeypatch):
    c, X, y = iris()
    K = 3
    uploads = []
    orig = sg.ProjectedProcessEngine.experts_upload_folds

    def counting(self, *a, **k):
        uploads.append(1)
        return orig(self, *a, **k)
    monkeypatch.setattr(sg.ProjectedProcessEngine, "experts_upload_folds", counting)
    ovr = iris_ovr(maxIter=4)
    maps = sg.ParamGridBuilder().addGrid("kernel", [lambda: sg.RBFKernel(1.0),
                                                    lambda: sg.ARDRBFKernel(np.ones(4))]).build()
    cv = (sg.CrossValidator().setEstimator(ovr).setEvaluator(sg.MulticlassClassificationEvaluator("accuracy"))
          .setEstimatorParamMaps(maps).setNumFolds(K).setSeed(4))
    model = cv.fit(X, y)
    groups = model.last_objective["groups"]
    assert len(groups) == 2 and len(uploads) == 2
    for p, g in enumerate(groups):
        assert {s["map"] for s in g["slots"]} == {p}
        assert g["calls"] == g["rounds"] + 1
        assert g["launches"] == 3 * g["calls"]    # per call: the on-chip kernel, its row sum and the status words
    monkeypatch.undo()
    check_folds_against_independent(cv, model, ovr, maps, X, y, kfold_assignment(len(X), K, 4), K)


# ---------------- 9. CUDA tensors --------------------------------------------------------------------------------
def test_cv_cuda_tensors_equal_host(monkeypatch):
    import torch
    c, X, y = iris()
    K = 5
    make = lambda: (sg.CrossValidator().setEstimator(iris_ovr(maxIter=5))
                    .setEvaluator(sg.MulticlassClassificationEvaluator("accuracy"))
                    .setEstimatorParamMaps(sg.ParamGridBuilder().addGrid("sigma2", [1e-3, 1e-2]).build())
                    .setNumFolds(K).setSeed(6))
    host_cv = make()
    host = host_cv.fit(X, y)
    seen = []
    for name in ("cpu", "numpy", "__array__"):
        orig = getattr(torch.Tensor, name)

        def wrapped(self, *a, _orig=orig, **k):
            seen.append(tuple(self.shape))
            return _orig(self, *a, **k)
        monkeypatch.setattr(torch.Tensor, name, wrapped)
    dev_cv = make()
    dev = dev_cv.fit(torch.as_tensor(X, device="cuda:0"), torch.as_tensor(y, device="cuda:0"))
    monkeypatch.undo()
    assert not [s for s in seen if s and s[0] >= len(X)], seen
    assert dev.avgMetrics == host.avgMetrics and dev.bestIndex == host.bestIndex
    for key, out in host_cv.last_folds.items():
        assert np.array_equal(bits(dev_cv.last_folds[key]["theta"]), bits(out["theta"])), key
        assert np.array_equal(bits(dev_cv.last_folds[key]["prediction"]), bits(out["prediction"])), key
        for a, b in zip(dev_cv.last_folds[key]["magicVector"], out["magicVector"]):
            assert np.array_equal(bits(a), bits(b)), key
