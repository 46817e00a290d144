"""TrainValidationSplit on the GPU (run on an H100: `pytest -m gpu`).

`sgp_laplace_nll_slots_any_size` evaluates the binary Laplace objective of several (map, class) slots in one launch,
each slot with latent modes of its own.  Slot i's value, gradient and modes must equal, bit for bit, what
`sgp_laplace_nll_any_size` returns on an upload of the labels (y == classes[i]) after the same sequence of evaluations of
its mode slot, whichever other slots are in the call, on the on-chip kernel (experts of at most 117 points) and on the
global-memory kernel.  `TrainValidationSplit.fit` must then give every param map exactly the validation predictions of
the independent `estimator.copy(map).fit(X[train], y[train])`.
"""
import os

import numpy as np
import pytest

import oracle
import spark_gp_b200 as sg
from oracle import train_validation_split as otvs
from spark_gp_b200 import _native as N
from spark_gp_b200.hyperopt import pack_experts
from spark_gp_b200.regression import ExplicitActiveSetProvider
from spark_gp_b200.tuning import best_index

pytestmark = pytest.mark.gpu

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")


@pytest.fixture(scope="module")
def engs():
    a, b = sg.ProjectedProcessEngine(0), sg.ProjectedProcessEngine(0)
    yield a, b
    a.close()
    b.close()


def bits(a):
    return np.ascontiguousarray(a, dtype=np.float64).view(np.int64)


def mk_ard(d):
    return 1.2 * sg.ARDRBFKernel(np.linspace(0.6, 1.1, d)) + sg.const(1e-2) * sg.EyeKernel()


def mk_rbf(d):
    return 1.0 * sg.RBFKernel(1.3) + sg.const(1e-2) * sg.EyeKernel()


def class_data(N_, d, C, seed):
    rng = np.random.default_rng(seed)
    X = rng.standard_normal((N_, d))
    s = np.sin(2 * X[:, 0]) + X[:, -1] + 0.3 * rng.standard_normal(N_)
    y = np.digitize(s, np.quantile(s, np.linspace(0, 1, C + 1)[1:-1])).astype(np.float64)
    return X, y


def theta_of(mk, d, m, step):
    return mk(d).getHyperparameters() * (1.0 + 0.05 * m) * (1.0 + 0.12 * step)


def slots_call(eng, mk, d, n_mode_slots, listed, steps, tol=1e-6):
    """One slots call over listed [(mode slot, class)], each mode slot at its own theta for its next step."""
    kernels = [mk(d).setHyperparameters(theta_of(mk, d, m, steps[m])) for m, _ in listed]
    return eng.laplace_nll_slots_any_size(n_mode_slots, [m for m, _ in listed], [c for _, c in listed], kernels, tol)


# ---------------- 1. the slot entry against single uploads of (y == c), bit for bit ------------------------------------
CASES = [  # (kernel, n_e, ragged, E, d, expected Laplace path)
    ("ard", 40, True, 5, 3, 0),
    ("rbf", 117, False, 3, 2, 0),
    ("ard", 150, True, 3, 4, 1),
    ("rbf", 300, False, 2, 3, 1),
]


@pytest.mark.parametrize("kind,n_e,ragged,E,d,path", CASES)
def test_slots_match_single_uploads_bitwise(engs, kind, n_e, ragged, E, d, path):
    eng, ref = engs
    mk = {"ard": mk_ard, "rbf": mk_rbf}[kind]
    C, P = 3, 2                                   # mode slot p * C + c; class 1 shared by both maps and a binary slot
    N_ = E * n_e + (E // 2 if ragged else 0)
    assert int(np.floor(N_ / n_e + 0.5)) == E
    X, y = class_data(N_, d, C, seed=n_e * 10 + d)
    eng.experts_upload(*pack_experts(X, y, n_e))
    n_mode = P * C + 1
    cls_of = {p * C + c: c for p in range(P) for c in range(C)}
    cls_of[P * C] = 1                             # a further slot of class 1 (several maps sharing class 1)
    calls = [
        [(m, cls_of[m]) for m in range(n_mode)],                  # every slot
        [(m, cls_of[m]) for m in (6, 4, 1, 3)],                   # a permuted subset, warm-started
        [(m, cls_of[m]) for m in range(n_mode)][::-1],            # every slot reversed
        [(1, 1)],                                                 # one slot alone
    ]
    steps = np.zeros(n_mode, dtype=int)
    got = {m: [] for m in range(n_mode)}
    for k, call in enumerate(calls):
        before = {m: eng.experts_f_slot(m, N_) for m in range(n_mode)} if k > 0 else None
        vals, grads = slots_call(eng, mk, d, n_mode, call, steps)
        assert eng.last_laplace_path() == path
        listed = [m for m, _ in call]
        for i, m in enumerate(listed):
            got[m].append((vals[i], grads[i], eng.experts_f_slot(m, N_)))
            steps[m] += 1
        if before is not None:                    # mode slots not listed keep their modes
            for m in set(range(n_mode)) - set(listed):
                assert np.array_equal(bits(eng.experts_f_slot(m, N_)), bits(before[m])), (k, m)
    for m in range(n_mode):
        ref.experts_upload(*pack_experts(X, (y == cls_of[m]).astype(np.float64), n_e))
        for step, (v, g, f) in enumerate(got[m]):
            v0, g0 = ref.laplace_nll_any_size(mk(d).setHyperparameters(theta_of(mk, d, m, step)), 1e-6)
            assert bits(v) == bits(v0), (m, step, v, v0)
            assert np.array_equal(bits(g), bits(g0)), (m, step)
            assert np.array_equal(bits(f), bits(ref.experts_f(N_))), (m, step)


@pytest.mark.parametrize("n_e", [60, 200])
def test_store_resets_and_classes_entry_interleaved(engs, n_e):
    eng, _ = engs
    d, C = 2, 3
    X, y = class_data(3 * n_e, d, C, seed=n_e)
    N_ = len(X)
    eng.experts_upload(*pack_experts(X, y, n_e))
    with pytest.raises(sg.TrainingVectorsNotInitializedException):
        eng.experts_f_slot(0, N_)                 # no slot modes since the upload
    k0 = mk_rbf(d)
    v_fresh, g_fresh = eng.laplace_nll_slots_any_size(4, [2], [1], [k0], 1e-6)
    f_fresh = eng.experts_f_slot(2, N_)
    assert np.any(f_fresh != 0.0) and np.all(eng.experts_f_slot(0, N_) == 0.0)
    # classes-entry calls interleaved: neither store moves the other
    fc_before = None
    for rnd in range(2):
        slot_modes = [eng.experts_f_slot(m, N_) for m in range(4)]
        kc = [mk_rbf(d).setHyperparameters(theta_of(mk_rbf, d, c, rnd)) for c in range(C)]
        eng.laplace_nll_classes_any_size(C, range(C), kc, 1e-6)
        for m in range(4):
            assert np.array_equal(bits(eng.experts_f_slot(m, N_)), bits(slot_modes[m]))
        fc_before = [eng.experts_f_class(c, N_) for c in range(C)]
        ks = [mk_rbf(d).setHyperparameters(theta_of(mk_rbf, d, m, rnd + 1)) for m in (0, 2)]
        eng.laplace_nll_slots_any_size(4, [0, 2], [1, 1], ks, 1e-6)
        for c in range(C):
            assert np.array_equal(bits(eng.experts_f_class(c, N_)), bits(fc_before[c]))
    # another n_mode_slots: every mode slot restarts at zero, so slot 2 at theta0 gives the fresh result again
    v, g = eng.laplace_nll_slots_any_size(5, [2], [1], [k0], 1e-6)
    assert bits(v[0]) == bits(v_fresh[0]) and np.array_equal(bits(g), bits(g_fresh))
    assert np.array_equal(bits(eng.experts_f_slot(2, N_)), bits(f_fresh))
    assert np.all(eng.experts_f_slot(0, N_) == 0.0)
    with pytest.raises(ValueError):
        eng.experts_f_slot(5, N_)
    # an upload resets the store too
    eng.experts_upload(*pack_experts(X, y, n_e))
    with pytest.raises(sg.TrainingVectorsNotInitializedException):
        eng.experts_f_slot(2, N_)
    v, g = eng.laplace_nll_slots_any_size(5, [2], [1], [k0], 1e-6)
    assert bits(v[0]) == bits(v_fresh[0]) and np.array_equal(bits(eng.experts_f_slot(2, N_)), bits(f_fresh))


# ---------------- 2. every error ---------------------------------------------------------------------------------------
def test_slots_errors(engs):
    eng, _ = engs
    d = 2
    fresh = sg.ProjectedProcessEngine(0)                  # no upload: SGP_E_STATE
    fresh._experts_d = d
    with pytest.raises(sg.TrainingVectorsNotInitializedException):
        fresh.laplace_nll_slots_any_size(2, [0], [1], [mk_rbf(d)], 1e-6)
    with pytest.raises(sg.TrainingVectorsNotInitializedException):
        fresh.experts_f_slot(0, 10)
    fresh.close()
    X, y = class_data(300, d, 3, seed=9)
    eng.experts_upload(*pack_experts(X, y, 100))
    eng.laplace_nll_slots_any_size(4, [0, 1, 3], [0, 1, 1], [mk_rbf(d)] * 3, 1e-6)
    snap = [eng.experts_f_slot(m, 300) for m in range(4)]

    def untouched():
        for m in range(4):
            assert np.array_equal(bits(eng.experts_f_slot(m, 300)), bits(snap[m])), m

    bad = [
        (4, [0, 0], [1, 1]),                      # repeated mode slot
        (4, [4], [1]),                            # out of range
        (4, [-1], [1]),
        (4, [0], [-1]),                           # negative class
        (1, [0, 1], [1, 1]),                      # n_eval > n_mode_slots
        (0, [0], [1]),
    ]
    for n_mode, modes, classes in bad:
        launches = eng.launch_count()
        with pytest.raises(ValueError):
            eng.laplace_nll_slots_any_size(n_mode, modes, classes, [mk_rbf(d)] * len(modes), 1e-6)
        assert eng.launch_count() == launches
        untouched()
    with pytest.raises(ValueError, match="same kernel structure"):
        eng.laplace_nll_slots_any_size(4, [0, 1], [1, 1], [mk_rbf(d), sg.RBFKernel(1.3) + sg.RBFKernel(2.0)], 1e-6)
    untouched()
    # n_eval above 65535, refused before the lists are read
    vals = np.zeros(1)
    rc = eng._lib.sgp_laplace_nll_slots_any_size(eng._h, 70000, N.ptr(np.zeros(1, np.int32)),
                                                 N.ptr(np.zeros(1, np.int32)), 65536, None, None, 0, 1e-6,
                                                 N.ptr(vals), None)
    assert rc == N.SGP_E_BADARG
    # tol >= 1: no Newton iteration runs -> MatrixSingularException before any launch, every mode as it was
    for tol in (1.0, 1.5, np.inf):
        launches = eng.launch_count()
        with pytest.raises(sg.MatrixSingularException, match="no Newton iteration runs"):
            eng.laplace_nll_slots_any_size(4, [0, 1], [0, 1], [mk_rbf(d)] * 2, tol)
        assert eng.launch_count() == launches
        untouched()
    with pytest.raises(ValueError):
        eng.experts_f_slot(4, 300)
    # a store larger than the device: SGP_E_NOMEM before any launch, and the store of 4 slots stays usable
    launches = eng.launch_count()
    with pytest.raises(sg.SgpError, match="error %d" % N.SGP_E_NOMEM):
        eng.laplace_nll_slots_any_size(2 ** 31 - 1, [0], [1], [mk_rbf(d)], 1e-6)
    assert eng.launch_count() == launches
    untouched()
    # B not positive definite (NaN feature scales make every pivot NaN): SGP_E_NOT_PD naming the first listed failing
    # mode slot
    t = mk_ard(d).getHyperparameters()
    nan = mk_ard(d).setHyperparameters(np.concatenate([t[:1], np.full(d, np.nan)]))
    with pytest.raises(sg.NotPositiveDefiniteException, match="mode slot 3:"):
        eng.laplace_nll_slots_any_size(4, [0, 3, 1], [1, 1, 1], [mk_ard(d), nan, nan], 1e-6)


def test_slots_global_workspace_too_large(engs):
    """One expert of 75 000 points needs a 90 GB workspace slice: SGP_E_NOMEM before any launch."""
    eng, _ = engs
    rng = np.random.default_rng(8)
    n = 75000
    X = rng.standard_normal((n, 1)); y = (X[:, 0] > 0).astype(np.float64)
    eng.experts_upload(X, y, np.array([0, n]))
    launches = eng.launch_count()
    with pytest.raises(sg.SgpError, match="error %d" % N.SGP_E_NOMEM):
        eng.laplace_nll_slots_any_size(2, [1], [1], [sg.RBFKernel(1.0) + sg.const(1e-2) * sg.EyeKernel()], 1e-6)
    assert eng.launch_count() == launches


# ---------------- 3. TrainValidationSplit over the binary classifier on the mnist68 rows --------------------------------
def mnist68():
    c = np.load(os.path.join(GOLD, "mnist68_case.npz"))
    X = (c["pixels"].astype(np.float64) - c["mean"]) / c["std"]
    return c, X, c["y01"]


def check_against_independent(tvs, model, est, maps, X, y, mask):
    """Every map's validation predictions, the metrics, the best index and the best model equal the independent fits'."""
    ev = tvs._evaluator
    for p, m in enumerate(maps):
        ind = est.copy(m).fit(X[mask], y[mask])
        assert np.array_equal(bits(tvs.last_predictions[p]), bits(ind.predict(X[~mask]))), p
        assert model.validationMetrics[p] == ev.evaluate(y[~mask], tvs.last_predictions[p])
        del ind
    assert model.bestIndex == best_index(model.validationMetrics, ev.isLargerBetter())
    return est.copy(maps[model.bestIndex]).fit(X, y)


@pytest.mark.parametrize("n_e,sigmas", [(100, [8.0, 10.0, 12.0]), (200, [9.0, 11.0])])
def test_tvs_binary_mnist68_equals_independent_fits(n_e, sigmas):
    c, X, y = mnist68()
    gp = (sg.GaussianProcessClassifier().setDatasetSizeForExpert(n_e).setActiveSetSize(100)
          .setKernel(lambda: sg.RBFKernel(10.0)).setTol(1e-3).setMaxIter(5))
    maps = sg.ParamGridBuilder().addGrid("kernel", [(lambda s: lambda: sg.RBFKernel(s))(s) for s in sigmas]).build()
    tvs = (sg.TrainValidationSplit().setEstimator(gp).setEvaluator(sg.MulticlassClassificationEvaluator("accuracy"))
           .setEstimatorParamMaps(maps).setTrainRatio(0.8).setSeed(3))
    model = tvs.fit(X, y)
    mask = otvs.train_mask(len(X), 0.8, 3)
    assert len(model.validationMetrics) == len(maps)
    best = check_against_independent(tvs, model, gp, maps, X, y, mask)
    assert np.array_equal(bits(model.bestModel.rawPredictor.magicVector), bits(best.rawPredictor.magicVector))
    assert np.array_equal(model.predict(X[:50]), best.predict(X[:50]))
    (group,) = model.last_objective["groups"]
    assert group["calls"] == group["rounds"] + 1
    assert group["rounds"] == max(s["evaluations"] for s in group["slots"])
    assert [s["mode_slot"] for s in group["slots"]] == list(range(len(maps)))
    assert min(model.validationMetrics) > 0.9


@pytest.mark.parametrize("n_e", [100, 200])
def test_tvs_binary_fixed_theta_accuracy_vs_oracle(n_e):
    """maxIter = 0: every map keeps its kernel's own theta; with the active set given, each map's validation accuracy is
    the oracle pipeline's (Laplace modes from zero, projected process with y := f, class 1 iff f* > 0).  Rows whose
    oracle f* is below 1e-6 of the largest (images far from every active point, f* ~ 1e-50) may take either class."""
    c, X, y = mnist68()
    mask = otvs.train_mask(len(X), 0.8, 4)
    Xtr = X[mask]
    Z = Xtr[::len(Xtr) // 100][:100]
    sigma2 = float(c["sigma2"])
    gp = (sg.GaussianProcessClassifier().setDatasetSizeForExpert(n_e).setActiveSetSize(100).setSigma2(sigma2)
          .setKernel(lambda: sg.RBFKernel(10.0)).setTol(1e-3).setMaxIter(0)
          .setActiveSetProvider(ExplicitActiveSetProvider(Z)))
    sigmas = [9.0, 10.0]
    maps = sg.ParamGridBuilder().addGrid("kernel", [(lambda s: lambda: sg.RBFKernel(s))(s) for s in sigmas]).build()
    tvs = (sg.TrainValidationSplit().setEstimator(gp).setEvaluator(sg.MulticlassClassificationEvaluator("accuracy"))
           .setEstimatorParamMaps(maps).setTrainRatio(0.8).setSeed(4))
    model = tvs.fit(X, y)
    check_against_independent(tvs, model, gp, maps, X, y, mask)
    assert model.last_objective["groups"][0]["calls"] == 1 and model.last_objective["groups"][0]["rounds"] == 0
    for p, s in enumerate(sigmas):
        factory = oracle.get_kernel(lambda s=s: oracle.RBFKernel(s), sigma2)
        theta = factory().get_hyperparameters()
        fstar, pred = otvs.binary_fixed_theta_predictions(Xtr, y[mask], X[~mask], factory, theta, Z, n_e, 1e-3)
        clear = np.abs(fstar) > 1e-6 * np.abs(fstar).max()
        assert np.array_equal(tvs.last_predictions[p][clear], pred[clear]), p
        n_val = len(pred)
        assert abs(model.validationMetrics[p] - otvs.metric("accuracy", y[~mask], pred)) * n_val <= (~clear).sum() + 1e-9
        assert model.validationMetrics[p] > 0.95


# ---------------- 4. TrainValidationSplit over one-vs-rest on the Iris rows ---------------------------------------------
def test_tvs_one_vs_rest_iris_equals_independent_fits():
    c = np.load(os.path.join(GOLD, "iris_case.npz"))
    X, y = c["X"], c["y"]
    ovr = sg.OneVsRest().setClassifier(sg.GaussianProcessClassifier().setDatasetSizeForExpert(20).setActiveSetSize(30))
    maps = sg.ParamGridBuilder().addGrid("sigma2", [1e-3, 1e-1]).build()
    tvs = (sg.TrainValidationSplit().setEstimator(ovr).setEvaluator(sg.MulticlassClassificationEvaluator())
           .setEstimatorParamMaps(maps).setTrainRatio(0.8).setSeed(5))
    model = tvs.fit(X, y)
    mask = otvs.train_mask(len(X), 0.8, 5)
    for p, m in enumerate(maps):                  # each (map, class) slot follows the independent class's optimisation
        ind = ovr.copy(m)
        ind_model = ind.fit(X[mask], y[mask])
        slots = [s for s in model.last_objective["groups"][0]["slots"] if s["map"] == p]
        assert [s["cls"] for s in slots] == [0, 1, 2]
        for s in slots:
            assert np.array_equal(bits(s["theta"]), bits(ind_model.hyperparameters[s["cls"]]))
            assert s["evaluations"] == ind.last_objective["classes"][s["cls"]]["evaluations"]
    best = check_against_independent(tvs, model, ovr, maps, X, y, mask)
    for k in range(3):
        assert np.array_equal(bits(model.bestModel.models[k].rawPredictor.magicVector),
                              bits(best.models[k].rawPredictor.magicVector))
    (group,) = model.last_objective["groups"]
    assert group["calls"] == group["rounds"] + 1         # one slots call per optimisation round, one at theta*
    assert group["rounds"] == max(s["evaluations"] for s in group["slots"])
    assert np.array_equal(model.transform(X), best.predict(X))
    assert min(model.validationMetrics) > 0.8


# ---------------- 5. TrainValidationSplit over regression ---------------------------------------------------------------
def test_tvs_regression_equals_independent_fits():
    rng = np.random.default_rng(17)
    X = rng.random((900, 3))
    y = np.sin(3 * X.sum(1)) + 0.05 * rng.standard_normal(900)
    gp = (sg.GaussianProcessRegression().setKernel(lambda: 1.0 * sg.ARDRBFKernel(np.ones(3)))
          .setDatasetSizeForExpert(50).setActiveSetSize(40).setMaxIter(10))
    maps = sg.ParamGridBuilder().addGrid("sigma2", [1e-3, 1e-2]).addGrid("activeSetSize", [30, 40]).build()
    tvs = (sg.TrainValidationSplit().setEstimator(gp).setEvaluator(sg.RegressionEvaluator("rmse"))
           .setEstimatorParamMaps(maps).setSeed(2))
    model = tvs.fit(X, y)
    mask = otvs.train_mask(len(X), 0.75, 2)
    best = check_against_independent(tvs, model, gp, maps, X, y, mask)
    assert np.array_equal(bits(model.bestModel.rawPredictor.magicVector), bits(best.rawPredictor.magicVector))
    assert len(model.last_objective["maps"]) == len(maps)
    assert min(model.validationMetrics) < 0.2
