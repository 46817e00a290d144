"""Cross-validation of the regression estimator on the GPU (run on an H100: `pytest -m gpu`).

`sgp_bcm_nll_folds` evaluates the BCM objective of several fold training sets in one launch.  Slot s must return, bit
for bit, what `sgp_bcm_nll` returns on a grouped upload of that fold's training rows.  `CrossValidator.fit` must then
give every (map, fold) slot exactly the independent `estimator.copy(map).fit(X[train], y[train])` result.

Tolerances against the fp64 oracle (written here once): 1e-9 relative on the value, 1e-8 on the gradient (relative to its
largest component), as the per-expert objective tests.
"""
import os
import subprocess
import sys

import numpy as np
import pytest

import oracle
import spark_gp_b200 as sg
from oracle.cross_validation import fold_bcm_objective
from spark_gp_b200.regression import KMeansActiveSetProvider
from spark_gp_b200.utils import kfold_assignment

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLD = os.path.join(ROOT, "tests", "golden")
TOL_VAL, TOL_GRAD = 1e-9, 1e-8


@pytest.fixture(scope="module")
def engs():
    a, b = sg.ProjectedProcessEngine(0), sg.ProjectedProcessEngine(0)
    yield a, b
    a.close()
    b.close()


def bits(a):
    return np.ascontiguousarray(a, dtype=np.float64).view(np.int64)


KERNELS = {
    "ard": (lambda d: 1.2 * sg.ARDRBFKernel(np.linspace(0.6, 1.1, d)) + sg.const(1e-2) * sg.EyeKernel(),
            lambda d: 1.2 * oracle.ARDRBFKernel(np.linspace(0.6, 1.1, d)) + oracle.const(1e-2) * oracle.EyeKernel()),
    "rbf": (lambda d: sg.RBFKernel(1.3) + sg.const(1e-2) * sg.EyeKernel(),
            lambda d: oracle.RBFKernel(1.3) + oracle.const(1e-2) * oracle.EyeKernel()),
    "two_term": (lambda d: 1.5 * sg.ARDRBFKernel(np.full(d, 0.7)) + 0.5 * sg.RBFKernel(2.0) + sg.const(1e-2) * sg.EyeKernel(),
                 lambda d: 1.5 * oracle.ARDRBFKernel(np.full(d, 0.7)) + 0.5 * oracle.RBFKernel(2.0)
                 + oracle.const(1e-2) * oracle.EyeKernel()),
    "eye_only": (lambda d: sg.const(0.3) * sg.EyeKernel() + sg.const(1e-2) * sg.EyeKernel(),
                 lambda d: oracle.const(0.3) * oracle.EyeKernel() + oracle.const(1e-2) * oracle.EyeKernel()),
}


def data(N, d, seed):
    rng = np.random.default_rng(seed)
    X = rng.standard_normal((N, d))
    y = np.sin(2 * X[:, 0]) + X[:, -1] + 0.1 * rng.standard_normal(N)
    return X, y


def theta_of(mk, d, s):
    t0 = mk(d).getHyperparameters()
    return t0 * (1.0 + 0.05 * (s % 7))


def check_slots(eng, ref, X, y, fold_of, K, n_e, mk, sets, f32=False):
    """Slots over `sets` (each at its own theta) against single-set grouped uploads, bit for bit."""
    Xu = X.astype(np.float32) if f32 else X
    E = eng.experts_upload_folds(Xu, y, fold_of, K, n_e)
    d = X.shape[1]
    kernels = [mk(d).setHyperparameters(theta_of(mk, d, s)) for s in range(len(sets))]
    vals, grads = eng.bcm_nll_folds(sets, kernels)
    for k in sorted(set(sets)):
        tr = fold_of != k
        assert ref.experts_upload_grouped(Xu[tr], y[tr], n_e) == E[k]
        for s in [s for s in range(len(sets)) if sets[s] == k]:
            v0, g0 = ref.bcm_nll(kernels[s])
            assert bits(vals[s]) == bits(v0), (k, s, vals[s], v0)
            assert np.array_equal(bits(grads[s]), bits(g0)), (k, s)
    return vals, grads


# ---------------- 1. fold slots against single-set uploads, bit for bit -------------------------------------------------
CASES = [  # (kernel, K, N, d, n_e, f32)
    ("ard", 2, 1003, 3, 60, False),
    ("rbf", 3, 1501, 2, 100, True),
    ("two_term", 10, 1203, 4, 40, False),
    ("eye_only", 3, 613, 2, 50, False),
    ("ard", 10, 2500, 5, 100, True),
]


@pytest.mark.parametrize("kind,K,N,d,n_e,f32", CASES)
def test_fold_slots_match_single_set_bitwise(engs, kind, K, N, d, n_e, f32):
    eng, ref = engs
    X, y = data(N, d, seed=K * 1000 + N)
    fold_of = kfold_assignment(N, K, seed=K + d)
    mk = KERNELS[kind][0]
    check_slots(eng, ref, X, y, fold_of, K, n_e, mk, list(range(K)), f32)
    # a subset, a permutation, and repeated sets at distinct theta
    check_slots(eng, ref, X, y, fold_of, K, n_e, mk, [K - 1, 0, K - 1, 1 % K, 0], f32)


def test_fold_slots_ragged_sets(engs):
    eng, ref = engs
    X, y = data(997, 3, seed=3)
    fold_of = kfold_assignment(997, 3, seed=11)
    for k in range(3):
        n_k = int(np.sum(fold_of != k))
        assert n_k % int(np.floor(n_k / 70 + 0.5)) != 0
    check_slots(eng, ref, X, y, fold_of, 3, 70, KERNELS["ard"][0], [0, 1, 2])


def test_fold_slots_shared_memory_variant():
    """SGP_BCM_IMPL is read once per process: the shared-memory kernel runs in a subprocess."""
    code = ("import numpy as np, sys; sys.path.insert(0, %r); sys.path.insert(0, %r)\n"
            "import test_gpu_cross_validation as t, spark_gp_b200 as sg\n"
            "a, b = sg.ProjectedProcessEngine(0), sg.ProjectedProcessEngine(0)\n"
            "X, y = t.data(1203, 3, 5)\n"
            "f = t.kfold_assignment(1203, 4, 9)\n"
            "t.check_slots(a, b, X, y, f, 4, 90, t.KERNELS['ard'][0], [0, 1, 2, 3, 2])\n"
            "assert a.last_bcm_path() == 0\n"
            "print('smem ok')\n" % (ROOT, os.path.join(ROOT, "tests")))
    env = dict(os.environ, SGP_BCM_IMPL="smem")
    r = subprocess.run([sys.executable, "-c", code], env=env, capture_output=True, text=True, timeout=300)
    assert r.returncode == 0 and "smem ok" in r.stdout, r.stdout + r.stderr


def test_fold_slots_large_experts_lu(engs):
    eng, ref = engs
    X, y = data(1600, 3, seed=8)
    fold_of = kfold_assignment(1600, 3, seed=8)
    check_slots(eng, ref, X, y, fold_of, 3, 400, KERNELS["ard"][0], [0, 1, 2, 1])
    assert eng.last_bcm_path() == 1


def test_fold_slots_one_set_breaks_down(engs):
    """A near-duplicate point (1e-9 apart) without an Eye term: the on-chip Cholesky breaks down on the one set whose
    expert holds both copies, while LU still factors it.  Only that slot runs LU, in the same call; the other slots keep
    the on-chip bits."""
    eng, ref = engs
    N, d, K, n_e = 300, 2, 3, 40
    X, y = data(N, d, seed=21)
    fold_of = (np.arange(N) % K).astype(np.int32)
    rank = lambda k: np.cumsum(fold_of != k) - 1          # training rank of each point in set k
    E = [int(np.floor(np.sum(fold_of != k) / n_e + 0.5)) for k in range(K)]
    # point 0 (fold 0) and a point j of fold 1 in the same expert of set 2 only
    j = next(j for j in range(1, N, K) if rank(2)[j] % E[2] == 0)
    X[j], y[j] = X[0] + 1e-9, y[0]
    mk = lambda d: 1.0 * sg.RBFKernel(1.0)
    eng.experts_upload_folds(X, y, fold_of, K, n_e)
    kernels = [mk(d) for _ in range(K)]
    vals, grads = eng.bcm_nll_folds(list(range(K)), kernels)
    assert eng.last_bcm_path() == 1
    for k in range(K):
        tr = fold_of != k
        ref.experts_upload_grouped(X[tr], y[tr], n_e)
        v0, g0 = ref.bcm_nll(kernels[k])
        assert ref.last_bcm_path() == (1 if k == 2 else 0), k
        assert bits(vals[k]) == bits(v0), k
        assert np.array_equal(bits(grads[k]), bits(g0)), k


def test_fold_slots_subset_below_the_upload_largest_expert(engs):
    """The shared-memory kernel (two non-Eye terms) on a call that lists only sets whose largest expert is smaller than
    the upload's largest: the call plans and lays out shared memory for the listed sets."""
    eng, ref = engs
    N, d, K, n_e = 1203, 4, 10, 40
    X, y = data(N, d, seed=K * 1000 + N)
    fold_of = kfold_assignment(N, K, seed=K + d)
    n_k = np.array([np.sum(fold_of != k) for k in range(K)])
    E_k = np.floor(n_k / n_e + 0.5).astype(int)
    nmax = -(-n_k // E_k)
    small = [k for k in range(K) if nmax[k] < nmax.max()]
    assert small and len(small) < K
    check_slots(eng, ref, X, y, fold_of, K, n_e, KERNELS["two_term"][0], small + small[:1])


def test_fold_slots_cross_variant_boundary(engs):
    """Sets whose largest experts fall in different 16-row blocks of the register kernel's shapes: the call plans on the
    largest, the single-set calls on their own.  The padded shapes add exact zeros, so the bits still agree."""
    eng, ref = engs
    N, K = 260, 2
    X, y = data(N, 2, seed=31)
    fold_of = np.zeros(N, dtype=np.int32)
    fold_of[:70] = 1                          # set 0 (without fold 0): 70 points, set 1: 190 points
    # n_e = 64: set 0 -> E = 1 expert of 70 points; set 1 -> E = 3 experts of <= 64 points (the 16-row block below)
    E = eng.experts_upload_folds(X, y, fold_of, K, 64)
    assert E.tolist() == [1, 3]
    check_slots(eng, ref, X, y, fold_of, K, 64, KERNELS["rbf"][0], [0, 1])


def test_fold_errors(engs):
    eng, _ = engs
    X, y = data(300, 2, seed=1)
    mk = KERNELS["rbf"][0]
    eng.experts_upload_grouped(X, y, 50)
    with pytest.raises(sg.TrainingVectorsNotInitializedException):
        eng.bcm_nll_folds([0], [mk(2)])
    with pytest.raises(ValueError):
        eng.experts_upload_folds(X, y, np.full(300, 2), 2, 50)         # fold index out of range
    with pytest.raises(ValueError):
        eng.experts_upload_folds(X, y, np.zeros(300), 1, 50)           # n_folds < 2
    f = np.zeros(300, dtype=np.int32)
    f[:290] = 1                                                         # set 1 has 10 points: E_1 == 0 at n_e = 50
    with pytest.raises(ValueError, match="numberOfExperts"):
        eng.experts_upload_folds(X, y, f, 2, 50)
    eng.experts_upload_folds(X, y, kfold_assignment(300, 3, 0), 3, 50)
    with pytest.raises(ValueError):
        eng.bcm_nll_folds([3], [mk(2)])
    with pytest.raises(ValueError):
        eng.bcm_nll_folds([0, 1], [mk(2), KERNELS["ard"][0](2)])       # structures differ


# ---------------- 2. fixed theta against the oracle --------------------------------------------------------------------
def test_fold_slots_vs_oracle(engs):
    eng, _ = engs
    N, d, K, n_e = 700, 3, 4, 50
    X, y = data(N, d, seed=77)
    fold_of = kfold_assignment(N, K, seed=5)
    for kind in ("ard", "two_term"):
        mk, mo = KERNELS[kind]
        theta = theta_of(mk, d, 3)
        eng.experts_upload_folds(X, y, fold_of, K, n_e)
        vals, grads = eng.bcm_nll_folds(list(range(K)), [mk(d).setHyperparameters(theta)] * K)
        for k in range(K):
            v0, g0 = fold_bcm_objective(X, y, fold_of, k, lambda: mo(d), n_e, theta)
            assert abs(vals[k] - v0) <= TOL_VAL * abs(v0), (kind, k)
            assert np.max(np.abs(grads[k] - g0)) <= TOL_GRAD * np.max(np.abs(g0)), (kind, k)


def airfoil():
    z = np.load(os.path.join(GOLD, "airfoil_cv_case.npz"))
    return z


def airfoil_gp():
    return (sg.GaussianProcessRegression().setDatasetSizeForExpert(100).setActiveSetSize(1000).setSigma2(1e-4)
            .setKernel(lambda: 1 * sg.ARDRBFKernel(5) + sg.const(1.0) * sg.EyeKernel()))


def test_airfoil_fixture_vs_oracle(engs):
    eng, _ = engs
    z = airfoil()
    gp = airfoil_gp()
    K = len(z["bcm_nll"])
    eng.experts_upload_folds(z["X"], z["y"], z["fold_of"], K, int(z["n_e"]))
    vals, grads = eng.bcm_nll_folds(list(range(K)), [gp.getKernel().setHyperparameters(z["theta"])] * K)
    for k in range(K):
        assert abs(vals[k] - z["bcm_nll"][k]) <= TOL_VAL * abs(z["bcm_nll"][k]), k
        g0 = z["bcm_grad"][k]
        assert np.max(np.abs(grads[k] - g0)) <= TOL_GRAD * np.max(np.abs(g0)), k
    assert np.array_equal(kfold_assignment(len(z["X"]), K, int(z["seed"])), z["fold_of"])


# ---------------- 3. the estimator against independent fits ------------------------------------------------------------
def synthetics():
    rng = np.random.default_rng(13)
    X = np.linspace(0, 1, 2000)[:, None]
    y = np.sin(X[:, 0]) + np.sqrt(0.01) * rng.standard_normal(2000)
    return X, y


def synthetics_gp():
    return (sg.GaussianProcessRegression()
            .setKernel(lambda: 1 * sg.RBFKernel(0.1, 1e-6, 10) + sg.WhiteNoiseKernel(0.5, 0, 1))
            .setDatasetSizeForExpert(100).setActiveSetProvider(KMeansActiveSetProvider(on_gpu=True))
            .setActiveSetSize(100).setSeed(13).setSigma2(1e-3))


def check_against_independent(cv, model, gp, maps, X, y, K, seed):
    fold_of = kfold_assignment(len(X), K, seed)
    ev = sg.RegressionEvaluator()
    indep_avg = []
    for p, m in enumerate(maps):
        metrics = []
        for k in range(K):
            tr, va = fold_of != k, fold_of == k
            g = gp.copy(m)
            fm = g.fit(X[tr], y[tr])
            pred = fm.predict(X[va])
            got = cv.last_folds[p, k]
            assert np.array_equal(bits(got["theta"]), bits(fm.hyperparameters)), (p, k)
            assert np.array_equal(bits(got["magicVector"]), bits(fm.rawPredictor.magicVector)), (p, k)
            assert np.array_equal(bits(got["prediction"]), bits(pred)), (p, k)
            metrics.append(ev.evaluate(y[va], pred))
            del fm
        indep_avg.append(sum(metrics) / K)
    assert model.avgMetrics == indep_avg
    best = gp.copy(maps[model.bestIndex]).fit(X, y)
    assert np.array_equal(bits(model.bestModel.hyperparameters), bits(best.hyperparameters))
    assert np.array_equal(bits(model.bestModel.predict(X[:50])), bits(best.predict(X[:50])))
    return indep_avg


def test_synthetics_cross_validation_equals_independent_fits():
    X, y = synthetics()
    gp = synthetics_gp().setMaxIter(15)
    maps = sg.ParamGridBuilder().addGrid("sigma2", [1e-3, 1e-2]).build()
    cv = sg.CrossValidator().setEstimator(gp).setEvaluator(sg.RegressionEvaluator()).setEstimatorParamMaps(maps) \
        .setNumFolds(3).setSeed(5)
    model = cv.fit(X, y)
    check_against_independent(cv, model, gp, maps, X, y, 3, 5)
    (group,) = model.last_objective["groups"]
    evaluations = sum(s["evaluations"] for s in group["slots"])
    assert group["rounds"] < evaluations
    assert group["launches"] < 2 * evaluations          # the independent fits make 2 launches per evaluation


def test_airfoil_cross_validation_equals_independent_fits():
    z = airfoil()
    X, y = z["X"], z["y"]
    gp = airfoil_gp().setMaxIter(5)
    cv = sg.CrossValidator().setEstimator(gp).setNumFolds(3).setSeed(2)
    model = cv.fit(X, y)
    check_against_independent(cv, model, gp, [{}], X, y, 3, 2)


# ---------------- 4. the reference's gates -----------------------------------------------------------------------------
def test_airfoil_reference_start_is_trapped():
    """Airfoil.scala's configuration as written misses the reference's 2.1, and this pins why.  From theta0 = (1, 1, ..., 1)
    the labels (~125 dB, uncentred) make the objective of a fold ~2e6, and while the scale is still small (about 2.3
    after three iterations, against the labels' mean square of ~15 600) the steepest way down is to flatten the kernel:
    within three L-BFGS-B iterations the ARD betas reach their lower bound 0.  There d/d beta_k = -2 beta_k (x_k - z_k)^2 k
    is 0 identically, so a beta that reaches 0 stays there, whatever the tolerance.  On this split at least four of the
    five betas end at 0 in every fold: the fold models are (nearly) constant, and the RMSE is about the labels' spread
    (6.9)."""
    z = airfoil()
    cv = sg.CrossValidator().setEstimator(airfoil_gp()).setNumFolds(10)
    model = cv.fit(z["X"], z["y"], folds=z["fold_of"])
    zeros = [int(np.sum(cv.last_folds[0, k]["theta"][1:] == 0.0)) for k in range(10)]
    assert min(zeros) >= 4, zeros
    assert 6.0 < model.avgMetrics[0] < 7.5


AIRFOIL_SCALE0 = 15600.0     # about the labels' mean square (15 620): the prior variance that explains their offset


def test_airfoil_gate():
    """Airfoil.scala:18-24: 10-fold cross-validated RMSE below 2.1, with the reference's configuration except where the
    optimisation starts and stops: the trainable scale starts at AIRFOIL_SCALE0 instead of 1 (see the test above), and tol
    is 1e-12, since at 1e-6 the relative-reduction test stops most folds before the scale has moved from its start."""
    z = airfoil()
    gp = airfoil_gp().setKernel(lambda: AIRFOIL_SCALE0 * sg.ARDRBFKernel(5) + sg.const(1.0) * sg.EyeKernel()).setTol(1e-12)
    model = sg.CrossValidator().setEstimator(gp).setNumFolds(10).fit(z["X"], z["y"], folds=z["fold_of"])
    print("airfoil 10-fold CV RMSE %.4f; iterations per fold %s" % (
        model.avgMetrics[0], [s["iterations"] for s in model.last_objective["groups"][0]["slots"]]))
    assert model.avgMetrics[0] < 2.1


def test_synthetics_gate():
    """Synthetics.scala:25-33: 10-fold cross-validated RMSE below 0.11."""
    X, y = synthetics()
    model = sg.CrossValidator().setEstimator(synthetics_gp()).setNumFolds(10).setSeed(13).fit(X, y)
    print("synthetics 10-fold CV RMSE %.4f" % model.avgMetrics[0])
    assert model.avgMetrics[0] < 0.11
