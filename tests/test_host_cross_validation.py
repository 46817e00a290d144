"""Host side of cross-validation (no GPU): the fold split, the grid, the metrics, best-index selection, the slot grouping,
`copy`, the lock-step optimiser driving slots that share a fold, and the slot optimiser every estimator uses."""
import threading

import numpy as np
import pytest

import spark_gp_b200 as sg
from oracle import cross_validation as ocv
from oracle.kmeans import u
from spark_gp_b200.hyperopt import lbfgsb, lbfgsb_lockstep, optimise_slots
from spark_gp_b200.tuning import best_index, group_slots, regression_metric
from spark_gp_b200.utils import kfold_assignment


@pytest.mark.parametrize("seed,K", [(0, 2), (7, 10), (123456789, 3), (-5, 7)])
def test_fold_assignment_matches_the_generator(seed, K):
    n = 500
    got = kfold_assignment(n, K, seed)
    assert got.dtype == np.int32
    assert np.array_equal(got, np.floor(u(seed, 200, np.arange(n)) * K).astype(np.int32))
    assert np.array_equal(got, ocv.fold_assignment(n, K, seed))


def test_grid_order():
    b = sg.ParamGridBuilder().addGrid("sigma2", [1, 2]).addGrid("maxIter", [3, 4, 5]).addGrid("seed", [9])
    maps = b.build()
    assert maps == ocv.param_grid([("sigma2", [1, 2]), ("maxIter", [3, 4, 5]), ("seed", [9])])
    assert [m["sigma2"] for m in maps] == [1, 2, 1, 2, 1, 2]             # the first param varies fastest
    assert sg.ParamGridBuilder().build() == [{}]
    assert sg.ParamGridBuilder().addGrid("tol", [1]).addGrid("tol", [2, 3]).build() == [{"tol": 2}, {"tol": 3}]
    with pytest.raises(ValueError):
        sg.ParamGridBuilder().addGrid("lengthScale", [1])


@pytest.mark.parametrize("name", ["rmse", "mse", "r2", "mae", "var"])
def test_metrics_match_the_oracle(name):
    rng = np.random.default_rng(3)
    y, p = rng.standard_normal(57), rng.standard_normal(57)
    got = sg.RegressionEvaluator(name).evaluate(y, p)
    assert got == pytest.approx(ocv.metric(name, y, p), rel=1e-13)
    assert sg.RegressionEvaluator(name).isLargerBetter() == ocv.larger_is_better(name)
    assert regression_metric(name, y, y + 0.0) == pytest.approx(ocv.metric(name, y, y), abs=1e-15)


def test_best_index_takes_the_first_of_ties():
    for name in ("rmse", "r2"):
        larger = sg.RegressionEvaluator(name).isLargerBetter()
        for m in ([1.0, 0.5, 0.5, 2.0], [2.0, 2.0, 1.0], [0.5, 0.5], [3.0, 1.0, 3.0, 1.0]):
            assert best_index(m, larger) == ocv.best_index(m, name)
    assert best_index([1.0, 0.5, 0.5], False) == 1
    assert best_index([1.0, 2.0, 2.0], True) == 1
    with pytest.raises(ValueError):
        sg.RegressionEvaluator("auc")


def test_slot_grouping():
    gp = sg.GaussianProcessRegression().setKernel(lambda: 1.0 * sg.RBFKernel(1.0))
    ests = [gp.copy(m) for m in [{"sigma2": 1e-3}, {"sigma2": 1e-2}, {"datasetSizeForExpert": 50},
                                 {"kernel": lambda: 1.0 * sg.ARDRBFKernel(np.ones(3))}, {"maxIter": 7},
                                 {"activeSetSize": 20}, {"seed": 4}]]
    groups = list(group_slots(ests, 3).values())
    # sigma2, activeSetSize and seed leave the objective's structure alone: those maps share one group
    assert groups[0] == [(p, k) for p in (0, 1, 5, 6) for k in range(3)]
    assert [g[0][0] for g in groups[1:]] == [2, 3, 4]
    assert all(len(g) == 3 for g in groups[1:])


def test_copy():
    gp = sg.GaussianProcessRegression(device=0, shard_points=1234).setSigma2(0.5).setMaxIter(9)
    c = gp.copy({"sigma2": 0.25, "datasetSizeForExpert": 40, "seed": 3})
    assert (c._sigma2, c._datasetSizeForExpert, c._seed, c._maxIter, c._shard_points) == (0.25, 40, 3, 9, 1234)
    assert gp._sigma2 == 0.5 and gp._datasetSizeForExpert == 100 and gp._seed == 0
    assert isinstance(c, sg.GaussianProcessRegression)
    assert gp.copy()._sigma2 == 0.5
    with pytest.raises(ValueError):
        gp.copy({"sigma": 1.0})


def test_cross_validator_arguments():
    cv = sg.CrossValidator()
    assert cv.getNumFolds() == 3
    with pytest.raises(TypeError):
        cv.setEstimator(sg.GaussianProcessClassifier())
    with pytest.raises(ValueError):
        cv.setNumFolds(1)
    cv.setEstimator(sg.GaussianProcessRegression()).setNumFolds(4)
    X = np.zeros((10, 1))
    with pytest.raises(ValueError, match="no rows"):
        cv.fit(X, np.zeros(10), folds=np.array([0, 1, 2] * 3 + [0]))
    with pytest.raises(ValueError):
        cv.fit(X, np.zeros(10), folds=np.full(10, 4))


def _quadratic(c, theta):
    """A smooth bounded test objective with a slot-dependent minimum."""
    t = np.asarray(theta)
    centre = np.linspace(0.3, 1.7, len(t)) * (1.0 + 0.1 * c)
    return float(np.sum((t - centre) ** 2 * (1.0 + np.arange(len(t))))), 2.0 * (t - centre) * (1.0 + np.arange(len(t)))


def test_lockstep_slots_sharing_a_fold_follow_their_independent_runs():
    """Slots (map, fold) where several maps share one fold: each slot gets exactly the x, iteration and evaluation
    counts of an independent lbfgsb."""
    slots = [(p, k) for p in range(3) for k in range(2)]
    x0s = [np.full(3, 0.5 + 0.2 * p) for p, _ in slots]
    bounds = [(0.1, None), (0.1, 5.0), (0.0, None)]
    calls = []

    def evaluate(batch):
        calls.append(len(batch))
        return [_quadratic(slots[i][0] + 3 * slots[i][1], t) for i, t in batch]

    results, rounds = lbfgsb_lockstep(evaluate, x0s, bounds, 30, 1e-9)
    for i, (p, k) in enumerate(slots):
        ref, ev = lbfgsb(lambda t: _quadratic(p + 3 * k, t), x0s[i], bounds, 30, 1e-9)
        res, ev_l = results[i]
        assert np.array_equal(res.x, ref.x)
        assert res.nit == ref.nit and ev_l == ev
    assert rounds == len(calls) and rounds < sum(ev for _, ev in results)


@pytest.mark.parametrize("n_slots", [1, 4])
def test_optimise_slots_equals_independent_lbfgsb_runs(n_slots):
    """One slot is `lbfgsb` itself on the calling thread (no thread is started); several run in lock-step.  Either way
    every slot's theta, value, evaluations and iterations are those of its independent `lbfgsb`."""
    x0s = [np.full(3, 0.5 + 0.2 * i) for i in range(n_slots)]
    bounds = [(0.1, None), (0.1, 5.0), (0.0, None)]
    threads_alive, calls = threading.active_count(), []

    def evaluate(batch):
        calls.append(threading.active_count())
        return [_quadratic(i, t) for i, t in batch]

    thetas, records, rounds = optimise_slots(evaluate, x0s, bounds, 30, 1e-9)
    evaluations = []
    for i in range(n_slots):
        ref, ev = lbfgsb(lambda t: _quadratic(i, t), x0s[i], bounds, 30, 1e-9)
        assert thetas[i].dtype == np.float64 and np.array_equal(thetas[i], ref.x)
        assert records[i] == dict(value=float(ref.fun), evaluations=ev, iterations=int(ref.nit))
        evaluations.append(ev)
    assert rounds == len(calls) == max(evaluations)
    if n_slots == 1:
        assert all(n == threads_alive for n in calls)
    else:
        assert all(n > threads_alive for n in calls) and rounds < sum(evaluations)


@pytest.mark.parametrize("n_slots", [1, 3])
@pytest.mark.parametrize("max_iter", [0, -1])
def test_optimise_slots_without_iterations_evaluates_nothing(n_slots, max_iter):
    def evaluate(batch):
        raise AssertionError("evaluated at maxIter %d" % max_iter)

    x0s = [np.arange(3) + i for i in range(n_slots)]
    thetas, records, rounds = optimise_slots(evaluate, x0s, [(None, None)] * 3, max_iter, 1e-9)
    assert records is None and rounds == 0
    for theta, x0 in zip(thetas, x0s):
        assert theta.dtype == np.float64 and np.array_equal(theta, x0)
