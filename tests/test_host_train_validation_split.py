"""Host side of TrainValidationSplit (no GPU): the split, the multiclass metrics, the best-map rule, the argument errors,
`OneVsRest.copy`, and the numbering and grouping of the (map, class) mode slots."""
import numpy as np
import pytest

import spark_gp_b200 as sg
from oracle import train_validation_split as otvs
from oracle.kmeans import u
from spark_gp_b200.tuning import best_index, multiclass_metric, tvs_slot_groups
from spark_gp_b200.utils import train_validation_assignment


# ---------------- the split --------------------------------------------------------------------------------------------
@pytest.mark.parametrize("seed,ratio", [(0, 0.75), (7, 0.8), (123456789, 0.5), (-5, 0.1)])
def test_split_matches_the_generator_and_the_oracle(seed, ratio):
    n = 600
    got = train_validation_assignment(n, ratio, seed)
    assert got.dtype == bool
    assert np.array_equal(got, u(seed, 201, np.arange(n)) < ratio)
    assert np.array_equal(got, otvs.train_mask(n, ratio, seed))
    assert abs(got.mean() - ratio) < 0.1


def test_split_stream_is_not_the_kfold_stream():
    a = train_validation_assignment(1000, 0.5, 3)
    b = np.floor(u(3, 200, np.arange(1000)) * 2) == 0
    assert not np.array_equal(a, b)


# ---------------- the metrics ------------------------------------------------------------------------------------------
CRAFTED = {
    "random": (np.random.default_rng(1).integers(0, 4, 97).astype(float),
               np.random.default_rng(2).integers(0, 4, 97).astype(float)),
    "true_class_never_predicted": (np.array([0, 0, 1, 1, 2, 2, 2], float), np.array([0, 1, 1, 1, 0, 1, 0], float)),
    "predicted_class_absent_from_truth": (np.array([0, 0, 1, 1, 1], float), np.array([0, 3, 1, 3, 1], float)),
    "single_class": (np.array([1, 1, 1, 1], float), np.array([1, 0, 1, 1], float)),
    "single_class_never_predicted": (np.array([2, 2, 2], float), np.array([0, 1, 0], float)),
    "perfect": (np.array([0, 1, 2, 1], float), np.array([0, 1, 2, 1], float)),
}


@pytest.mark.parametrize("case", sorted(CRAFTED))
@pytest.mark.parametrize("name", otvs.METRICS)
def test_metrics_match_the_oracle(case, name):
    y, p = CRAFTED[case]
    ev = sg.MulticlassClassificationEvaluator(name)
    assert ev.isLargerBetter()
    assert ev.getMetricName() == name
    assert ev.evaluate(y, p) == otvs.metric(name, y, p)
    assert multiclass_metric(name, y, p) == otvs.metric(name, y, p)


def test_metric_values_by_hand():
    y, p = CRAFTED["true_class_never_predicted"]
    # label 0: tp 1, fp 2, n 2 -> p 1/3, r 1/2;  label 1: tp 2, fp 2, n 2 -> p 1/2, r 1;  label 2: tp 0, n 3 -> 0, 0
    assert sg.MulticlassClassificationEvaluator("accuracy").evaluate(y, p) == pytest.approx(3 / 7)
    assert sg.MulticlassClassificationEvaluator("weightedRecall").evaluate(y, p) == pytest.approx((1 + 2) / 7)
    assert sg.MulticlassClassificationEvaluator("weightedPrecision").evaluate(y, p) == pytest.approx((2 / 3 + 1) / 7)
    f1 = (2 * (2 * (1 / 3) * 0.5 / (1 / 3 + 0.5)) + 2 * (2 * 0.5 * 1 / 1.5)) / 7
    assert sg.MulticlassClassificationEvaluator().evaluate(y, p) == pytest.approx(f1)
    assert sg.MulticlassClassificationEvaluator().getMetricName() == "f1"       # Spark's default
    y, p = CRAFTED["single_class_never_predicted"]
    for name in otvs.METRICS:
        assert sg.MulticlassClassificationEvaluator(name).evaluate(y, p) == 0.0


def test_metric_errors():
    for bad in ("auc", "logLoss", "precisionByLabel", "rmse"):
        with pytest.raises(ValueError, match="f1, accuracy, weightedPrecision, weightedRecall"):
            sg.MulticlassClassificationEvaluator(bad)
    ev = sg.MulticlassClassificationEvaluator("accuracy")
    with pytest.raises(ValueError):
        ev.setMetricName("areaUnderROC")
    with pytest.raises(ValueError):
        ev.evaluate([], [])
    with pytest.raises(ValueError):
        ev.evaluate([0.0, 1.0], [0.0])


def test_best_map_is_the_first_best():
    for m in ([0.5, 0.9, 0.9, 0.1], [0.3, 0.3], [0.1, 0.2, 0.3], [0.7, 0.2, 0.7]):
        assert best_index(m, True) == otvs.best_index(m, True)
        assert best_index(m, False) == otvs.best_index(m, False)
    assert best_index([0.5, 0.9, 0.9], True) == 1


# ---------------- argument errors (raised before any GPU work) ----------------------------------------------------------
def test_train_ratio_bounds():
    tvs = sg.TrainValidationSplit()
    assert tvs.getTrainRatio() == 0.75
    for bad in (0.0, 1.0, -0.1, 1.5):
        with pytest.raises(ValueError, match="trainRatio"):
            tvs.setTrainRatio(bad)
    assert tvs.setTrainRatio(0.8).getTrainRatio() == 0.8


def test_estimator_and_evaluator_types():
    tvs = sg.TrainValidationSplit()
    for est in (sg.GaussianProcessRegression(), sg.GaussianProcessClassifier(),
                sg.OneVsRest().setClassifier(sg.GaussianProcessClassifier())):
        assert tvs.setEstimator(est) is tvs
    for bad in (None, object(), sg.CrossValidator(), sg.RBFKernel()):
        with pytest.raises(TypeError):
            tvs.setEstimator(bad)
    for ev in (sg.RegressionEvaluator(), sg.MulticlassClassificationEvaluator()):
        assert tvs.setEvaluator(ev) is tvs
    for bad in (None, "accuracy", sg.ParamGridBuilder()):
        with pytest.raises(TypeError):
            tvs.setEvaluator(bad)
    with pytest.raises(ValueError):
        tvs.setEstimatorParamMaps([])


def test_fit_argument_errors():
    X, y = np.random.default_rng(0).standard_normal((40, 2)), np.zeros(40)
    with pytest.raises(TypeError):                                        # no estimator
        sg.TrainValidationSplit().setEvaluator(sg.RegressionEvaluator()).fit(X, y)
    with pytest.raises(ValueError, match="setEvaluator"):                 # no evaluator, no default
        sg.TrainValidationSplit().setEstimator(sg.GaussianProcessClassifier()).fit(X, y)
    tvs = sg.TrainValidationSplit().setEstimator(sg.GaussianProcessClassifier()) \
        .setEvaluator(sg.MulticlassClassificationEvaluator("accuracy"))
    with pytest.raises(ValueError, match="training side"):
        tvs.fit(X, y, train=np.zeros(40, dtype=bool))
    with pytest.raises(ValueError, match="validation side"):
        tvs.fit(X, y, train=np.ones(40, dtype=bool))
    with pytest.raises(ValueError):
        tvs.fit(X, y, train=np.ones(39, dtype=bool))
    with pytest.raises(ValueError):
        tvs.fit(X, y, train=np.full(40, 2))
    with pytest.raises(ValueError):
        tvs.fit(X, y[:-1])
    with pytest.raises(ValueError, match="side of the split is empty"):  # the seeded split of one row leaves a side empty
        tvs.fit(X[:1], y[:1])


# ---------------- OneVsRest.copy ---------------------------------------------------------------------------------------
def test_one_vs_rest_copy():
    gp = sg.GaussianProcessClassifier().setDatasetSizeForExpert(20).setTol(1e-3)
    ovr = sg.OneVsRest().setClassifier(gp)
    c = ovr.copy({"sigma2": 0.5, "maxIter": 3})
    assert isinstance(c, sg.OneVsRest) and c is not ovr
    assert c.getClassifier() is not gp
    assert c.getClassifier()._sigma2 == 0.5 and c.getClassifier()._maxIter == 3
    assert c.getClassifier()._datasetSizeForExpert == 20 and c.getClassifier()._tol == 1e-3
    assert gp._sigma2 == 1e-3 and gp._maxIter == 100                     # the original is untouched
    plain = ovr.copy()
    assert plain.getClassifier() is not gp and plain.getClassifier()._sigma2 == gp._sigma2
    assert sg.OneVsRest().copy().getClassifier() is None
    with pytest.raises(ValueError, match="unknown param"):
        ovr.copy({"numClasses": 3})


# ---------------- mode slots -------------------------------------------------------------------------------------------
def test_mode_slot_numbering_and_grouping():
    gp = sg.GaussianProcessClassifier().setKernel(lambda: sg.RBFKernel(1.0))
    maps = [{"kernel": lambda: sg.RBFKernel(2.0)}, {"sigma2": 1e-2}, {"datasetSizeForExpert": 50},
            {"kernel": lambda: 1.0 * sg.ARDRBFKernel(np.ones(3))}, {"tol": 1e-3}, {"activeSetSize": 20}]
    gps = [gp.copy(m) for m in maps]
    for C in (1, 3):
        groups = list(tvs_slot_groups(gps, C).values())
        # a different sigma (a kernel value), sigma2 or active-set size shares a launch; a different expert size, kernel
        # structure or tol does not
        assert [sorted({p for p, _, _ in g}) for g in groups] == [[0, 1, 5], [2], [3], [4]]
        slots = [s for g in groups for s in g]
        assert sorted(m for _, _, m in slots) == list(range(len(maps) * C))
        for p, c, m in slots:
            assert m == p * C + c and 0 <= c < C
        assert groups[0] == [(p, c, p * C + c) for p in (0, 1, 5) for c in range(C)]   # map-major


def test_slot_grouping_of_one_vs_rest_maps_uses_the_classifier():
    ovr = sg.OneVsRest().setClassifier(sg.GaussianProcessClassifier())
    ests = [ovr.copy(m) for m in ({"sigma2": 1e-3}, {"sigma2": 1e-1}, {"maxIter": 5})]
    groups = list(tvs_slot_groups([e.getClassifier() for e in ests], 3).values())
    assert [sorted({p for p, _, _ in g}) for g in groups] == [[0, 1], [2]]
