"""Host side of the binary evaluator and of the batched regression TrainValidationSplit (no GPU):
`BinaryClassificationEvaluator` against the restatement of Spark's BinaryClassificationMetrics in
oracle/binary_metrics.py and against hand-computed curves, the selectors' type refusals, and the grouping of regression
param maps into one upload and one lock-step optimisation per `slot_group_key`."""
import numpy as np
import pytest

import spark_gp_b200 as sg
from oracle import binary_metrics as obm
from spark_gp_b200 import tuning
from spark_gp_b200.regression import GaussianProcessRegression
from spark_gp_b200.tuning import binary_metric, slot_group_key

METRICS = ("areaUnderROC", "areaUnderPR")


def both(name, y, s, num_bins=1000):
    """The evaluator's value, checked equal (==) to the oracle's."""
    got = sg.BinaryClassificationEvaluator(name, num_bins).evaluate(y, s)
    assert got == obm.binary_metric(name, y, s, num_bins), (name, num_bins)
    return got


# ---------------- hand-computed curves ---------------------------------------------------------------------------------
def test_small_case_by_hand():
    # points 0.9 (+), 0.8 (-), 0.7 (+), 0.1 (-): (TP, FP) = (1, 0), (1, 1), (2, 1), (2, 2) of P = N = 2
    # ROC (0,0) (0,.5) (.5,.5) (.5,1) (1,1) (1,1): 0.25 + 0.5;  PR (0,1) (.5,1) (.5,.5) (1,2/3) (1,.5): 0.5 + 7/24
    y, s = [1, 0, 1, 0], [0.9, 0.8, 0.7, 0.1]
    assert both("areaUnderROC", y, s) == pytest.approx(0.75, abs=1e-15)
    assert both("areaUnderPR", y, s) == pytest.approx(19 / 24, abs=1e-15)
    assert obm.naive_auc(y, s) == 0.75


def test_ties_collapse_into_one_point():
    # points 0.5 (1+, 1-), 0.2 (1+, 1-): ROC (0,0) (.5,.5) (1,1) (1,1) = 0.5;  PR (0,.5) (.5,.5) (1,.5) = 0.5
    y, s = [1, 0, 1, 0], [0.5, 0.5, 0.2, 0.2]
    assert both("areaUnderROC", y, s) == 0.5
    assert both("areaUnderPR", y, s) == 0.5
    # a tie between a positive and a negative counts half, as in the Mann-Whitney statistic
    y, s = [1, 0, 1, 0, 0], [0.9, 0.9, 0.4, 0.3, 0.1]
    assert both("areaUnderROC", y, s) == pytest.approx(obm.naive_auc(y, s), abs=1e-15)


def test_all_equal_scores():
    # one point (2+, 3-): ROC (0,0) (1,1) (1,1) = 0.5;  PR (0,.4) (1,.4) = 0.4
    y, s = [1, 1, 0, 0, 0], [3.0] * 5
    assert both("areaUnderROC", y, s) == 0.5
    assert both("areaUnderPR", y, s) == pytest.approx(0.4, abs=1e-15)


def test_a_single_class():
    """Spark's recall is 0 without positives and its false positive rate 0 without negatives, so only positives give
    ROC (0,0) (0,r)... (1,1): area 1, and PR at precision 1 throughout: area 1; only negatives give recall 0 and
    precision 0 everywhere: both areas 0."""
    s = [3.0, 2.0, 2.0, 1.0]
    assert both("areaUnderROC", [1, 1, 1, 1], s) == 1.0
    assert both("areaUnderPR", [1, 1, 1, 1], s) == 1.0
    assert both("areaUnderROC", [0, 0, 0, 0], s) == 0.0
    assert both("areaUnderPR", [0, 0, 0, 0], s) == 0.0


def test_num_bins_by_hand():
    # scores 6..1, labels + - + + - -.  No binning: AUC = 7/9.
    y, s = [1, 0, 1, 1, 0, 0], [6.0, 5.0, 4.0, 3.0, 2.0, 1.0]
    assert both("areaUnderROC", y, s, 0) == pytest.approx(7 / 9, abs=1e-15)
    # numBins 4: 6 // 4 = 1 < 2, no binning
    assert both("areaUnderROC", y, s, 4) == both("areaUnderROC", y, s, 0)
    # numBins 3: runs of 2 -> (1+,1-) (2+,0-) (0+,2-): ROC (0,0) (1/3,1/3) (1/3,1) (1,1) (1,1) = 1/18 + 2/3
    assert both("areaUnderROC", y, s, 3) == pytest.approx(13 / 18, abs=1e-15)
    # numBins 2: runs of 3 -> (2+,1-) (1+,2-): ROC (0,0) (1/3,2/3) (1,1) (1,1) = 1/9 + 5/9
    assert both("areaUnderROC", y, s, 2) == pytest.approx(2 / 3, abs=1e-15)
    # PR at numBins 2: precision 2/3 then 1/2, recall 2/3 then 1: (0,2/3) (2/3,2/3) (1,1/2)
    assert both("areaUnderPR", y, s, 2) == pytest.approx(4 / 9 + (1 / 3) * (7 / 6) / 2, abs=1e-15)


@pytest.mark.parametrize("n,distinct,num_bins", [(5000, 5000, 1000), (5000, 5000, 2500), (5000, 5000, 3000),
                                                 (4003, 4003, 1000), (3001, 700, 100), (3001, 700, 2000),
                                                 (200, 7, 3), (1000, 1000, 0)])
@pytest.mark.parametrize("name", METRICS)
def test_against_the_oracle(name, n, distinct, num_bins):
    """numBins below and above the distinct-score count, with and without a short last run, and ties."""
    rng = np.random.default_rng(n + distinct + num_bins)
    y = (rng.random(n) < 0.4).astype(np.float64)
    levels = rng.standard_normal(distinct)
    s = levels[rng.integers(0, distinct, n)] + 0.8 * y
    got = both(name, y, s, num_bins)
    if name == "areaUnderROC" and (num_bins == 0 or len(np.unique(s)) // num_bins < 2):
        assert got == pytest.approx(obm.naive_auc(y, s), abs=1e-12)
    assert 0.0 <= got <= 1.0


def test_evaluator_params_and_refusals():
    ev = sg.BinaryClassificationEvaluator()
    assert ev.getMetricName() == "areaUnderROC" and ev.getNumBins() == 1000 and ev.isLargerBetter()
    assert sg.BinaryClassificationEvaluator("areaUnderPR").isLargerBetter()
    with pytest.raises(ValueError, match="areaUnderROC, areaUnderPR"):
        ev.setMetricName("accuracy")
    for bad in (1, -1, 2.5):
        with pytest.raises(ValueError, match="numBins"):
            ev.setNumBins(bad)
    assert ev.setNumBins(0).getNumBins() == 0
    with pytest.raises(ValueError):
        ev.evaluate([], [])
    with pytest.raises(ValueError):
        ev.evaluate([0, 1], [0.5])
    for labels in ([0, 2], [0.5, 1], [-1, 1]):
        with pytest.raises(ValueError, match="0 or 1"):
            ev.evaluate(labels, [0.1, 0.2])
        with pytest.raises(ValueError, match="0 or 1"):
            obm.binary_metric("areaUnderROC", labels, [0.1, 0.2])
    with pytest.raises(ValueError, match="NaN"):
        ev.evaluate([0, 1], [0.1, np.nan])
    with pytest.raises(ValueError):
        binary_metric("areaUnderROC", [], [])


# ---------------- the selectors' type refusals -------------------------------------------------------------------------
def test_selectors_refuse_the_binary_evaluator_off_the_binary_classifier():
    X, y = np.random.default_rng(0).random((40, 2)), np.arange(40) % 2
    ev = sg.BinaryClassificationEvaluator()
    for est in (sg.GaussianProcessRegression(), sg.OneVsRest().setClassifier(sg.GaussianProcessClassifier())):
        tvs = sg.TrainValidationSplit().setEstimator(est).setEvaluator(ev)
        with pytest.raises(TypeError, match="BinaryClassificationEvaluator scores the binary"):
            tvs.fit(X, y)
    sg.TrainValidationSplit().setEstimator(sg.GaussianProcessClassifier()).setEvaluator(ev)       # accepted
    with pytest.raises(TypeError, match="evaluator must be"):
        sg.CrossValidator().setEvaluator(ev)


# ---------------- regression maps: one upload and one lock-step optimisation per group ----------------------------------
class FakeEngine:
    """Stands in for the device: records the uploads and the slot calls; the objective of each slot is
    sum (theta - 0.7)^2, minimised inside the kernels' bounds."""
    log = []

    @classmethod
    def acquire(cls, device):
        return cls()

    def __init__(self):
        self.launches = 0

    def release(self):
        pass

    def launch_count(self):
        return self.launches

    def experts_upload_grouped(self, X, y, n_e):
        FakeEngine.log.append(("upload", len(X), n_e))
        return int(np.floor(len(X) / n_e + 0.5))

    def bcm_nll_slots(self, kernels):
        self.launches += 3
        FakeEngine.log.append(("slots", len(kernels)))
        t = np.array([k.getHyperparameters() for k in kernels])
        return ((t - 0.7) ** 2).sum(axis=1), 2.0 * (t - 0.7)


class FakeModel:
    def __init__(self, theta):
        self.theta = theta
        self.rawPredictor = type("Raw", (), dict(magicVector=np.asarray(theta)))()

    def predict(self, X):
        return np.full(len(X), self.theta[0])


def test_tvs_groups_regression_maps_by_slot_group_key(monkeypatch):
    FakeEngine.log = []
    monkeypatch.setattr(tuning, "ProjectedProcessEngine", FakeEngine)
    monkeypatch.setattr(GaussianProcessRegression, "_produce_model", lambda self, X, y, theta: FakeModel(theta))
    gp = sg.GaussianProcessRegression().setKernel(lambda: 1.0 * sg.RBFKernel(2.0)).setMaxIter(20)
    maps = (sg.ParamGridBuilder().addGrid("sigma2", [1e-3, 1e-2, 1e-1]).addGrid("datasetSizeForExpert", [20, 40])
            .build())
    maps.append({"datasetSizeForExpert": 20, "maxIter": 0})
    ests = [gp.copy(m) for m in maps]
    keys = [slot_group_key(e) for e in ests]
    # sigma2 is no part of the key; datasetSizeForExpert alone, and maxIter, split the maps
    assert len(set(keys)) == 3 and keys[0] == keys[1] == keys[2] and keys[3] == keys[4] == keys[5]
    X, y = np.random.default_rng(1).random((200, 2)), np.zeros(200)
    train = np.arange(200) % 4 != 0
    preds, record = tuning.TrainValidationSplit._fit_regression(ests, X, y, train)
    uploads = [e for e in FakeEngine.log if e[0] == "upload"]
    assert uploads == [("upload", 150, 20), ("upload", 150, 40)]          # the maxIter = 0 group uploads nothing
    groups = record["groups"]
    assert [g["maps"] for g in groups] == [[0, 1, 2], [3, 4, 5]]
    for g in groups:
        assert g["launches"] == 3 * g["rounds"]                              # one slots call per round
        assert g["rounds"] == max(record["maps"][p]["evaluations"] for p in g["maps"])
    assert max(e[1] for e in FakeEngine.log if e[0] == "slots") == 3
    assert len(record["maps"]) == len(maps)
    assert record["maps"][6]["evaluations"] == record["maps"][6]["iterations"] == 0
    assert [record["maps"][p]["n_experts"] for p in range(6)] == [8, 8, 8, 4, 4, 4]
    for p in range(6):
        assert preds[p] == pytest.approx(np.full(50, 0.7), abs=1e-5)
        assert np.array_equal(record["maps"][p]["magicVector"], record["maps"][p]["theta"])
    theta0 = ests[6].getKernel().getHyperparameters()                        # the kernel's own theta
    assert np.any(theta0 != 0.7) and np.array_equal(preds[6], np.full(50, theta0[0]))
