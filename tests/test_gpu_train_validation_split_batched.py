"""TrainValidationSplit over regression in one BCM launch per round, and the binary evaluator on the binary classifier (run
on an H100: `pytest -m gpu`).

Every regression param map's theta, magic vector and validation predictions must equal, bit for bit, those of the
independent `estimator.copy(map).fit(X[train], y[train])`, for host and CUDA-tensor inputs, and so must the metrics,
the best index and the refitted best model.  Over the binary classifier, a BinaryClassificationEvaluator must score
each map's validation latent mean f exactly as the oracle evaluator scores the independent fit's.
"""
import os

import numpy as np
import pytest

import spark_gp_b200 as sg
from oracle import binary_metrics as obm
from oracle import train_validation_split as otvs
from spark_gp_b200.tuning import best_index

pytestmark = pytest.mark.gpu

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")


def bits(a):
    return np.ascontiguousarray(a, dtype=np.float64).view(np.int64)


def reg_data(n=900, d=3, seed=17):
    rng = np.random.default_rng(seed)
    X = rng.random((n, d))
    y = np.sin(3 * X.sum(1)) + 0.05 * rng.standard_normal(n)
    return X, y


def check_regression(est, maps, X, y, seed=2, device=False):
    """The batched selection against the independent fits, bit for bit; returns the model's record."""
    Xin, yin = X, y
    if device:
        import torch
        Xin, yin = torch.as_tensor(X, device="cuda:0"), torch.as_tensor(y, device="cuda:0")
    tvs = (sg.TrainValidationSplit().setEstimator(est).setEvaluator(sg.RegressionEvaluator("rmse"))
           .setEstimatorParamMaps(maps).setSeed(seed))
    model = tvs.fit(Xin, yin)
    mask = otvs.train_mask(len(X), 0.75, seed)
    rec = model.last_objective
    assert len(rec["maps"]) == len(maps)
    for p, m in enumerate(maps):
        e = est.copy(m)
        ind = e.fit(X[mask], y[mask])
        assert np.array_equal(bits(rec["maps"][p]["theta"]), bits(ind.hyperparameters)), p
        assert np.array_equal(bits(rec["maps"][p]["magicVector"]), bits(ind.rawPredictor.magicVector)), p
        assert np.array_equal(bits(tvs.last_predictions[p]), bits(ind.predict(X[~mask]))), p
        assert model.validationMetrics[p] == sg.RegressionEvaluator("rmse").evaluate(y[~mask], ind.predict(X[~mask]))
        if e._maxIter > 0:
            for key in ("evaluations", "iterations", "value", "n_experts"):
                assert rec["maps"][p][key] == e.last_objective[key], (p, key)
        del ind
    assert model.bestIndex == best_index(model.validationMetrics, False)
    best = est.copy(maps[model.bestIndex]).fit(X, y)
    assert np.array_equal(bits(model.bestModel.rawPredictor.magicVector), bits(best.rawPredictor.magicVector))
    for g in rec["groups"]:                               # one slots call (3 launches on chip) per round
        assert g["launches"] == 3 * g["rounds"]
        assert g["rounds"] == max(rec["maps"][p]["evaluations"] for p in g["maps"])
    return rec


@pytest.mark.parametrize("device", [False, True])
def test_grid_sigma2_by_active_set_size(device):
    X, y = reg_data()
    gp = (sg.GaussianProcessRegression().setKernel(lambda: 1.0 * sg.ARDRBFKernel(np.ones(3)))
          .setDatasetSizeForExpert(50).setActiveSetSize(40).setMaxIter(10))
    maps = sg.ParamGridBuilder().addGrid("sigma2", [1e-3, 1e-2]).addGrid("activeSetSize", [30, 40]).build()
    rec = check_regression(gp, maps, X, y, device=device)
    (group,) = rec["groups"]
    assert group["maps"] == [0, 1, 2, 3]


@pytest.mark.parametrize("device", [False, True])
def test_grid_split_by_dataset_size_for_expert(device):
    X, y = reg_data(1100, 2, seed=5)
    gp = (sg.GaussianProcessRegression().setKernel(lambda: 1.0 * sg.RBFKernel(0.5))
          .setActiveSetSize(50).setMaxIter(15))
    maps = sg.ParamGridBuilder().addGrid("sigma2", [1e-3, 1e-1]).addGrid("datasetSizeForExpert", [40, 70]).build()
    rec = check_regression(gp, maps, X, y, seed=4, device=device)
    assert sorted(g["maps"] for g in rec["groups"]) == [[0, 1], [2, 3]]


def test_max_iter_zero():
    X, y = reg_data(700, 3, seed=9)
    gp = (sg.GaussianProcessRegression().setKernel(lambda: 1.0 * sg.ARDRBFKernel(np.ones(3)))
          .setDatasetSizeForExpert(50).setActiveSetSize(40).setMaxIter(0))
    maps = sg.ParamGridBuilder().addGrid("sigma2", [1e-3, 1e-2, 1e-1]).build()
    maps.append({"sigma2": 1e-2, "maxIter": 5})             # one optimised map beside them
    rec = check_regression(gp, maps, X, y, seed=6)
    assert [g["maps"] for g in rec["groups"]] == [[3]]
    assert all(rec["maps"][p]["evaluations"] == 0 for p in range(3))


# ---------------- the binary evaluator over the binary classifier on the mnist68 rows ------------------------------------
def mnist68():
    c = np.load(os.path.join(GOLD, "mnist68_case.npz"))
    X = (c["pixels"].astype(np.float64) - c["mean"]) / c["std"]
    return X, c["y01"]


@pytest.mark.parametrize("metric", ["areaUnderROC", "areaUnderPR"])
def test_tvs_binary_mnist68_area_under_curve(metric):
    X, y = mnist68()
    gp = (sg.GaussianProcessClassifier().setDatasetSizeForExpert(100).setActiveSetSize(100)
          .setKernel(lambda: sg.RBFKernel(10.0)).setTol(1e-3).setMaxIter(5))
    maps = sg.ParamGridBuilder().addGrid("kernel", [(lambda s: lambda: sg.RBFKernel(s))(s) for s in (8.0, 12.0)]).build()
    ev = sg.BinaryClassificationEvaluator(metric)
    tvs = (sg.TrainValidationSplit().setEstimator(gp).setEvaluator(ev).setEstimatorParamMaps(maps)
           .setTrainRatio(0.8).setSeed(3))
    model = tvs.fit(X, y)
    mask = otvs.train_mask(len(X), 0.8, 3)
    for p, m in enumerate(maps):
        ind = gp.copy(m).fit(X[mask], y[mask])
        f = ind.predictRaw(X[~mask])[:, 1]
        assert model.validationMetrics[p] == obm.binary_metric(metric, y[~mask], f), p
        assert np.array_equal(bits(tvs.last_predictions[p]), bits(ind.predict(X[~mask]))), p
        del ind
    assert model.bestIndex == best_index(model.validationMetrics, True)
    assert min(model.validationMetrics) > 0.95
