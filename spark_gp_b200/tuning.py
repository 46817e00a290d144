"""Model selection for the regression estimator: Spark 3.1's `ParamGridBuilder`, `RegressionEvaluator` and
`CrossValidator`, as the reference's own examples use them (regression/examples/GPExample.scala:17-27, Airfoil.scala:18-24,
Synthetics.scala:25-33: 10-fold cross-validation of the RMSE).

Spark's ml/tuning and ml/evaluation are not part of the reference project; they are restated here from Spark 3.1's
documented behaviour:
  - ParamGridBuilder.build() is the Cartesian product of the added grids; the first param added varies fastest.  An empty
    builder gives one empty param map.  Adding a param again replaces its values.
  - RegressionEvaluator computes rmse (default), mse, r2, mae or var from the labels y and predictions p:
    mse = sum (y - p)^2 / n, rmse = sqrt(mse), mae = sum |y - p| / n, r2 = 1 - sum (y - p)^2 / sum (y - mean y)^2,
    var = sum (p - mean y)^2 / n; r2 and var are larger-is-better.  No weightCol, no throughOrigin.
  - CrossValidator fits the estimator with every param map on every fold's training split (the rows outside the fold, in
    their order), evaluates it on the fold, averages each map's metric over the folds (sum in fold order / numFolds),
    takes the first best map and refits it on all rows.  numFolds defaults to 3.
Deviations: Spark's MLUtils.kFold draws a fold for each row per partition, so its split depends on the partitioning and
is not reproducible here.  The default split draws from the counter-based generator the K-means provider uses (stream
200): fold(i) = floor(u(seed, 200, i) * numFolds); `fit(X, y, folds=...)` takes a given split, as Spark 3.1's foldCol.
An empty validation fold raises ValueError, where Spark would evaluate an empty frame.

All (map, fold) slots that share datasetSizeForExpert, the kernel's structure and hyper-parameter layout, the bounds,
maxIter and tol are optimised together: the training sets of every fold are uploaded once
(`sgp_experts_upload_folds`), and each round of their L-BFGS-B runs is one `sgp_bcm_nll_folds` launch over experts x
slots.  Each slot's objective values equal the independent fit's bit for bit, so every fold model, prediction and metric
is the one `estimator.copy(map).fit(X[train], y[train])` gives."""
from __future__ import annotations

import numpy as np

from . import _native as N
from .engine import ProjectedProcessEngine
from .hyperopt import lbfgsb_bounds, lbfgsb_lockstep
from .regression import GaussianProcessRegression
from .utils import kfold_assignment


class ParamGridBuilder:
    """Spark's ParamGridBuilder over the estimator's params (GaussianProcessParams.PARAMS)."""

    def __init__(self):
        self._grid = {}

    def addGrid(self, name: str, values):
        if name not in GaussianProcessRegression.PARAMS:
            raise ValueError("unknown param %s; the params are %s" % (name, ", ".join(GaussianProcessRegression.PARAMS)))
        self._grid[name] = list(values)
        return self

    def build(self):
        maps = [{}]
        for name, values in self._grid.items():
            maps = [dict(m, **{name: v}) for v in values for m in maps]
        return maps


def regression_metric(name: str, y, p) -> float:
    """Spark's RegressionMetrics for one metric name, unweighted."""
    y = np.asarray(y, dtype=np.float64)
    p = np.asarray(p, dtype=np.float64)
    n = len(y)
    err = y - p
    if name in ("mse", "rmse"):
        mse = float(np.sum(err * err) / n)
        return float(np.sqrt(mse)) if name == "rmse" else mse
    if name == "mae":
        return float(np.sum(np.abs(err)) / n)
    ybar = np.sum(y) / n
    if name == "r2":
        return float(1.0 - np.sum(err * err) / np.sum((y - ybar) ** 2))
    if name == "var":
        return float(np.sum((p - ybar) ** 2) / n)
    raise ValueError("metricName must be one of rmse, mse, r2, mae, var, not %r" % (name,))


class RegressionEvaluator:
    METRICS = ("rmse", "mse", "r2", "mae", "var")

    def __init__(self, metricName: str = "rmse"):
        self.setMetricName(metricName)

    def setMetricName(self, value: str):
        if value not in self.METRICS:
            raise ValueError("metricName must be one of %s, not %r" % (", ".join(self.METRICS), value))
        self._metric = value
        return self

    def getMetricName(self) -> str:
        return self._metric

    def isLargerBetter(self) -> bool:
        return self._metric in ("r2", "var")

    def evaluate(self, y, prediction) -> float:
        y = np.asarray(y, dtype=np.float64)
        if len(y) == 0 or np.shape(prediction) != y.shape:
            raise ValueError("evaluate: labels and predictions must be non-empty vectors of one length")
        return regression_metric(self._metric, y, prediction)


def best_index(metrics, larger_is_better: bool) -> int:
    """The first maximal (larger is better) or minimal metric, as Scala's maxBy / minBy."""
    m = np.asarray(metrics, dtype=np.float64)
    return int(np.argmax(m) if larger_is_better else np.argmin(m))


def slot_group_key(est: GaussianProcessRegression):
    """Slots with equal keys run in one lock-step optimisation over one fold upload: the expert grouping, the flattened
    kernel structure and hyper-parameter layout (one batched launch needs them equal), and what L-BFGS-B shares."""
    k = est.getKernel()
    terms = tuple(t["type"] for t in k.flatten())
    layout = tuple((h["kind"], h.get("term", 0), h.get("dim", 0)) for h in k.hyper_descriptors())
    return (est._datasetSizeForExpert, terms, layout, tuple(lbfgsb_bounds(k)), est._maxIter, est._tol)


def group_slots(estimators, n_folds: int):
    """{key: [(map index, fold), ...]} over every (map, fold) slot, in map-major order."""
    groups = {}
    for p, est in enumerate(estimators):
        key = slot_group_key(est)
        groups.setdefault(key, []).extend((p, k) for k in range(n_folds))
    return groups


class CrossValidatorModel:
    """Spark's CrossValidatorModel: the best map refitted on every row, and each map's metric averaged over the folds."""

    def __init__(self, bestModel, avgMetrics, bestIndex, last_objective):
        self.bestModel = bestModel
        self.avgMetrics = list(avgMetrics)
        self.bestIndex = bestIndex
        self.last_objective = last_objective

    def predict(self, features):
        return self.bestModel.predict(features)

    transform = predict


class CrossValidator:
    def __init__(self):
        self._estimator = None
        self._evaluator = RegressionEvaluator()
        self._maps = None
        self._num_folds = 3
        self._seed = 0
        self.last_folds = None            # {(map, fold): theta, magicVector and validation prediction of the fold model}

    def setEstimator(self, value):
        if not isinstance(value, GaussianProcessRegression):
            raise TypeError("CrossValidator: the estimator must be a GaussianProcessRegression, not %s"
                            % type(value).__name__)
        self._estimator = value
        return self

    def setEvaluator(self, value):
        if not isinstance(value, RegressionEvaluator):
            raise TypeError("CrossValidator: the evaluator must be a RegressionEvaluator")
        self._evaluator = value
        return self

    def setEstimatorParamMaps(self, value):
        maps = [dict(m) for m in value]
        if not maps:
            raise ValueError("CrossValidator: at least one param map")
        self._maps = maps
        return self

    def setNumFolds(self, value: int):
        if int(value) < 2:
            raise ValueError("CrossValidator: numFolds must be >= 2")
        self._num_folds = int(value)
        return self

    def setSeed(self, value: int):
        self._seed = int(value)
        return self

    def getNumFolds(self) -> int:
        return self._num_folds

    def fit(self, X, y, folds=None) -> CrossValidatorModel:
        """folds: the fold of every row (integers in [0, numFolds)); default: the seeded split of the module docstring."""
        est = self._estimator
        if est is None:
            raise TypeError("CrossValidator: setEstimator(GaussianProcessRegression) first")
        X = np.asarray(X)
        y = np.asarray(y, dtype=np.float64)
        if X.ndim != 2 or len(y) != len(X):
            raise ValueError("CrossValidator: X must be n x d and y n labels")
        K = self._num_folds
        if folds is None:
            fold_of = kfold_assignment(len(X), K, self._seed)
        else:
            f = np.asarray(folds)
            if f.shape != (len(X),) or not np.all((f == np.floor(f)) & (f >= 0) & (f < K)):
                raise ValueError("CrossValidator: folds must hold one integer in [0, numFolds) per row")
            fold_of = f.astype(np.int32)
        sizes = np.bincount(fold_of, minlength=K)
        if np.any(sizes == 0):
            raise ValueError("CrossValidator: fold %d has no rows to validate on" % int(np.argmin(sizes)))
        maps = self._maps or [{}]
        ests = [est.copy(m) for m in maps]
        thetas, objective = self._optimise(ests, X, y, fold_of, K)
        metrics = np.empty((len(maps), K))
        folds_out = {}
        for p, e in enumerate(ests):
            for k in range(K):
                train, val = fold_of != k, fold_of == k
                model = e._produce_model(X[train], y[train], thetas[p][k])
                pred = model.predict(X[val])
                folds_out[p, k] = dict(theta=thetas[p][k], magicVector=model.rawPredictor.magicVector, prediction=pred)
                metrics[p, k] = self._evaluator.evaluate(y[val], pred)
                del model                         # its context goes back to the pool before the next slot
        avg = [sum(metrics[p, k] for k in range(K)) / K for p in range(len(maps))]
        best = best_index(avg, self._evaluator.isLargerBetter())
        self.last_folds = folds_out
        objective["fold_metrics"] = metrics
        return CrossValidatorModel(est.copy(maps[best]).fit(X, y), avg, best, objective)

    @staticmethod
    def _optimise(ests, X, y, fold_of, K):
        """Optimal hyper-parameters of every (map, fold) slot (thetas[p][k]), and what the optimisation took."""
        x0s = [e.getKernel().getHyperparameters() for e in ests]
        thetas = [[np.asarray(x0s[p], dtype=np.float64) for _ in range(K)] for p in range(len(ests))]
        groups = []
        for key, slots in group_slots(ests, K).items():
            e0 = ests[slots[0][0]]
            if e0._maxIter <= 0:
                continue                          # GPR.fit takes the kernel's own hyper-parameters
            eng = ProjectedProcessEngine.acquire(e0._device)
            try:
                eng.experts_upload_folds(X, y, fold_of, K, e0._datasetSizeForExpert)
                launches0 = eng.launch_count()
                kernel_at = lambda p, t: ests[p].getKernel().setHyperparameters(np.asarray(t, dtype=np.float64))

                def evaluate(batch):
                    vals, grads = eng.bcm_nll_folds([slots[i][1] for i, _ in batch],
                                                    [kernel_at(slots[i][0], t) for i, t in batch])
                    return [(float(v), g) for v, g in zip(vals, grads)]

                k0 = e0.getKernel()
                results, rounds = lbfgsb_lockstep(evaluate, [x0s[p] for p, _ in slots], lbfgsb_bounds(k0), e0._maxIter,
                                                  e0._tol)
                groups.append(dict(
                    slots=[dict(map=p, fold=k, value=float(res.fun), evaluations=ev, iterations=int(res.nit))
                           for (p, k), (res, ev) in zip(slots, results)],
                    rounds=rounds, launches=eng.launch_count() - launches0))
            finally:
                eng.set_precision(N.SGP_PREC_AUTO)
                eng.release()
            for (p, k), (res, _) in zip(slots, results):
                thetas[p][k] = np.asarray(res.x, dtype=np.float64)
        return thetas, dict(groups=groups)
