"""Model selection: Spark 3.1's `ParamGridBuilder`, `RegressionEvaluator`, `MulticlassClassificationEvaluator`,
`BinaryClassificationEvaluator`, `CrossValidator` (regression estimator and one-vs-rest) and `TrainValidationSplit` (any estimator), as the reference's own
examples use them (regression/examples/GPExample.scala:17-27, Airfoil.scala:18-24, Synthetics.scala:25-33: 10-fold
cross-validation of the RMSE; classification/examples/Iris.scala: 10-fold cross-validation of one-vs-rest scored by
accuracy; classification/examples/MNIST.scala:34-40: a train/validation split scored by accuracy).

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
is the one `estimator.copy(map).fit(X[train], y[train])` gives.
Over one-vs-rest, fold k has C_k = max(y[train]) + 1 classes, as an independent `OneVsRest.fit(X[train], y[train])`
counts them.  The (map p, fold k, class c) slots are grouped by `slot_group_key` of the wrapped classifier; a group uploads
the fold sets once, and each round of its L-BFGS-B runs is one `sgp_laplace_nll_fold_slots_any_size` call, every slot
with its own mode slot (`fold_class_slot_groups`), plus one call at every slot's optimum (GPCls:60).  Each fold's class
models are then produced on its training rows, and its validation prediction is the first argmax over the C_k raw
columns.  The evaluator is a RegressionEvaluator (the default) or a MulticlassClassificationEvaluator.  The binary
classifier is refused; the fold-slot entry already serves it (class 1 over 0/1 labels, one mode slot per (map, fold)).

TrainValidationSplit (Spark 3.1): fit every param map on the training rows (in row order), evaluate each fitted model on
the validation rows (validationMetrics, in map order), take the first best map and refit it on all rows.  trainRatio
defaults to 0.75 and lies strictly in (0, 1); there is no default evaluator.  Deviation: Spark's randomSplit depends on the
partitioning; here row i trains iff u(seed, 201, i) < trainRatio (the K-means generator, stream 201), and
`fit(X, y, train=mask)` takes a given split.  An empty training or validation side raises ValueError.
Over the binary classifier and one-vs-rest, the maps are grouped by `slot_group_key` of the classifier; a group's
training rows are uploaded once, and every (map p, class c) is one slot with mode slot p * C + c (binary: C = 1, class 1)
in `sgp_laplace_nll_slots_any_size`, so each round of the slots' L-BFGS-B runs is one launch.  Each slot's values and
modes equal the independent fit's bit for bit, so every validation prediction is that of
`estimator.copy(map).fit(X[train], y[train])`.  Over regression, the maps are grouped by `slot_group_key` too; a
group's training rows are uploaded once (`sgp_experts_upload_grouped`), and each round of its maps' L-BFGS-B runs is one
`sgp_bcm_nll_slots` launch, each map's values equal to the independent fit's bit for bit; each map's model is then
produced on the training rows at its theta.
A BinaryClassificationEvaluator (Spark 3.1's, over rawPrediction(1) = f; see `binary_metric`) is accepted over the
binary classifier only, and scores each map's validation latent mean f; over any other estimator `fit` raises TypeError.
CrossValidator does not take it, as it does not take the binary classifier.

Both selectors take X (and y) as CUDA tensors on the estimator's device as well: the fold upload reads them in place
(`sgp_experts_upload_folds_device`), the training and validation rows are gathered on the device and predicted there, and
only the validation labels and predictions go to the host, for the evaluator.  `folds=` and `train=` stay host arrays.
The results are the host fit's, bit for bit.

Over a process group (the estimator, or one-vs-rest's classifier, built with `process_group=`), every rank passes its
own shard, host array or CUDA tensor, uneven or empty, and a given `folds=` / `train=` is its slice of the split.  The
seeded splits draw at the global row index (`kfold_assignment(..., offset)`), so they are the plain splits of the
concatenation.  The drivers below are the plain ones, handed a `distributed.Selection` in place of `_Local`: every
training set's rows move to their experts' owners (`sgp_experts_upload_fold_sets_device`, or the strided upload for the
one training set of a split), the slot groups run in lock step on the group's context over the all-reducing batched
objectives, each fold or map model is produced there with the set's active set, each rank predicts its own validation
rows and one gather gives every rank every rank's labels and predictions in rank order.  So the metrics, bestIndex and
the refitted map (the group fit of the estimator) are the same on every rank, and at one rank they are the plain
selector's bit for bit (DESIGN.md section 5)."""
from __future__ import annotations

import contextlib

import numpy as np

from . import _native as N
from .classification import GaussianProcessClassifier, OneVsRest, assert_labels_are_01, binary_prediction, laplace_fit, \
    one_vs_rest_labels, one_vs_rest_prediction
from .engine import ProjectedProcessEngine, host_copy, is_cuda_tensor, take_rows
from .hyperopt import expert_count, fit_data, fit_slots, lbfgsb_bounds, produce, slot_modes, slot_objective
from .regression import GaussianProcessRegression
from .utils import kfold_assignment, train_validation_assignment


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


class _Evaluator:
    """What the evaluators share: the metric name, one of METRICS, and `evaluate`, which checks its arguments and hands
    them to `_metric_of(name, y, prediction)`."""
    METRICS = ()

    def setMetricName(self, value: str):
        if value not in self.METRICS:
            raise ValueError("metricName must be one of %s, not %r" % (", ".join(self.METRICS), value))
        self._metric = value
        return self

    def getMetricName(self) -> str:
        return self._metric

    def evaluate(self, y, prediction) -> float:
        y = np.asarray(y, dtype=np.float64)
        if len(y) == 0 or np.shape(prediction) != y.shape:
            raise ValueError("evaluate: labels and predictions must be non-empty vectors of one length")
        return self._metric_of(self._metric, y, prediction)


class RegressionEvaluator(_Evaluator):
    METRICS = ("rmse", "mse", "r2", "mae", "var")
    _metric_of = staticmethod(regression_metric)

    def __init__(self, metricName: str = "rmse"):
        self.setMetricName(metricName)

    def isLargerBetter(self) -> bool:
        return self._metric in ("r2", "var")


def multiclass_metric(name: str, y, p) -> float:
    """Spark 3.1's MulticlassMetrics for one metric name, unweighted: per true label l (sorted), n_l rows, tp_l hits and
    fp_l false predictions of l; precision_l = tp_l / (tp_l + fp_l) (0 if never predicted), recall_l = tp_l / n_l,
    f1_l = 2 p r / (p + r) (0 if p + r = 0); the weighted metrics sum v_l * n_l / n over the labels in order."""
    y = np.asarray(y, dtype=np.float64)
    p = np.asarray(p, dtype=np.float64)
    n = len(y)
    if name == "accuracy":
        return float(np.count_nonzero(y == p)) / n
    if name not in MulticlassClassificationEvaluator.METRICS:
        raise ValueError("metricName must be one of %s, not %r" % (", ".join(MulticlassClassificationEvaluator.METRICS),
                                                                  name))
    total = 0.0
    for label in np.unique(y):
        truth, hit = y == label, p == label
        nl = int(np.count_nonzero(truth))
        tp = int(np.count_nonzero(hit & truth))
        fp = int(np.count_nonzero(hit)) - tp
        precision = tp / (tp + fp) if tp + fp > 0 else 0.0
        recall = tp / nl
        value = {"weightedPrecision": precision, "weightedRecall": recall,
                 "f1": 2.0 * precision * recall / (precision + recall) if precision + recall > 0.0 else 0.0}[name]
        total += value * nl / n
    return total


class MulticlassClassificationEvaluator(_Evaluator):
    """Spark's MulticlassClassificationEvaluator over (label, prediction): f1 (default), accuracy, weightedPrecision,
    weightedRecall, all larger-is-better."""
    METRICS = ("f1", "accuracy", "weightedPrecision", "weightedRecall")
    _metric_of = staticmethod(multiclass_metric)

    def __init__(self, metricName: str = "f1"):
        self.setMetricName(metricName)

    def isLargerBetter(self) -> bool:
        return True


def binary_metric(name: str, y, scores, num_bins: int = 1000) -> float:
    """Spark 3.1's BinaryClassificationMetrics(scoreAndLabels, numBins) for one metric name, unweighted, on one partition.
    The distinct scores in descending order are the curve's points, each with its counts of labels 1 and 0.  With
    numBins > 0 and g = (distinct scores) // numBins >= 2, every g consecutive points are merged into one at the run's
    last (smallest) score, and the points left over into a last one; Spark merges within each partition, so its curve
    depends on the partitioning (this is its one-partition curve).  Cumulative counts give each point's recall TP / P
    (0 when P = 0), false positive rate FP / N (0 when N = 0) and precision TP / (TP + FP).  areaUnderROC is the
    trapezoidal area under (0, 0), (FPR, recall)..., (1, 1); areaUnderPR under (0, first precision),
    (recall, precision)...; the trapezoids are summed in curve order."""
    if name not in BinaryClassificationEvaluator.METRICS:
        raise ValueError("metricName must be one of %s, not %r" % (", ".join(BinaryClassificationEvaluator.METRICS),
                                                                  name))
    y = np.asarray(y, dtype=np.float64)
    s = np.asarray(scores, dtype=np.float64)
    if len(y) == 0 or s.shape != y.shape:
        raise ValueError("BinaryClassificationEvaluator: labels and scores must be non-empty vectors of one length")
    if not np.all((y == 0.0) | (y == 1.0)):
        raise ValueError("BinaryClassificationEvaluator: labels must be 0 or 1")
    if np.isnan(s).any():
        raise ValueError("BinaryClassificationEvaluator: a score is NaN")
    distinct, inv = np.unique(s, return_inverse=True)
    n = len(distinct)
    pos = np.bincount(inv[y == 1.0], minlength=n)[::-1]          # descending scores
    neg = np.bincount(inv, minlength=n)[::-1] - pos
    g = n // num_bins if num_bins > 0 else 0
    ends = np.arange(n) if g < 2 else np.unique(np.append(np.arange(g - 1, n, g), n - 1))
    tp, fp = np.cumsum(pos)[ends], np.cumsum(neg)[ends]
    P, N_ = tp[-1], fp[-1]
    recall = tp / P if P > 0 else np.zeros(len(ends))
    if name == "areaUnderROC":
        fpr = fp / N_ if N_ > 0 else np.zeros(len(ends))
        x, v = np.concatenate([[0.0], fpr, [1.0]]), np.concatenate([[0.0], recall, [1.0]])
    else:
        precision = tp / (tp + fp)                                  # every point holds a row: tp + fp > 0
        x, v = np.concatenate([[0.0], recall]), np.concatenate([precision[:1], precision])
    return float(np.cumsum((x[1:] - x[:-1]) * (v[1:] + v[:-1]) / 2.0)[-1])


class BinaryClassificationEvaluator(_Evaluator):
    """Spark's BinaryClassificationEvaluator over (label, rawPrediction(1)): areaUnderROC (default) or areaUnderPR,
    larger-is-better, with numBins (default 1000; 0 keeps every distinct score) as in `binary_metric`.  `evaluate(y,
    scores)` takes 0/1 labels and the raw score; for GaussianProcessClassifier that is the latent mean f."""
    METRICS = ("areaUnderROC", "areaUnderPR")

    def __init__(self, metricName: str = "areaUnderROC", numBins: int = 1000):
        self.setMetricName(metricName)
        self.setNumBins(numBins)

    def setNumBins(self, value: int):
        if int(value) != value or not (value == 0 or value > 1):
            raise ValueError("BinaryClassificationEvaluator: numBins must be 0 or an integer > 1")
        self._num_bins = int(value)
        return self

    def getNumBins(self) -> int:
        return self._num_bins

    def _metric_of(self, name, y, scores):
        return binary_metric(name, y, scores, self._num_bins)

    def isLargerBetter(self) -> bool:
        return True


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


def group_slots(estimators, n: int):
    """{slot_group_key: [(map index p, j), ...]} over every slot (p, j), j in [0, n), of one estimator per map, in
    map-major order; j is the fold of a cross-validation or the class of a train/validation split."""
    groups = {}
    for p, est in enumerate(estimators):
        groups.setdefault(slot_group_key(est), []).extend((p, j) for j in range(n))
    return groups


def fold_class_slot_groups(classifiers, n_classes):
    """`group_slots` over the (map p, fold k, class c) slots of a cross-validation over classifiers (one per map), fold k
    having n_classes[k] classes, each with the device mode slot it owns: {slot_group_key: [(p, k, c, mode slot), ...]}.
    Mode slot p * sum(n_classes) + (classes of the folds before k) + c.  The one place that numbers mode slots."""
    fc = [(k, c) for k, C in enumerate(n_classes) for c in range(C)]
    return {key: [(p, *fc[j], p * len(fc) + j) for p, j in slots]
            for key, slots in group_slots(classifiers, len(fc)).items()}


def tvs_slot_groups(classifiers, n_classes: int):
    """The (map p, class c) slots of a train/validation split over classifiers (one per map), each with the device mode
    slot it owns, p * n_classes + c: {slot_group_key: [(p, c, mode slot), ...]} (`fold_class_slot_groups` with one
    fold)."""
    return {key: [(p, c, m) for p, _, c, m in slots]
            for key, slots in fold_class_slot_groups(classifiers, [n_classes]).items()}


class _SelectedModel:
    """What the model selectors' models share: the best map refitted on every row predicts."""

    def __init__(self, bestModel, bestIndex, last_objective):
        self.bestModel = bestModel
        self.bestIndex = bestIndex
        self.last_objective = last_objective

    def predict(self, features):
        return self.bestModel.predict(features)

    transform = predict


class _Validator:
    """What the model selectors share: the param maps, the seed and the check of the data; NAME prefixes the errors."""
    NAME = ""

    def setEstimatorParamMaps(self, value):
        maps = [dict(m) for m in value]
        if not maps:
            raise ValueError("%s: at least one param map" % self.NAME)
        self._maps = maps
        return self

    def setSeed(self, value: int):
        self._seed = int(value)
        return self

    def _data(self, X, y, device: int, classifier: bool):
        """(X, y) as the estimator's fit reads them (`fit_data`)."""
        on_device = is_cuda_tensor(X)
        X, y = fit_data(X, y, device, self.NAME + ".fit", keep_float32=not classifier)
        if not on_device and (X.ndim != 2 or len(y) != len(X)):
            raise ValueError("%s: X must be n x d and y n labels" % self.NAME)
        return X, y


def _rows(X, mask):
    """The rows of X where the host bool mask is set, on X's side."""
    return take_rows(X, np.flatnonzero(mask))


def _host_predictions(p):
    """A model's predictions as the evaluator reads them (host float64)."""
    return np.asarray(host_copy(p), dtype=np.float64)


def _latent_mean(eng, X):
    """The latent mean of the model eng holds at the validation rows X, on X's side, as the evaluator reads it (host
    float64)."""
    if is_cuda_tensor(X):
        return _host_predictions(eng.predict_tensor(X, with_variance=False)[0])
    return eng.predict(X, with_variance=False)[0]


def _validate(est, Xt, yt, Xv, theta):
    """The validation predictions (host float64) and the magic vector of the regression estimator's model on the training
    rows at theta.  The model's context goes back to the pool on return, before the next slot's."""
    model = est._produce_model(Xt, yt, theta)
    return _host_predictions(model.predict(Xv)), model.rawPredictor.magicVector


@contextlib.contextmanager
def _pooled(device: int):
    """A context of the device's pool for the span of a `with`."""
    eng = ProjectedProcessEngine.acquire(device)
    try:
        yield eng
    finally:
        eng.release()


class _Local:
    """The plain selectors' side of the drivers below, on this process's rows: members[k] is the host bool mask of
    training set k (fold_of != k, or the training mask), the slot fits run on pooled contexts over the sets uploaded from
    every row, each fold model is the independent fit's, and the validation arrays are this process's.  Over a process
    group `distributed.Selection` takes its place, with the same methods."""

    def __init__(self, X, y, members, fold_of=None):
        self.X, self.y, self.members, self.fold_of = X, y, members, fold_of
        self.on_device = is_cuda_tensor(X)

    context = staticmethod(_pooled)

    @staticmethod
    def gather(v):
        return np.asarray(host_copy(v), dtype=np.float64)

    def set_classes(self, ovr: bool):
        """C_k of every training set: one-vs-rest's max(y[train]) + 1, as an independent OneVsRest.fit(X[train],
        y[train]) counts them (the labels checked first), or 1 for the binary classifier (its labels checked)."""
        if not ovr:
            assert_labels_are_01(self.y)
            return [1] * len(self.members)
        one_vs_rest_labels(self.y)
        return [one_vs_rest_labels(_rows(self.y, t))[1] for t in self.members]

    def upload_sets(self, eng, dataset_size_for_expert: int):
        """The fold upload of every training set.  Returns (rows, experts) per set."""
        rows = [int(np.count_nonzero(t)) for t in self.members]
        return rows, eng.experts_upload_folds(self.X, self.y, self.fold_of, len(self.members), dataset_size_for_expert)

    @staticmethod
    def upload_training(eng, dataset_size_for_expert: int, Xt, yt, laplace: bool = False):
        """The grouped upload of the one training set (Xt, yt).  Returns (rows, experts, experts)."""
        if laplace:
            expert_count(len(Xt), dataset_size_for_expert)
        n_experts = eng.experts_upload_grouped(Xt, yt, dataset_size_for_expert)
        return len(Xt), n_experts, n_experts

    @staticmethod
    def validate(est, k: int, Xt, yt, Xv, theta):
        return _validate(est, Xt, yt, Xv, theta)

    @staticmethod
    def fold_model(gp, eng, k: int, Xt, f, theta):
        return produce(gp, eng, Xt, f, theta)

    @staticmethod
    def latent_mean(eng, Xv):
        return _latent_mean(eng, Xv)


def _bcm_groups(ests, n: int, upload, entry, context=_pooled):
    """The lock-step BCM optimisation of each group of (map p, j) slots, j in [0, n) (`group_slots`), on one context of
    its own (`context(device)`, a context manager; a pooled one by default): upload(eng, datasetSizeForExpert) uploads the
    training rows, entry(eng, slots, kernels) evaluates the listed slots in one launch.  A group with maxIter <= 0 is
    skipped: it takes its kernels' own hyper-parameters, as GPR.fit does.  Yields (slots, thetas, the `fit_slots` record,
    upload's return) per optimised group."""
    for slots in group_slots(ests, n).values():
        e0 = ests[slots[0][0]]
        if e0._maxIter <= 0:
            continue
        with context(e0._device) as eng:
            uploaded = upload(eng, e0._datasetSizeForExpert)
            objective = slot_objective([ests[p] for p, _ in slots],
                                       lambda listed, kernels: entry(eng, [slots[i] for i in listed], kernels))
            thetas, fit = fit_slots(eng, e0, objective, [ests[p].getKernel().getHyperparameters() for p, _ in slots])
        yield slots, thetas, fit, uploaded


class CrossValidatorModel(_SelectedModel):
    """Spark's CrossValidatorModel: the best map refitted on every row, and each map's metric averaged over the folds."""

    def __init__(self, bestModel, avgMetrics, bestIndex, last_objective):
        super().__init__(bestModel, bestIndex, last_objective)
        self.avgMetrics = list(avgMetrics)


class CrossValidator(_Validator):
    NAME = "CrossValidator"
    ESTIMATORS = (GaussianProcessRegression, OneVsRest)
    EVALUATORS = (RegressionEvaluator, MulticlassClassificationEvaluator)

    def __init__(self):
        self._estimator = None
        self._evaluator = RegressionEvaluator()
        self._maps = None
        self._num_folds = 3
        self._seed = 0
        self.last_folds = None            # {(map, fold): theta, magicVector and validation prediction of the fold model}

    def setEstimator(self, value):
        """A GaussianProcessRegression or a OneVsRest.  The binary GaussianProcessClassifier is refused: the fold-slot
        objective already serves it (class 1 over 0/1 labels), but its selector path is not built."""
        if not isinstance(value, self.ESTIMATORS):
            raise TypeError("CrossValidator: the estimator must be a GaussianProcessRegression or a OneVsRest, not %s"
                            % type(value).__name__)
        self._estimator = value
        return self

    def setEvaluator(self, value):
        if not isinstance(value, self.EVALUATORS):
            raise TypeError("CrossValidator: the evaluator must be a RegressionEvaluator or a "
                            "MulticlassClassificationEvaluator, not %s" % type(value).__name__)
        self._evaluator = value
        return self

    def setNumFolds(self, value: int):
        if int(value) < 2:
            raise ValueError("CrossValidator: numFolds must be >= 2")
        self._num_folds = int(value)
        return self

    def getNumFolds(self) -> int:
        return self._num_folds

    def fit(self, X, y, folds=None) -> CrossValidatorModel:
        """folds: the fold of every row (integers in [0, numFolds)); default: the seeded split of the module docstring.
        When the estimator (or the wrapped classifier) has a process group, (X, y) and folds are this rank's shard of
        the rows (`distributed.selection`); every rank returns the same metrics, bestIndex and refitted model."""
        est = self._estimator
        if est is None:
            raise TypeError("CrossValidator: setEstimator(GaussianProcessRegression or OneVsRest) first")
        ovr = isinstance(est, OneVsRest)
        if ovr and not isinstance(est.getClassifier(), GaussianProcessClassifier):
            raise TypeError("OneVsRest: setClassifier(GaussianProcessClassifier) first")
        gp = est.getClassifier() if ovr else est
        K = self._num_folds
        if gp._process_group is not None:
            from . import distributed
            ests = [est.copy(m) for m in self._maps or [{}]]
            split = lambda n, offset: [f != k for f in [self._folds(folds, n, offset)] for k in range(K)]
            with distributed.selection(gp, [e.getClassifier() if ovr else e for e in ests],
                                       "classes" if ovr else "regression", X, y, split, self.NAME + ".fit",
                                       self._empty_fold) as site:
                return self._cross_validate(site, est, ests, site.X, site.y, (X, y))
        X, y = self._data(X, y, gp._device, ovr)
        fold_of = self._folds(folds, len(X), 0)
        train = [fold_of != k for k in range(K)]
        message = self._empty_fold(len(X), [int(np.count_nonzero(t)) for t in train])
        if message is not None:
            raise ValueError(message)
        ests = [est.copy(m) for m in self._maps or [{}]]
        return self._cross_validate(_Local(X, y, train, fold_of), est, ests, X, y, (X, y))

    def _folds(self, folds, n: int, offset: int):
        """The fold of each of n rows, the rows [offset, offset + n) of the data: the seeded split, or the given one
        checked."""
        if folds is None:
            return kfold_assignment(n, self._num_folds, self._seed, offset)
        f = np.asarray(folds)
        if f.shape != (n,) or not np.all((f == np.floor(f)) & (f >= 0) & (f < self._num_folds)):
            raise ValueError("CrossValidator: folds must hold one integer in [0, numFolds) per row")
        return f.astype(np.int32)

    @staticmethod
    def _empty_fold(n: int, n_train):
        """The refusal of a split of n rows whose training set k holds n_train[k] rows: the first empty fold."""
        empty = [k for k, t in enumerate(n_train) if t == n]
        return "CrossValidator: fold %d has no rows to validate on" % empty[0] if empty else None

    def _cross_validate(self, site, est, ests, X, y, refit):
        """Every (map, fold) of the split site.members (fold k's training mask) on the site's rows (X, y): the slot fits,
        the fold models, their metrics on the gathered validation arrays, and the refit of the best map on refit."""
        K = len(site.members)
        maps = self._maps or [{}]
        y_val = [site.gather(_rows(y, ~t)) for t in site.members]
        if isinstance(est, OneVsRest):
            folds_out, objective = self._fit_one_vs_rest([e.getClassifier() for e in ests], X, y, site)
            metrics = np.array([[self._evaluator.evaluate(y_val[k], folds_out[p, k]["prediction"]) for k in range(K)]
                                for p in range(len(maps))])
            return self._select(est, maps, refit, K, metrics, folds_out, objective)
        thetas, objective = self._optimise(ests, site)
        metrics = np.empty((len(maps), K))
        folds_out = {}
        for p, e in enumerate(ests):
            for k, train in enumerate(site.members):
                pred, mv = site.validate(e, k, _rows(X, train), _rows(y, train), _rows(X, ~train), thetas[p][k])
                folds_out[p, k] = dict(theta=thetas[p][k], magicVector=mv, prediction=pred)
                metrics[p, k] = self._evaluator.evaluate(y_val[k], pred)
        return self._select(est, maps, refit, K, metrics, folds_out, objective)

    def _select(self, est, maps, refit, K, metrics, folds_out, objective):
        """avgMetrics, the first best map refitted on the rows refit = (X, y), and the records of the fit."""
        avg = [sum(metrics[p, k] for k in range(K)) / K for p in range(len(maps))]
        best = best_index(avg, self._evaluator.isLargerBetter())
        self.last_folds = folds_out
        objective["fold_metrics"] = metrics
        return CrossValidatorModel(est.copy(maps[best]).fit(*refit), avg, best, objective)

    @staticmethod
    def _fit_one_vs_rest(gps, X, y, site):
        """Every (map p, fold k) of one-vs-rest over the classifiers gps (one per map): the fold's C_k class models, as
        `OneVsRest().setClassifier(gps[p]).fit(X[train], y[train])` fits them, and their validation prediction.  Per
        group of slots one upload of the training sets (`site.upload_sets`), one lock-step L-BFGS-B over the (map, fold,
        class) slots with one `sgp_laplace_nll_fold_slots_any_size` call per round, and one more call at every slot's
        optimum (GPCls:60).  Returns ({(p, k): theta (C_k x h), magicVector [C_k], prediction}, dict(groups=...))."""
        train = site.members
        K = len(train)
        C = site.set_classes(True)
        thetas, latent, groups = {}, {}, []
        for slots in fold_class_slot_groups(gps, C).values():
            g0 = gps[slots[0][0]]
            with site.context(g0._device) as eng:
                n_k, n_experts = site.upload_sets(eng, g0._datasetSizeForExpert)
                entry = lambda listed, kernels: eng.laplace_nll_fold_slots_any_size(
                    len(gps) * sum(C), [slots[i][3] for i in listed], [slots[i][1] for i in listed],
                    [slots[i][2] for i in listed], kernels, g0._tol)
                fitted, fit = fit_slots(eng, g0, slot_objective([gps[p] for p, _, _, _ in slots], entry),
                                        [gps[p].getKernel().getHyperparameters() for p, _, _, _ in slots], laplace=True)
                # every objective call is one round, and one more runs at the slots' thetas
                groups.append(dict(
                    slots=[dict(map=p, fold=k, cls=c, mode_slot=m, theta=theta, **r)
                           for (p, k, c, m), r, theta in zip(slots, fit["slots"] or [{}] * len(slots), fitted)],
                    rounds=fit["rounds"], calls=fit["rounds"] + 1, launches=fit["launches_total"]))
                for (p, k, c, m), theta in zip(slots, fitted):
                    thetas[p, k, c] = theta
                    latent[p, k, c] = slot_modes(eng, site.on_device, n_k[k], n_experts[k], None, m, fold=k)
        folds_out = {}
        with site.context(gps[0]._device) as eng:
            for p, gp in enumerate(gps):
                for k in range(K):
                    Xt, Xv = _rows(X, train[k]), _rows(X, ~train[k])
                    raw, mvs = np.empty((len(Xv), C[k])), []
                    for c in range(C[k]):
                        mvs.append(site.fold_model(gp, eng, k, Xt, latent[p, k, c], thetas[p, k, c]).magic_vector)
                        raw[:, c] = site.latent_mean(eng, Xv)
                    folds_out[p, k] = dict(theta=np.array([thetas[p, k, c] for c in range(C[k])]), magicVector=mvs,
                                           prediction=one_vs_rest_prediction(site.gather(raw)))
        return folds_out, dict(groups=groups)

    @staticmethod
    def _optimise(ests, site):
        """Optimal hyper-parameters of every (map, fold) slot (thetas[p][k]), and what the optimisation took: per group
        of slots one upload of the training sets (`site.upload_sets`), each round one `sgp_bcm_nll_folds` launch
        (`_bcm_groups`)."""
        K = len(site.members)
        thetas = [[np.asarray(e.getKernel().getHyperparameters(), dtype=np.float64)] * K for e in ests]
        groups = []
        for slots, fitted, fit, _ in _bcm_groups(
                ests, K, site.upload_sets, lambda eng, slots, kernels: eng.bcm_nll_folds([k for _, k in slots], kernels),
                site.context):
            groups.append(dict(slots=[dict(map=p, fold=k, **r) for (p, k), r in zip(slots, fit["slots"])],
                               rounds=fit["rounds"], launches=fit["launches"]))
            for (p, k), theta in zip(slots, fitted):
                thetas[p][k] = theta
        return thetas, dict(groups=groups)


class TrainValidationSplitModel(_SelectedModel):
    """Spark's TrainValidationSplitModel: the best map refitted on every row, and each map's validation metric."""

    def __init__(self, bestModel, validationMetrics, bestIndex, last_objective):
        super().__init__(bestModel, bestIndex, last_objective)
        self.validationMetrics = list(validationMetrics)


class TrainValidationSplit(_Validator):
    NAME = "TrainValidationSplit"
    ESTIMATORS = (GaussianProcessRegression, GaussianProcessClassifier, OneVsRest)
    EVALUATORS = (RegressionEvaluator, MulticlassClassificationEvaluator, BinaryClassificationEvaluator)

    def __init__(self):
        self._estimator = None
        self._evaluator = None
        self._maps = None
        self._train_ratio = 0.75
        self._seed = 0
        self.last_predictions = None      # each map's validation predictions, in map order

    def setEstimator(self, value):
        if not isinstance(value, self.ESTIMATORS):
            raise TypeError("TrainValidationSplit: the estimator must be a GaussianProcessRegression, a "
                            "GaussianProcessClassifier or a OneVsRest, not %s" % type(value).__name__)
        self._estimator = value
        return self

    def setEvaluator(self, value):
        """A RegressionEvaluator, a MulticlassClassificationEvaluator (on the predictions) or, over the binary
        GaussianProcessClassifier only, a BinaryClassificationEvaluator (on the validation latent mean f)."""
        if not isinstance(value, self.EVALUATORS):
            raise TypeError("TrainValidationSplit: the evaluator must be a RegressionEvaluator, a "
                            "MulticlassClassificationEvaluator or a BinaryClassificationEvaluator, not %s"
                            % type(value).__name__)
        self._evaluator = value
        return self

    def setTrainRatio(self, value: float):
        if not 0.0 < float(value) < 1.0:
            raise ValueError("TrainValidationSplit: trainRatio must lie in (0, 1)")
        self._train_ratio = float(value)
        return self

    def getTrainRatio(self) -> float:
        return self._train_ratio

    def fit(self, X, y, train=None) -> TrainValidationSplitModel:
        """train: a bool mask of the training rows; default: the seeded split of the module docstring.  When the
        estimator (or the wrapped classifier) has a process group, (X, y) and train are this rank's shard of the rows
        (`distributed.selection`); every rank returns the same metrics, bestIndex and refitted model."""
        est = self._estimator
        if est is None:
            raise TypeError("TrainValidationSplit: setEstimator first")
        if self._evaluator is None:
            raise ValueError("TrainValidationSplit: setEvaluator first (there is no default evaluator)")
        scored = isinstance(self._evaluator, BinaryClassificationEvaluator)
        if scored and not isinstance(est, GaussianProcessClassifier):
            raise TypeError("TrainValidationSplit: a BinaryClassificationEvaluator scores the binary "
                            "GaussianProcessClassifier only, not a %s" % type(est).__name__)
        gp = est.getClassifier() if isinstance(est, OneVsRest) else est
        if getattr(gp, "_process_group", None) is not None:
            from . import distributed
            ests = [est.copy(m) for m in self._maps or [{}]]
            kind = {GaussianProcessRegression: "regression", GaussianProcessClassifier: "binary"}.get(type(est), "classes")
            with distributed.selection(gp, [e.getClassifier() if kind == "classes" else e for e in ests], kind, X, y,
                                       lambda n, offset: [self._mask(train, n, offset)], self.NAME + ".fit",
                                       self._empty_side) as site:
                return self._validate_split(site, est, ests, scored, site.X, site.y, (X, y))
        X, y = self._data(X, y, getattr(gp, "_device", 0),          # a OneVsRest without a classifier fails below
                          not isinstance(est, GaussianProcessRegression))
        mask = self._mask(train, len(X), 0)
        message = self._empty_side(len(X), [int(np.count_nonzero(mask))])
        if message is not None:
            raise ValueError(message)
        ests = [est.copy(m) for m in self._maps or [{}]]
        return self._validate_split(_Local(X, y, [mask]), est, ests, scored, X, y, (X, y))

    def _mask(self, train, n: int, offset: int):
        """The training mask of n rows, the rows [offset, offset + n) of the data: the seeded split, or the given one
        checked."""
        if train is None:
            return train_validation_assignment(n, self._train_ratio, self._seed, offset)
        mask = np.asarray(train)
        if mask.shape != (n,) or not np.all((mask == 0) | (mask == 1)):
            raise ValueError("TrainValidationSplit: train must hold one bool per row")
        return mask.astype(bool)

    @staticmethod
    def _empty_side(n: int, n_train):
        """The refusal of a split of n rows with n_train[0] training rows: an empty side."""
        if n_train[0] == 0 or n_train[0] == n:
            return "TrainValidationSplit: the %s side of the split is empty" % ("training" if n_train[0] == 0
                                                                                else "validation")
        return None

    def _validate_split(self, site, est, ests, scored, X, y, refit):
        """Every map on the site's training rows (site.members[0]) of (X, y), its metric on the gathered validation
        arrays, and the refit of the best map on refit."""
        mask = site.members[0]
        maps = self._maps or [{}]
        if isinstance(est, GaussianProcessRegression):
            preds, objective = self._fit_regression(ests, X, y, mask, site)
            evaluated = preds
        else:
            preds, raw, objective = self._fit_classifiers(ests, isinstance(est, OneVsRest), X, y, mask, site)
            evaluated = [r[:, 0] for r in raw] if scored else preds      # rawPrediction(1) = f
        y_val = site.gather(_rows(y, ~mask))
        metrics = [self._evaluator.evaluate(y_val, p) for p in evaluated]
        best = best_index(metrics, self._evaluator.isLargerBetter())
        self.last_predictions = preds
        return TrainValidationSplitModel(est.copy(maps[best]).fit(*refit), metrics, best, objective)

    @staticmethod
    def _fit_regression(ests, X, y, train, site=None):
        """Validation predictions of every map of the regression estimator, and what the optimisation took: per group of
        maps (`group_slots`) one grouped upload of the training rows and one lock-step L-BFGS-B over the maps, each
        round one `sgp_bcm_nll_slots` launch.  A group with maxIter <= 0 takes its kernels' own hyper-parameters, as
        GPR.fit does.  Each map's model is then produced on the training rows.  site: the `_Local` of (X, y, train) by
        default.  Returns (predictions, dict(maps=[each map's dict(theta, magicVector, evaluations, iterations; value and
        n_experts when optimised)], groups=[dict(maps, rounds, launches)]))."""
        site = site or _Local(X, y, [train])
        Xt, yt, Xv = _rows(X, train), _rows(y, train), _rows(X, ~train)
        thetas = [np.asarray(e.getKernel().getHyperparameters(), dtype=np.float64) for e in ests]
        records, groups = [dict(evaluations=0, iterations=0) for _ in ests], []
        for slots, fitted, fit, uploaded in _bcm_groups(
                ests, 1, lambda eng, n_e: site.upload_training(eng, n_e, Xt, yt),
                lambda eng, slots, kernels: eng.bcm_nll_slots(kernels), site.context):
            groups.append(dict(maps=[p for p, _ in slots], rounds=fit["rounds"], launches=fit["launches"]))
            for (p, _), theta, r in zip(slots, fitted, fit["slots"]):
                thetas[p] = theta
                records[p] = dict(r, n_experts=uploaded[2])
        preds = []
        for e, theta, r in zip(ests, thetas, records):
            pred, mv = site.validate(e, 0, Xt, yt, Xv, theta)
            preds.append(pred)
            r.update(theta=theta, magicVector=mv)
        return preds, dict(maps=records, groups=groups)

    @staticmethod
    def _fit_classifiers(ests, ovr: bool, X, y, train, site=None):
        """Validation predictions of every map of the binary classifier (ovr False) or of one-vs-rest, their raw
        columns (each class's latent mean f), and what the optimisation took: per group of maps one upload, one
        lock-step L-BFGS-B over the (map, class) slots, one `sgp_laplace_nll_slots_any_size` call per round and one at
        every slot's optimum (GPCls:60).  site: the `_Local` of (X, y, train) by default."""
        site = site or _Local(X, y, [train])
        gps = [e.getClassifier() for e in ests] if ovr else ests
        if any(not isinstance(gp, GaussianProcessClassifier) for gp in gps):
            raise TypeError("OneVsRest: setClassifier(GaussianProcessClassifier) first")
        C = site.set_classes(ovr)[0]                        # as an independent OneVsRest.fit(X[train], y[train])
        label = (lambda c: c) if ovr else (lambda c: 1)     # binary: y == 1 is y itself
        Xt, yt, Xv = _rows(X, train), _rows(y, train), _rows(X, ~train)
        raw = [np.empty((len(Xv), C)) for _ in gps]
        groups = []
        for slots in tvs_slot_groups(gps, C).values():
            g0 = gps[slots[0][0]]
            modes = [m for _, _, m in slots]
            with site.context(g0._device) as eng:
                entry = lambda listed, kernels: eng.laplace_nll_slots_any_size(
                    len(gps) * C, [modes[i] for i in listed], [label(slots[i][1]) for i in listed], kernels, g0._tol)
                upload = lambda eng: site.upload_training(eng, g0._datasetSizeForExpert, Xt, yt, laplace=True)[:2]
                thetas, latent, fit = laplace_fit([gps[p] for p, _, _ in slots], eng, Xt, yt, entry, N.SGP_MODES_SLOT,
                                                  lambda i: modes[i], upload=upload)
                # every objective call is one round, and one more runs at the slots' thetas
                groups.append(dict(
                    slots=[dict(map=p, cls=c, mode_slot=m, theta=theta, **r)
                           for (p, c, m), r, theta in zip(slots, fit["slots"] or [], thetas)],
                    rounds=fit["rounds"], calls=fit["rounds"] + 1, launches=fit["launches_total"]))
                for (p, c, _), f, theta in zip(slots, latent, thetas):
                    site.fold_model(gps[p], eng, 0, Xt, f, theta)
                    raw[p][:, c] = site.latent_mean(eng, Xv)
        raw = [site.gather(r) for r in raw]
        if ovr:
            preds = [one_vs_rest_prediction(r) for r in raw]
        else:                                               # GaussianProcessClassificationModel.predict
            preds = [binary_prediction(np.stack([-r[:, 0], r[:, 0]], axis=-1)) for r in raw]
        return preds, raw, dict(groups=groups)
