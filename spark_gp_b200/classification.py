"""Host-side mirror of `classification/GaussianProcessClassifier.scala` (binary GP classification, Laplace
approximation per expert + the same projected-process model as regression with y := latent mode f)."""
from __future__ import annotations

import numpy as np

from . import _native as N
from .engine import ProjectedProcessEngine, is_cuda_tensor
from .hyperopt import each, expert_count, fit_data, fit_slots, own_context, produce, slot_modes, slot_objective
from .regression import GaussianProcessParams, GaussianProjectedProcessRawPredictor


class GaussianProcessClassificationModel:
    """GPCls:137-162."""

    def __init__(self, rawPredictor: GaussianProjectedProcessRawPredictor, hyperparameters):
        self.rawPredictor, self.hyperparameters = rawPredictor, hyperparameters
        self.numClasses = 2

    @classmethod
    def of(cls, fitted):
        """The model of a fitted slot (`hyperopt.Fitted`), on the context that holds its active set and magic pair."""
        return cls(GaussianProjectedProcessRawPredictor(fitted.engine, fitted.magic_vector, fitted.magic_matrix,
                                                        fitted.kernel, fitted.active_set), fitted.theta)

    def predictRaw(self, features):
        """(-f, f) per row (GPCls:153-156).  A CUDA torch tensor stays on the device (CUDA float64 result)."""
        if is_cuda_tensor(features):
            import torch
            f, _ = self.rawPredictor._engine.predict_tensor(features, with_variance=False)
            return torch.stack([-f, f], dim=-1)
        f, _ = self.rawPredictor._engine.predict(np.asarray(features, dtype=np.float64), with_variance=False)
        return np.stack([-f, f], axis=-1)

    def predictProbability(self, features):
        """raw2probabilityInPlace (GPCls:140-148), quirk included: values(0) = sigmoid(-values(0)) = sigmoid(f), so the
        probability column puts sigmoid(f) on class 0 although f > 0 votes for class 1."""
        raw = self.predictRaw(features)
        if is_cuda_tensor(raw):
            import torch
            p0 = 1.0 / (1.0 + torch.exp(raw[..., 0]))
            return torch.stack([p0, 1.0 - p0], dim=-1)
        p0 = 1.0 / (1.0 + np.exp(raw[..., 0]))          # sigmoid(-(-f))
        return np.stack([p0, 1.0 - p0], axis=-1)

    def predictAveragedProbability(self, features, numNodes: int = 100):
        """n x 2 rows [1 - p, p]: p the probability of class 1 averaged over the latent posterior N(f*, var*) of the raw
        predictor (GPML eq. 3.25), p = E[sigmoid(f)] by the numNodes-node Gauss-Hermite rule, as
        commons/util/Integrator.scala computes it (IntegratorTest's 100 nodes by default; a negative variance is taken as
        0, where the Integrator would return NaN).  Class 1 is column 1, unlike `predictProbability`.  One vector gives
        one row; a CUDA torch tensor stays on the device (CUDA float64 result)."""
        engine = self.rawPredictor._engine
        if is_cuda_tensor(features):
            import torch
            p, _, _ = engine.predict_probability_tensor(features, nodes=numNodes)
            return torch.stack([1.0 - p, p], dim=-1)
        p, _, _ = engine.predict_probability(np.asarray(features, dtype=np.float64), nodes=numNodes)
        return np.stack([1.0 - p, p], axis=-1)

    def predict(self, features):
        """ClassificationModel.predict = raw2prediction(predictRaw(x)); with no thresholds set (the reference sets none)
        Spark's ProbabilisticClassificationModel.raw2prediction is `rawPrediction.argmax`, i.e. class 1 iff f > 0 (first
        maximum on a tie) -- NOT the argmax of the (quirky) probability vector."""
        return binary_prediction(self.predictRaw(features))


class GaussianProcessClassifier(GaussianProcessParams):
    """GPCls:42-135."""

    def __init__(self, device: int = 0, process_group=None):
        """process_group: a torch.distributed process group (one process per GPU, NCCL) to fit over; each rank then
        passes its own shard to `fit` (`spark_gp_b200.distributed`)."""
        super().__init__()
        self._device = device
        self._process_group = process_group
        self.last_objective = None

    def fit(self, X, y, hyperparameters=None) -> GaussianProcessClassificationModel:
        """X may be a CUDA tensor on the classifier's device (y a CUDA tensor there too, or a host vector): X, the labels
        and the latent modes then stay on the device, and `last_latent` is a CUDA float64 tensor.
        With a process group, (X, y) is this rank's shard (possibly empty, 0 x d) and every rank returns the model of the
        concatenation of the shards in rank order, the same bits on every rank; `last_latent` then holds the modes of the
        rows of this rank's experts, in global row order."""
        if self._process_group is not None:
            from . import distributed
            fitted = distributed.fit(self, X, y, hyperparameters, True)
            self.last_stats, self.last_latent = fitted.stats, fitted.latent
            return GaussianProcessClassificationModel.of(fitted)
        X, y = fit_data(X, y, self._device, "GaussianProcessClassifier.fit")
        assert_labels_are_01(y)
        eng = ProjectedProcessEngine.acquire(self._device)
        (theta,), (f,), fit = laplace_fit(
            [self], eng, X, y, each(lambda k: eng.laplace_nll_any_size(k, self._tol)), N.SGP_MODES_BINARY, lambda _: 0,
            None if hyperparameters is None else [np.asarray(hyperparameters, dtype=np.float64)])
        if fit["slots"] is not None:
            self.last_objective = dict(fit["slots"][0], launches=fit["launches"])
        self.last_latent = f
        # GPCls:62-65 -> produceModel with (f, kernel): the same projected-process path as regression
        fitted = produce(self, eng, X, f, theta)
        self.last_stats = fitted.stats
        return GaussianProcessClassificationModel.of(fitted)


def assert_labels_are_01(y):
    """assertLabelsAre01 (GPCls:68-72), on a host array or on the device (only the verdict crosses PCIe)."""
    if not bool(((y == 0.0) | (y == 1.0)).all()):
        raise RuntimeError("Only 0 and 1 labels are supported.")


def laplace_fit(gps, eng, X, y, entry, store, index, thetas=None, upload=None):
    """The Laplace part of the binary fit (GPCls:53-60) for slot i of classifier gps[i], on one upload of (X, y) into eng
    grouped by gps[0]'s datasetSizeForExpert (every slot's modes start at 0), fitted by `fit_slots` from each classifier's
    kernel with gps[0]'s bounds, maxIter and tol.
      entry(slots, kernels) -> (values, gradients): the listed slots' Laplace objective (`slot_objective`), warm-started
                                                    from and moving their device-resident modes;
      store, index(i):                              where slot i's modes live (N.SGP_MODES_*, and the class or mode slot);
      upload(eng) -> (rows, experts):               another grouped upload in place of (X, y)'s (a data-parallel model
                                                    selection's rank uploads its experts' rows), X then only saying
                                                    on which side the modes go.
    Returns (thetas, modes [slot][row] in row order -- a CUDA float64 tensor, ungrouped on the device, when X is a CUDA
    tensor --, the fit record of `fit_slots`)."""
    if upload is None:
        n_rows, n_experts = len(X), expert_count(len(X), gps[0]._datasetSizeForExpert)
        eng.experts_upload_grouped(X, y, gps[0]._datasetSizeForExpert)
    else:
        n_rows, n_experts = upload(eng)
    thetas, fit = fit_slots(eng, gps[0], slot_objective(gps, entry), [gp.getKernel().getHyperparameters() for gp in gps],
                            thetas, laplace=True)
    latent = [slot_modes(eng, is_cuda_tensor(X), n_rows, n_experts, store, index(i)) for i in range(len(gps))]
    if is_cuda_tensor(X):
        import torch
        return thetas, torch.stack(latent), fit
    return thetas, np.stack(latent), fit


# ---- one-vs-rest ------------------------------------------------------------------------------------------------------
# Spark 3.1's ml/classification/OneVsRest.scala (not part of the reference project; restated here from Spark's
# documented behaviour, as the reference's own Iris example uses it: classification/examples/Iris.scala wraps the binary
# classifier in `new OneVsRest().setClassifier(...)`):
#   - numClasses = max(label) + 1; class c is trained on the labels (y == c) ? 1 : 0 with the wrapped classifier's params;
#   - OneVsRestModel's rawPrediction is the vector over classes of each class model's rawPrediction(1) (here f_c(x)), its
#     prediction the argmax with the first maximum winning a tie; there is no probability column.
# One deviation: a label that is not a non-negative integer raises ValueError, where Spark would silently leave the row
# out of every class's positives.
#
# All classes share X and the expert grouping (GPC:26-31), so the points are uploaded and grouped once, and each round of
# the C hyper-parameter optimisations is one `sgp_laplace_nll_classes_any_size` launch over experts x classes.  Each class runs the
# binary pipeline: f_c from 0, its own L-BFGS-B from the same x0 and bounds, the Laplace loop once more at theta*_c
# (GPCls:60), then produceModel with y := f_c.  The results are the binary classifier's on (y == c), bit for bit.


def one_vs_rest_labels(y):
    """Validated class labels and numClasses = max(label) + 1 (Spark's OneVsRest).  A CUDA tensor is checked on the
    device (only the verdict and the maximum cross PCIe) and returned as a CUDA float64 tensor."""
    if is_cuda_tensor(y):
        import torch
        y, fin, floor = y.to(torch.float64), torch.isfinite, torch.floor
    else:
        y, fin, floor = np.asarray(y, dtype=np.float64), np.isfinite, np.floor
    if y.ndim != 1 or len(y) == 0:
        raise ValueError("OneVsRest: labels must be a non-empty vector")
    if not bool((fin(y) & (y >= 0.0) & (y == floor(y))).all()):
        raise ValueError("OneVsRest: labels must be non-negative integers (class indices)")
    return y, int(y.max()) + 1


def binary_prediction(raw):
    """The binary classifier's prediction from its n x 2 raw matrix (-f, f): Spark's raw2prediction, `rawPrediction.argmax`
    (class 1 iff f > 0, the first maximum on a tie), as float64 class indices."""
    if is_cuda_tensor(raw):
        import torch
        return torch.argmax(raw, dim=-1).to(torch.float64)
    return np.argmax(raw, axis=-1).astype(np.float64)


def one_vs_rest_prediction(raw):
    """OneVsRestModel's prediction from the n x C raw matrix: the argmax over classes, the first maximum winning a tie, as
    float64 class indices."""
    if is_cuda_tensor(raw):
        import torch
        # torch.argmax does not promise the first maximum on ties: compare against the row maximum instead
        hit = raw == raw.max(dim=-1, keepdim=True).values
        first = torch.arange(raw.shape[-1], 0, -1, device=raw.device, dtype=torch.int64) * hit
        return torch.argmax(first, dim=-1).to(torch.float64)
    return np.argmax(raw, axis=-1).astype(np.float64)


class OneVsRestModel:
    """Spark's OneVsRestModel over GaussianProcessClassificationModel: one binary model per class."""

    def __init__(self, models, hyperparameters):
        self.models = list(models)
        self.numClasses = len(self.models)
        self.hyperparameters = hyperparameters          # numClasses x n_hypers

    def predictRaw(self, features):
        """n x numClasses: column c is class c's latent prediction f_c(x) (its model's rawPrediction(1)).  A CUDA torch
        tensor stays on the device (CUDA float64 result)."""
        cols = [m.predictRaw(features)[..., 1] for m in self.models]
        if is_cuda_tensor(features):
            import torch
            return torch.stack(cols, dim=-1)
        return np.stack(cols, axis=-1)

    def predictAveragedProbability(self, features, numNodes: int = 100):
        """n x numClasses: column c is class c's binary averaged probability (its model's
        `predictAveragedProbability` column 1).  These are one-vs-rest scores, each against the rest of the classes: a
        row is NOT normalised and need not sum to 1.  A CUDA torch tensor stays on the device (CUDA float64 result)."""
        cols = [m.predictAveragedProbability(features, numNodes)[..., 1] for m in self.models]
        if is_cuda_tensor(features):
            import torch
            return torch.stack(cols, dim=-1)
        return np.stack(cols, axis=-1)

    def predict(self, features):
        """The class index (float64) of the largest raw value, the first class winning a tie."""
        return one_vs_rest_prediction(self.predictRaw(features))

    transform = predict


class OneVsRest:
    """Spark's OneVsRest estimator over the binary GaussianProcessClassifier: `OneVsRest().setClassifier(gp).fit(X, y)`."""

    def __init__(self):
        self._classifier = None
        self.last_objective = None
        self.last_latent = None

    def setClassifier(self, value):
        if not isinstance(value, GaussianProcessClassifier):
            raise TypeError("OneVsRest: the classifier must be a GaussianProcessClassifier, not %s" % type(value).__name__)
        self._classifier = value
        return self

    def getClassifier(self):
        return self._classifier

    def copy(self, extra=None):
        """Spark's OneVsRest.copy(extra): a OneVsRest over classifier.copy(extra).  The params of `extra` are the wrapped
        classifier's (GaussianProcessParams.PARAMS)."""
        extra = dict(extra or {})
        unknown = sorted(set(extra) - set(GaussianProcessParams.PARAMS))
        if unknown:
            raise ValueError("unknown param(s) %s; the params are %s"
                             % (", ".join(unknown), ", ".join(GaussianProcessParams.PARAMS)))
        new = OneVsRest()
        if self._classifier is not None:
            new.setClassifier(self._classifier.copy(extra))
        return new

    def fit(self, X, y, hyperparameters=None) -> OneVsRestModel:
        """hyperparameters: None (optimise every class, as the binary fit does) or numClasses x n_hypers fixed values.
        When the classifier has a process group, (X, y) is this rank's shard (possibly empty, 0 x d) and every rank
        returns the model of the concatenation of the shards in rank order, the same bits on every rank; numClasses is
        the concatenation's, and `last_latent[c]` holds class c's modes at the rows of this rank's experts, in global
        row order (`spark_gp_b200.distributed`)."""
        gp = self._classifier
        if not isinstance(gp, GaussianProcessClassifier):
            raise TypeError("OneVsRest: setClassifier(GaussianProcessClassifier) first")
        if gp._process_group is not None:
            return self._fit_group(gp, X, y, hyperparameters)
        X, y = fit_data(X, y, gp._device, "OneVsRest.fit")
        y, C = one_vs_rest_labels(y)
        eng = ProjectedProcessEngine.acquire(gp._device)
        try:
            return self._fit(gp, eng, X, y, C, hyperparameters)
        finally:
            eng.release()

    def _fit(self, gp, eng, X, y, C, hyperparameters):
        n_hypers = len(gp.getKernel().getHyperparameters())
        given = None if hyperparameters is None else np.array(hyperparameters, dtype=np.float64).reshape(C, n_hypers)
        thetas, latent, fit = laplace_fit(
            [gp] * C, eng, X, y, lambda classes, kernels: eng.laplace_nll_classes_any_size(C, classes, kernels, gp._tol),
            N.SGP_MODES_CLASS, lambda c: c, given)
        thetas = np.array(thetas).reshape(C, n_hypers)
        self._record(fit)
        models = []
        for c in range(C):
            fitted = produce(gp, eng, X, latent[c], thetas[c])                  # produceModel in the fit's context
            models.append(GaussianProcessClassificationModel.of(own_context(fitted, gp._device)))
        self.last_latent = latent
        return OneVsRestModel(models, thetas)

    def _fit_group(self, gp, X, y, hyperparameters):
        from . import distributed
        slots, fit = distributed.group_fit(gp, X, y, hyperparameters, "classes")
        self._record(fit)
        thetas = np.array([fitted.theta for fitted in slots]).reshape(len(slots), -1)
        latent = [fitted.latent for fitted in slots]
        if is_cuda_tensor(latent[0]):
            import torch
            self.last_latent = torch.stack(latent)
        else:
            self.last_latent = np.stack(latent)
        models = [GaussianProcessClassificationModel.of(fitted) for fitted in slots]
        return OneVsRestModel(models, thetas)

    def _record(self, fit):
        if fit["slots"] is not None:
            self.last_objective = dict(classes=fit["slots"], rounds=fit["rounds"], launches=fit["launches"])
