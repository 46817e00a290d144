"""Host-side mirror of `classification/GaussianProcessClassifier.scala` (binary GP classification, Laplace
approximation per expert + the same projected-process model as regression with y := latent mode f)."""
from __future__ import annotations

import numpy as np
from scipy.optimize import minimize

from .engine import ProjectedProcessEngine, is_cuda_tensor
from .hyperopt import pack_experts, group_for_experts
from .regression import GaussianProcessParams, GaussianProjectedProcessRawPredictor


class GaussianProcessClassificationModel:
    """GPCls:137-162."""

    def __init__(self, rawPredictor: GaussianProjectedProcessRawPredictor, hyperparameters):
        self.rawPredictor, self.hyperparameters = rawPredictor, hyperparameters
        self.numClasses = 2

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

    def predict(self, features):
        """ClassificationModel.predict = raw2prediction(predictRaw(x)); with no thresholds set (the reference sets none)
        Spark's ProbabilisticClassificationModel.raw2prediction is `rawPrediction.argmax`, i.e. class 1 iff f > 0 (first
        maximum on a tie) -- NOT the argmax of the (quirky) probability vector."""
        raw = self.predictRaw(features)
        if is_cuda_tensor(raw):
            import torch
            return torch.argmax(raw, dim=-1).to(torch.float64)
        return np.argmax(raw, axis=-1).astype(np.float64)


class GaussianProcessClassifier(GaussianProcessParams):
    """GPCls:42-135."""

    def __init__(self, device: int = 0):
        super().__init__()
        self._device = device
        self.last_objective = None

    def fit(self, X, y, hyperparameters=None) -> GaussianProcessClassificationModel:
        X = np.asarray(X, dtype=np.float64)
        y = np.asarray(y, dtype=np.float64)
        if not np.all((y == 0.0) | (y == 1.0)):                     # assertLabelsAre01, GPCls:68-72
            raise RuntimeError("Only 0 and 1 labels are supported.")
        eng = ProjectedProcessEngine.acquire(self._device)
        groups = group_for_experts(len(X), self._datasetSizeForExpert)
        order = np.concatenate(groups)
        eng.experts_upload_grouped(X, y, self._datasetSizeForExpert)  # grouping on the device; f = zeros per expert (GPCls:53-55)
        memo = {}

        def objective(theta):                                       # memoised like DiffFunctionMemoized; f warm-starts
            key = tuple(theta)
            if key not in memo:
                memo[key] = eng.laplace_nll(self.getKernel().setHyperparameters(np.asarray(theta)), self._tol)
            return memo[key]

        if hyperparameters is None:
            k0 = self.getKernel()
            theta = k0.getHyperparameters()
            if self._maxIter > 0 and len(theta) > 0:
                lo, up = k0.hyperparameterBoundaries()
                bounds = [(float(l), None if np.isinf(u) else float(u)) for l, u in zip(lo, up)]
                res = minimize(objective, theta, jac=True, method="L-BFGS-B", bounds=bounds,
                               options=dict(maxiter=self._maxIter, ftol=self._tol, gtol=self._tol))
                theta = np.asarray(res.x, dtype=np.float64)
                self.last_objective = dict(value=float(res.fun), evaluations=len(memo), iterations=int(res.nit))
        else:
            theta = np.asarray(hyperparameters, dtype=np.float64)
        # GPCls:60: run the Laplace loop once more at the optimum so every expert's f is the mode at theta*
        eng.laplace_nll(self.getKernel().setHyperparameters(theta), self._tol)
        f_packed = eng.experts_f(len(X))
        f = np.empty(len(X))
        f[order] = f_packed
        self.last_latent = f
        # GPCls:62-65 -> produceModel with (f, kernel): the same projected-process path as regression
        active_set = self._activeSetProvider(self._activeSetSize, X, f, self.getKernel, theta, self._seed, gp=self)
        kernel = self.getKernel().setHyperparameters(theta)
        G, b = eng.statistics(kernel, active_set, X, f)             # same helper as regression (fp64-kernel fallback)
        mv, mm = eng.magic()
        self.last_stats = (G, b)
        return GaussianProcessClassificationModel(GaussianProjectedProcessRawPredictor(eng, mv, mm, kernel, active_set), theta)
