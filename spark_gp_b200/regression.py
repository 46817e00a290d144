"""Host-side mirror of the reference's Estimator surface for regression
(`regression/GaussianProcessRegression.scala`, `commons/GaussianProcessParams.scala`,
`commons/GaussianProcessCommons.scala`): the same setters, defaults and call order; the data-parallel
statistics, the m x m tail and prediction run in the CUDA library.

Spark `Dataset` plumbing (label/features columns, RDD caching) has no meaning here: `fit` takes the
feature matrix and the labels directly."""
from __future__ import annotations

import copy

import numpy as np

from . import _native as N
from .engine import ProjectedProcessEngine, OperandRangeError, NotPositiveDefiniteException, host_copy, is_cuda_tensor, \
    rows_to_host
from .hyperopt import draw_active_set, fit_data, optimize_hypers, produce
from .kernels import Kernel, RBFKernel, EyeKernel, const


class ActiveSetProvider:
    """commons/ActiveSetProvider.scala:13-20.  `gp` (keyword) is the estimator that calls the provider: the reference
    hands over the grouped RDD of experts, here the provider reads datasetSizeForExpert / device from it if it needs to."""
    def __call__(self, activeSetSize, X, y, kernel_factory, optimalHyperparameter, seed, gp=None):
        raise NotImplementedError


class _RandomActiveSetProvider(ActiveSetProvider):
    """commons/ActiveSetProvider.scala:48-56: uniform sample without replacement.  (Spark's `takeSample`
    RNG stream is not reproduced -- the reference pins no test on it; pass an explicit active set through
    `ExplicitActiveSetProvider` when results must be compared.)  A CUDA tensor X gives the same rows, gathered on the
    device: only they cross PCIe."""
    def __call__(self, activeSetSize, X, y, kernel_factory, optimalHyperparameter, seed, gp=None):
        rng = np.random.default_rng(seed)
        idx = rng.choice(len(X), size=min(activeSetSize, len(X)), replace=False)
        return rows_to_host(X, idx)                                 # index first: no fp64 copy of the whole shard


RandomActiveSetProvider = _RandomActiveSetProvider()


class ExplicitActiveSetProvider(ActiveSetProvider):
    def __init__(self, active_set):
        self.active_set = np.asarray(active_set, dtype=np.float64)

    def __call__(self, activeSetSize, X, y, kernel_factory, optimalHyperparameter, seed, gp=None):
        return self.active_set


class KMeansActiveSetProvider(ActiveSetProvider):
    """commons/ActiveSetProvider.scala:22-46: K-means on the training features, the centroids are the active set
    (`new KMeans().setK(activeSetSize).setSeed(seed).setMaxIter(maxIter)`, Spark defaults otherwise: tol 1e-4).
    Host-side only: the clustering is a library call in the reference too (Spark MLlib); here scikit-learn's Lloyd
    iterations with k-means++ seeding stand in for Spark's k-means|| -- same objective and stopping rule, but Spark's
    initialisation RNG stream is unpinned, so results are comparable on metrics (RMSE), not centroid by centroid.

    `on_gpu=True` runs Spark's own algorithm on the device instead (`ProjectedProcessEngine.kmeans`, `sgp_kmeans`): k-means||
    seeding, empty clusters keep their centre, absolute centre-movement tolerance; float32 X is used without a copy.  May
    return fewer than activeSetSize centres when the data have fewer distinct points, as Spark does.  It reads a CUDA tensor
    X in place (`sgp_kmeans_device`); scikit-learn runs on the host, on an explicit host copy of such an X."""

    def __init__(self, maxIter: int = 20, on_gpu: bool = False):
        self.maxIter = int(maxIter)
        self.on_gpu = bool(on_gpu)

    def __call__(self, activeSetSize, X, y, kernel_factory, optimalHyperparameter, seed, gp=None):
        if self.on_gpu:
            eng = ProjectedProcessEngine.acquire(gp._device if gp is not None else 0)
            try:
                centres, _, _, _ = eng.kmeans(X, int(activeSetSize), max_iter=self.maxIter, tol=1e-4, seed=int(seed))
            finally:
                eng.release()
            return centres
        from sklearn.cluster import KMeans
        km = KMeans(n_clusters=int(activeSetSize), init="k-means++", n_init=1, max_iter=self.maxIter, tol=1e-4,
                    random_state=int(seed) % (2 ** 32), algorithm="lloyd")
        km.fit(np.asarray(host_copy(X), dtype=np.float64))
        return np.ascontiguousarray(km.cluster_centers_, dtype=np.float64)


class GreedilyOptimizingActiveSetProvider(ActiveSetProvider):
    """commons/ActiveSetProvider.scala:58-139 (Seeger et al. 2003 forward selection as the reference codes it).

    Every round is one pass of the hot path plus two passes of per-point quadratic forms, all on the GPU:
      (G, b)  = projected-process statistics for the current active set          (sgp_stats_*, ASP:90-96)
      p_i     = k_i' inv(K_mm) k_i,  q_i = k_i' inv(s2 K_mm + G) k_i,  mu_i = k_i' magicVector     (sgp_set_magic +
                sgp_predict, ASP:109-113); the small m x m inverses are host LAPACK like the reference's driver code.
    Reference semantics kept: `s2` is the kernel's whiteNoiseVar (ASP:76); candidates are folded per expert (point i
    belongs to expert i % E) with later-wins ties and NaN poisoning, NaN experts are dropped (ASP:108-131), the first
    expert with the best score wins; points already selected are not excluded.  The first point is `takeSample(1,
    seed)` in the reference (Spark's RNG stream is unpinned): `first_index` fixes it, else a seeded NumPy draw.

    `incremental=True` (default) runs the whole selection in `sgp_greedy_active_set`: the N x m cross kernel stays on the
    device and p_i, q_i, mu_i and the two inverses follow from rank-1 (bordered-matrix) updates -- O(N m) per round, all
    in fp64; `incremental=False` is the round-by-round form above (kept as the cross-check: both must select the points
    the CPU restatement selects).  On a CUDA tensor X the incremental selection converts X to float64 on the device and
    reads it in place (`sgp_greedy_active_set_device`), only the selected rows cross PCIe; the round-by-round form runs on
    an explicit host copy."""

    def __init__(self, first_index=None, precision=None, incremental=True):
        self.first_index = first_index
        self.precision = precision            # None: SGP_PREC_F64 (fp64 DMMA kernel); tests use SGP_PREC_F64_STRICT
        self.incremental = incremental

    def __call__(self, activeSetSize, X, y, kernel_factory, optimalHyperparameter, seed, gp=None):
        if is_cuda_tensor(X) and not self.incremental:
            X, y = host_copy(X), host_copy(y)
        on_device = is_cuda_tensor(X)
        X64 = X if on_device else np.ascontiguousarray(X, dtype=np.float64)
        y = y if on_device else np.asarray(y, dtype=np.float64)
        n = len(X64)
        n_e = gp._datasetSizeForExpert if gp is not None else 100
        E = int(np.floor(n / n_e + 0.5))
        if E <= 0:
            raise ZeroDivisionError("numberOfExperts == 0 (N < datasetSizeForExpert / 2)")
        first = self.first_index if self.first_index is not None else int(np.random.default_rng(seed).integers(n))
        theta = np.asarray(optimalHyperparameter, dtype=np.float64)
        eng = ProjectedProcessEngine.acquire(gp._device if gp is not None else 0)
        eng.set_precision(N.SGP_PREC_F64 if self.precision is None else self.precision)
        try:
            if self.incremental:
                kernel = kernel_factory().setHyperparameters(theta)
                return rows_to_host(X64, eng.greedy_active_set(kernel, X64, y, E, first, activeSetSize))
            active = X64[[first]].copy()
            while len(active) < activeSetSize:
                kernel = kernel_factory().setHyperparameters(theta)
                active = np.vstack([active, self._get_next(eng, kernel, X64, y, active, E)])
        finally:
            eng.release()
        return active

    @staticmethod
    def _get_next(eng, kernel, X, y, active, E):
        m, n = len(active), len(X)
        terms = kernel.flatten()
        s2 = kernel.whiteNoiseVar                                   # what ASP:76 passes as `sigma2`
        kii = sum(t["scale"] for t in terms)                        # trainingKernelDiag == selfKernel (Kernel.scala:111-114)
        eng.begin(kernel, active)
        eng.accumulate(X, y)
        G, b = eng.finish()
        kmm = eng.cross_kernel(active) + s2 * np.eye(m)             # trainingKernel: Eye terms on the diagonal
        pdm = s2 * kmm + G
        if np.linalg.eigvalsh((pdm + pdm.T) * 0.5).min() < 0:       # assertSymPositiveDefinite, PGPH:62-65
            raise NotPositiveDefiniteException()
        magic_vector = np.linalg.solve(pdm, b)
        eng.set_magic(np.zeros(m), np.linalg.inv(kmm))
        _, v = eng.predict(X)
        p = v - kii
        eng.set_magic(magic_vector, np.linalg.inv(pdm))
        mu, v = eng.predict(X)
        q = v - kii
        with np.errstate(all="ignore"):                             # ASP:114-124
            sigma = np.sqrt(s2)
            li = np.sqrt(kii - p)
            ksi = 1.0 / ((sigma / li) ** 2 + 1.0 - q)
            kappa = ksi * (1.0 + 2.0 * (sigma / li) ** 2)
            delta = -np.log(sigma / li) - (np.log(ksi) + ksi * (1.0 - kappa) / s2 * (y - mu) ** 2 - kappa + 2.0) / 2.0
        return X[GreedilyOptimizingActiveSetProvider.select_index(delta, E)]

    @staticmethod
    def select_index(delta, E: int) -> int:
        """ASP:108-135 vectorised: per-expert fold (expert e = points e, e+E, ...: any NaN drops the expert, ties go to
        the LATER point), then the FIRST expert with the maximal score."""
        n = len(delta)
        rows = -(-n // E)
        D = np.full(rows * E, -np.inf)
        D[:n] = delta
        D = D.reshape(rows, E)
        poisoned = np.isnan(D).any(axis=0)
        if poisoned.all():
            raise ValueError("empty.max")                           # RDD.max() on an empty RDD
        Dm = np.where(np.isnan(D), -np.inf, D)
        best = Dm.max(axis=0)
        last = rows - 1 - np.argmax(Dm[::-1] == best[None, :], axis=0)
        best = np.where(poisoned, -np.inf, best)
        e = int(np.argmax(best))                                    # first expert with the maximal score
        return int(last[e]) * E + e


class GaussianProcessParams:
    """commons/GaussianProcessParams.scala:8-54 (defaults at :33-51)."""

    def __init__(self):
        self._activeSetProvider = RandomActiveSetProvider
        self._kernel = lambda: RBFKernel()
        self._datasetSizeForExpert = 100
        self._sigma2 = 1e-3
        self._activeSetSize = 100
        self._maxIter = 100
        self._tol = 1e-6
        self._seed = 0

    def setActiveSetProvider(self, value): self._activeSetProvider = value; return self
    def setDatasetSizeForExpert(self, value: int): self._datasetSizeForExpert = int(value); return self
    def setMaxIter(self, value: int): self._maxIter = int(value); return self
    def setSigma2(self, value: float): self._sigma2 = float(value); return self
    def setKernel(self, value): self._kernel = value; return self
    def setTol(self, value: float): self._tol = float(value); return self
    def setActiveSetSize(self, value: int): self._activeSetSize = int(value); return self
    def setSeed(self, value: int): self._seed = int(value); return self

    def getKernel(self) -> Kernel:
        """commons/GaussianProcessCommons.scala:18: user kernel + sigma2.const * EyeKernel."""
        return self._kernel() + const(self._sigma2) * EyeKernel()

    # the params a ParamMap may set: the setter names without "set"
    PARAMS = ("sigma2", "datasetSizeForExpert", "activeSetSize", "maxIter", "tol", "seed", "kernel", "activeSetProvider")

    def copy(self, extra=None):
        """Spark's Params.copy(extra): a new estimator with this one's params (and device and shard size), then the
        params of `extra` ({name: value}, names as in PARAMS) set through their setters."""
        extra = dict(extra or {})
        unknown = sorted(set(extra) - set(self.PARAMS))
        if unknown:
            raise ValueError("unknown param(s) %s; the params are %s" % (", ".join(unknown), ", ".join(self.PARAMS)))
        new = copy.copy(self)
        for name in ("last_stats", "last_objective"):
            if hasattr(new, name):
                setattr(new, name, None)
        for name, value in extra.items():
            getattr(new, "set" + name[0].upper() + name[1:])(value)
        return new


class GaussianProjectedProcessRawPredictor:
    """commons/GaussianProcessCommons.scala:118-126.  Holds the engine whose device memory carries the
    active set, magicVector and magicMatrix."""

    def __init__(self, engine: ProjectedProcessEngine, magicVector, magicMatrix, kernel: Kernel, activeSet):
        self._engine = engine
        self.magicVector, self.magicMatrix, self.kernel, self.activeSet = magicVector, magicMatrix, kernel, activeSet

    def __del__(self):                          # the context goes back to the per-device pool
        try:
            self._engine.release()
        except Exception:
            pass

    def predict(self, features):
        """(mean, variance) for one vector or a block of vectors.  A CUDA torch tensor stays on the device: the results
        are CUDA float64 tensors (0-dim for one vector)."""
        if is_cuda_tensor(features):
            mean, var = self._engine.predict_tensor(features, with_variance=True)
            return (mean[0], var[0]) if features.ndim == 1 else (mean, var)
        f = np.asarray(features, dtype=np.float64)
        mean, var = self._engine.predict(f, with_variance=True)
        if f.ndim == 1:
            return float(mean[0]), float(var[0])
        return mean, var


class GaussianProcessRegressionModel:
    """regression/GaussianProcessRegression.scala:75-87: `predict` returns the mean only."""

    def __init__(self, rawPredictor: GaussianProjectedProcessRawPredictor, hyperparameters):
        self.rawPredictor = rawPredictor
        self.hyperparameters = hyperparameters

    @classmethod
    def of(cls, fitted):
        """The model of a fitted slot (`hyperopt.Fitted`), on the context that holds its active set and magic pair."""
        return cls(GaussianProjectedProcessRawPredictor(fitted.engine, fitted.magic_vector, fitted.magic_matrix,
                                                        fitted.kernel, fitted.active_set), fitted.theta)

    def predict(self, features):
        if is_cuda_tensor(features):                 # CUDA torch tensor in, CUDA float64 tensor out
            mean, _ = self.rawPredictor._engine.predict_tensor(features, with_variance=False)
            return mean[0] if features.ndim == 1 else mean
        f = np.asarray(features, dtype=np.float64)
        mean, _ = self.rawPredictor._engine.predict(f, with_variance=False)
        return float(mean[0]) if f.ndim == 1 else mean

    transform = predict


class GaussianProcessRegression(GaussianProcessParams):
    """regression/GaussianProcessRegression.scala:36-73."""

    def __init__(self, device: int = 0, shard_points: int = 1 << 22, process_group=None):
        """process_group: a torch.distributed process group (one process per GPU, NCCL) to fit over; each rank then
        passes its own shard to `fit` (`spark_gp_b200.distributed`)."""
        super().__init__()
        self._device = device
        self._shard_points = shard_points
        self._process_group = process_group
        self.last_stats = None

    def fit(self, X, y, hyperparameters=None) -> GaussianProcessRegressionModel:
        """GPR.train (:43-53).  `hyperparameters` short-circuits optimizeHypers (:48) with a given theta;
        otherwise the BCM objective is optimised when maxIter > 0.
        X may be a CUDA tensor on the estimator's device (y a CUDA tensor there too, or a host vector): X then never
        leaves the device; only the active set's rows and the small outputs cross PCIe.
        With a process group, (X, y) is this rank's shard (possibly empty, 0 x d) and every rank returns the model of the
        concatenation of the shards in rank order, the same bits on every rank."""
        if self._process_group is not None:
            from . import distributed
            fitted = distributed.fit(self, X, y, hyperparameters, False)
            self.last_stats = fitted.stats
            return GaussianProcessRegressionModel.of(fitted)
        X, y = fit_data(X, y, self._device, "GaussianProcessRegression.fit", keep_float32=True)
        if hyperparameters is None:
            if self._maxIter > 0:                   # per-expert BCM NLL on the GPU + L-BFGS-B on the host
                eng = ProjectedProcessEngine.acquire(self._device)
                try:
                    # expert grouping (GPC:26-31) as a strided gather on the device while the points stream in
                    hyperparameters = optimize_hypers(self, eng, eng.experts_upload_grouped(X, y,
                                                                                            self._datasetSizeForExpert))
                finally:
                    eng.release()
            else:
                hyperparameters = self.getKernel().getHyperparameters()
        return self._produce_model(X, y, np.asarray(hyperparameters, dtype=np.float64))

    def _produce_model(self, X, y, theta) -> GaussianProcessRegressionModel:
        """produceModel (commons/GaussianProcessCommons.scala:40-59, 102-110) on a context of the pool that the model
        keeps.  The active set is drawn first, so that a provider that takes a context of its own reuses the pooled one."""
        active_set = draw_active_set(self, X, y, theta)
        eng = ProjectedProcessEngine.acquire(self._device)
        fitted = produce(self, eng, X, y, theta, active_set)
        self.last_stats = fitted.stats
        return GaussianProcessRegressionModel.of(fitted)
