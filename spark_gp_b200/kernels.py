"""Host-side mirror of the reference's kernel DSL (`commons/kernel/*.scala`): same class names, the same
hyperparameter layout and bounds, the same sugar, and the same evaluation methods (setTrainingVectors, trainingKernel,
trainingKernelDiag, trainingKernelAndDerivative, crossKernel, selfKernel).  A kernel object here is a *description*:
`flatten()` turns the tree into the term list of `sgp_kernel_desc` (include/sgp.h), `hyper_descriptors()` says how the
matrix depends on each hyper-parameter, and the arithmetic runs in the CUDA library (`sgp_kernel_eval`, or
`sgp_kernel_eval_device` for CUDA tensors).  Only the diagonal quantities (selfKernel, trainingKernelDiag), sums of the
term scales, are computed here.

Scala                                   Python
  1 * new ARDRBFKernel(5)                 1 * ARDRBFKernel(5)
  1.const * new EyeKernel                 const(1) * EyeKernel()
  (0.5 between 0 and 1) * new EyeKernel   Scalar(0.5).between(0).and_(1) * EyeKernel()
  k1 + k2                                 k1 + k2
"""
from __future__ import annotations

import numpy as np

from . import _native as N


class Kernel:
    """commons/kernel/Kernel.scala:12-98."""

    def getHyperparameters(self) -> np.ndarray: raise NotImplementedError
    def setHyperparameters(self, value): raise NotImplementedError
    def numberOfHyperparameters(self) -> int: raise NotImplementedError
    def hyperparameterBoundaries(self): raise NotImplementedError
    def flatten(self, scale: float = 1.0) -> list: raise NotImplementedError

    def hyper_descriptors(self, scale: float = 1.0, term_offset: int = 0) -> list:
        """One dict per hyper-parameter, in getHyperparameters order, saying how the kernel matrix depends on it
        (consumed by sgp_bcm_nll): {"kind": SCALE, "coef": {term_index: d scale_t / d theta}} for a trainable scalar,
        {"kind": ARD_BETA, "term": t, "dim": k, "value": beta_k}, {"kind": RBF_SIGMA, "term": t, "value": sigma}."""
        raise NotImplementedError

    @property
    def whiteNoiseVar(self) -> float:
        return sum(t["scale"] for t in self.flatten() if t["type"] == N.SGP_TERM_EYE)

    def __add__(self, other): return SumOfKernels(self, other)

    def __rmul__(self, c):
        return (c if isinstance(c, Scalar) else Scalar(float(c))) * self

    # ---- evaluation (Kernel.scala:37-98) ----------------------------------------------------------------------------
    def _children(self) -> list: return []

    def setTrainingVectors(self, vectors, device: int = 0):
        """Kernel.scala:44-49: n x d vectors (one d-vector is one row), a host array or a CUDA tensor.  The kernel is
        evaluated on the tensor's device, or on cuda:`device` for a host array.  float32 is kept as it is (the library
        converts it to float64 exactly); other dtypes become float64.  Composite kernels pass the vectors on, as the
        reference's do."""
        from .engine import is_cuda_tensor
        if is_cuda_tensor(vectors):
            v, dev = (vectors if vectors.ndim == 2 else vectors.reshape(1, -1)), vectors.device.index
        else:
            v = np.asarray(vectors)
            v, dev = np.atleast_2d(v if v.dtype == np.float32 else v.astype(np.float64)), int(device)
        self._training = (v, dev)
        for child in self._children():
            child.setTrainingVectors(vectors, device)
        return self

    def getTrainingVectors(self):
        return self._training_vectors()[0]

    def _training_vectors(self):
        tv = getattr(self, "_training", None)
        if tv is None:
            from .engine import TrainingVectorsNotInitializedException
            raise TrainingVectorsNotInitializedException("setTrainingVectors method should have been called first")
        return tv

    def _evaluate(self, test, derivatives: bool):
        """(K, dK or None) from the library on a pooled context: the training kernel (test None) or crossKernel(test).
        When one side is a CUDA tensor the other goes to its device, and the results are CUDA float64 tensors."""
        from .engine import ProjectedProcessEngine, is_cuda_tensor
        train, device = self._training_vectors()
        if test is not None:
            if is_cuda_tensor(test) and not is_cuda_tensor(train):
                import torch
                device = test.device.index
                train = torch.as_tensor(train, device=test.device)
            elif is_cuda_tensor(train) and not is_cuda_tensor(test):
                import torch
                test = torch.as_tensor(np.asarray(test), device=train.device)
        eng = ProjectedProcessEngine.acquire(device)
        try:
            if test is None:
                return eng.kernel_eval(self, train, None, derivatives)
            return eng.kernel_eval(self, test, train, derivatives)
        finally:
            eng.release()

    def trainingKernel(self):
        """Kernel.scala:51-55: K[i][j] = k(x_i, x_j) over the training vectors, the Eye terms on the diagonal."""
        return self._evaluate(None, False)[0]

    def trainingKernelDiag(self):
        """Kernel.scala:57-61: the diagonal of trainingKernel, selfKernel on every row (computed here, no GPU call)."""
        from .engine import is_cuda_tensor
        train, _ = self._training_vectors()
        if is_cuda_tensor(train):
            import torch
            return torch.full((len(train),), self.selfKernel(None), dtype=torch.float64, device=train.device)
        return np.zeros(len(train)) + self.selfKernel(None)

    def trainingKernelAndDerivative(self):
        """Kernel.scala:63-68: (K, dK) with dK[i] = dK / d getHyperparameters()[i], an n_hypers x n x n array."""
        return self._evaluate(None, True)

    def crossKernel(self, test):
        """Kernel.scala:70-84: len(test) x len(trainingVectors) for n x d test vectors; one row for a single d-vector."""
        from .engine import is_cuda_tensor
        if not is_cuda_tensor(test):
            test = np.asarray(test)
            test = test if test.dtype == np.float32 else test.astype(np.float64)
        if test.ndim == 1:
            return self._evaluate(test.reshape(1, -1), False)[0][0]
        return self._evaluate(test, False)[0]

    def selfKernel(self, test) -> float:
        """Kernel.scala:86-90: k(x, x), the same for every x -- the sum of the term scales (every leaf has k(x, x) = 1)."""
        return float(sum(t["scale"] for t in self.flatten()))


class EyeKernel(Kernel):
    """Kernel.scala:142-164."""
    def getHyperparameters(self): return np.zeros(0)
    def setHyperparameters(self, value): return self
    def numberOfHyperparameters(self): return 0
    def hyperparameterBoundaries(self): return np.zeros(0), np.zeros(0)
    def flatten(self, scale=1.0): return [dict(type=N.SGP_TERM_EYE, scale=scale)]
    def hyper_descriptors(self, scale=1.0, term_offset=0): return []
    def __str__(self): return "I"


class ARDRBFKernel(Kernel):
    """ARDRBFKernel.scala:20-96; `ARDRBFKernel(p)` with an int is the `this(p: Int, beta = 1, ...)` ctor."""

    def __init__(self, beta, lower=None, upper=None):
        if isinstance(beta, (int, np.integer)):
            p = int(beta)
            self.beta = np.ones(p)
            self.lower = np.zeros(p) if lower is None else np.zeros(p) + lower
            self.upper = np.full(p, np.inf) if upper is None else np.zeros(p) + upper
        else:
            self.beta = np.array(beta, dtype=np.float64)
            self.lower = self.beta * 0.0 if lower is None else np.array(lower, dtype=np.float64)
            self.upper = np.full(len(self.beta), np.inf) if upper is None else np.array(upper, dtype=np.float64)

    def getHyperparameters(self): return self.beta
    def setHyperparameters(self, value):
        self.beta = np.array(value, dtype=np.float64)
        return self
    def numberOfHyperparameters(self): return len(self.beta)
    def hyperparameterBoundaries(self): return self.lower, self.upper
    def flatten(self, scale=1.0): return [dict(type=N.SGP_TERM_ARD, scale=scale, beta=self.beta.copy())]
    def hyper_descriptors(self, scale=1.0, term_offset=0):
        return [dict(kind=N.SGP_HYPER_ARD_BETA, term=term_offset, dim=k, value=float(b)) for k, b in enumerate(self.beta)]
    def __str__(self): return "ARDRBFKernel(beta=[" + ", ".join("%1.1e" % e for e in self.beta) + "])"


class RBFKernel(Kernel):
    """RBFKernel.scala:14-85."""

    def __init__(self, sigma: float = 1.0, lower: float = 1e-6, upper: float = np.inf):
        self.sigma, self.lower, self.upper = float(sigma), float(lower), float(upper)

    def getHyperparameters(self): return np.array([self.sigma])
    def setHyperparameters(self, value):
        self.sigma = float(np.asarray(value, dtype=np.float64)[0])
        return self
    def numberOfHyperparameters(self): return 1
    def hyperparameterBoundaries(self): return np.array([self.lower]), np.array([self.upper])
    def flatten(self, scale=1.0): return [dict(type=N.SGP_TERM_RBF, scale=scale, sigma=self.sigma)]
    def hyper_descriptors(self, scale=1.0, term_offset=0):
        return [dict(kind=N.SGP_HYPER_RBF_SIGMA, term=term_offset, dim=0, value=self.sigma)]
    def __str__(self): return "RBFKernel(sigma=%1.1e)" % self.sigma


class ConstantTimesKernel(Kernel):
    """ScalarTimesKernel.scala:41-59."""

    def __init__(self, kernel: Kernel, C: float):
        if not C >= 0:
            raise ValueError("requirement failed: C should be positive")
        self.kernel, self.C = kernel, float(C)

    def getHyperparameters(self): return self.kernel.getHyperparameters()
    def setHyperparameters(self, value):
        self.kernel.setHyperparameters(value)
        return self
    def numberOfHyperparameters(self): return self.kernel.numberOfHyperparameters()
    def hyperparameterBoundaries(self): return self.kernel.hyperparameterBoundaries()
    def flatten(self, scale=1.0): return self.kernel.flatten(scale * self.C)
    def hyper_descriptors(self, scale=1.0, term_offset=0):
        return self.kernel.hyper_descriptors(scale * self.C, term_offset)
    def _children(self): return [self.kernel]
    def __str__(self): return ("%1.1e * %s" % (self.C, self.kernel)) if self.C != 0 else ""


class TrainableScalarTimesKernel(ConstantTimesKernel):
    """ScalarTimesKernel.scala:71-98: C is a hyperparameter, PREPENDED to the inner kernel's vector."""

    def __init__(self, kernel: Kernel, C: float, Clower: float = 0.0, Cupper: float = np.inf):
        super().__init__(kernel, C)
        self.Clower, self.Cupper = float(Clower), float(Cupper)

    def getHyperparameters(self): return np.concatenate([[self.C], self.kernel.getHyperparameters()])
    def setHyperparameters(self, value):
        value = np.asarray(value, dtype=np.float64)
        self.C = float(value[0])
        self.kernel.setHyperparameters(value[1:])
        return self
    def numberOfHyperparameters(self): return 1 + self.kernel.numberOfHyperparameters()
    def hyperparameterBoundaries(self):
        lo, up = self.kernel.hyperparameterBoundaries()
        return np.concatenate([[self.Clower], lo]), np.concatenate([[self.Cupper], up])
    def hyper_descriptors(self, scale=1.0, term_offset=0):
        # dK/dC = (outer scale) * inner kernel matrix  (ScalarTimesKernel.scala:93-97): per inner term, its scale without C
        inner = self.kernel.flatten(scale)
        own = dict(kind=N.SGP_HYPER_SCALE, coef={term_offset + i: t["scale"] for i, t in enumerate(inner)})
        return [own] + self.kernel.hyper_descriptors(scale * self.C, term_offset)


class Scalar:
    """ScalarTimesKernel.scala:100-141."""

    def __init__(self, C, lower=0.0, upper=np.inf, isTrainable=True):
        if not ((lower < upper and isTrainable) or not isTrainable):
            raise ValueError("The scalar should either have its lower limit below its upper limit "
                             "or not be trainable")
        self.C, self.lower, self.upper, self.isTrainable = float(C), float(lower), float(upper), isTrainable

    def __mul__(self, kernel: Kernel):
        if self.isTrainable:
            return TrainableScalarTimesKernel(kernel, self.C, self.lower, self.upper)
        return ConstantTimesKernel(kernel, self.C)

    def between(self, lower):
        outer = self

        class _And:
            def and_(self, upper): return Scalar(outer.C, lower, upper, outer.isTrainable)
        return _And()

    def below(self, newUpper): return Scalar(self.C, self.lower, newUpper, self.isTrainable)

    @property
    def const(self): return Scalar(self.C, self.C, self.C, False)


def const(c: float) -> Scalar:
    return Scalar(c).const


def WhiteNoiseKernel(initial, lower, upper) -> Kernel:
    """Kernel.scala:166-169."""
    return Scalar(initial).between(lower).and_(upper) * EyeKernel()


class SumOfKernels(Kernel):
    """SumOfKernels.scala:15-65: hyperparameters are concatenated left to right."""

    def __init__(self, kernel1: Kernel, kernel2: Kernel):
        self.kernel1, self.kernel2 = kernel1, kernel2

    def getHyperparameters(self):
        return np.concatenate([self.kernel1.getHyperparameters(), self.kernel2.getHyperparameters()])
    def setHyperparameters(self, value):
        value = np.asarray(value, dtype=np.float64)
        n1 = self.kernel1.numberOfHyperparameters()
        self.kernel1.setHyperparameters(value[:n1])
        self.kernel2.setHyperparameters(value[n1:])
        return self
    def numberOfHyperparameters(self):
        return self.kernel1.numberOfHyperparameters() + self.kernel2.numberOfHyperparameters()
    def hyperparameterBoundaries(self):
        l1, u1 = self.kernel1.hyperparameterBoundaries()
        l2, u2 = self.kernel2.hyperparameterBoundaries()
        return np.concatenate([l1, l2]), np.concatenate([u1, u2])
    def flatten(self, scale=1.0): return self.kernel1.flatten(scale) + self.kernel2.flatten(scale)
    def hyper_descriptors(self, scale=1.0, term_offset=0):
        n1 = len(self.kernel1.flatten(scale))
        return (self.kernel1.hyper_descriptors(scale, term_offset)
                + self.kernel2.hyper_descriptors(scale, term_offset + n1))
    def _children(self): return [self.kernel1, self.kernel2]
    def __str__(self): return " + ".join(s for s in (str(self.kernel1), str(self.kernel2)) if len(s) > 0)
