"""Small host-side helpers of the reference's examples."""
from __future__ import annotations

import numpy as np

from .engine import ProjectedProcessEngine, is_cuda_tensor


def scale(X, process_group=None):
    """commons/util/Scaling.scala:10-25 (used by regression/examples/Airfoil.scala:26-32 and
    classification/examples/MNIST.scala:42-45): subtract the column mean, divide by the POPULATION standard deviation
    (variance / n); a zero variance counts as 1.

    A host array is scaled on the host (numpy, float64).  A CUDA tensor X (n x d) is scaled on its GPU and never leaves
    it: two fixed-order column-sum passes give the mean and the variance (`moments`), and the result is a CUDA float64
    tensor on X's device whose every element is the host formula's on that mean and standard deviation.  With a
    torch.distributed process_group, each rank passes its shard and gets its own rows back scaled with the mean and
    standard deviation of the concatenation of the shards (`distributed.scale`)."""
    if process_group is not None:
        from .distributed import scale as group_scale
        return group_scale(X, process_group)
    if is_cuda_tensor(X):
        return device_scale(X)
    X = np.asarray(X, dtype=np.float64)
    n = float(len(X))
    mean = X.sum(axis=0) / n
    centered = X - mean
    variance = (centered * centered).sum(axis=0) / n
    return centered / np.sqrt(np.where(variance > 0.0, variance, 1.0))


def moments(eng, X, total=lambda v: v):
    """The mean and the standard deviation `scale` uses, for the rows of the CUDA tensor X on eng's device: mean = S / n
    from the column sums S, variance = Q / n from the sums Q of the squares centred on that mean, a variance that is not
    > 0 taken as 1, sd = sqrt(variance) on the host in fp64.  total(v) sums a host vector over the ranks of a process
    group ([S; n], then Q); without one it is the identity.  Returns (mean, sd) as host arrays of d values."""
    s = total(np.append(eng.column_sums(X), float(len(X))))
    n = s[-1]
    mean = s[:-1] / n
    variance = total(eng.column_sums(X, mean)) / n
    return mean, np.sqrt(np.where(variance > 0.0, variance, 1.0))


def device_scale(X):
    """`scale` of a CUDA tensor X (n x d) on its GPU: a CUDA float64 tensor on X's device (0 x d for an empty X)."""
    if X.ndim != 2:
        raise ValueError("scale: X must be n x d")
    if len(X) == 0:
        import torch
        return torch.empty(tuple(X.shape), dtype=torch.float64, device=X.device)
    eng = ProjectedProcessEngine.acquire(X.device.index)
    try:
        mean, sd = moments(eng, X)
        return eng.scale_apply(X, mean, sd)
    finally:
        eng.release()


_M64 = (1 << 64) - 1


def _mix(z):
    """SplitMix64's finaliser on Python ints (scalar) or uint64 arrays."""
    if isinstance(z, np.ndarray):
        with np.errstate(over="ignore"):
            z = z + np.uint64(0x9E3779B97F4A7C15)
            z = (z ^ (z >> np.uint64(30))) * np.uint64(0xBF58476D1CE4E5B9)
            z = (z ^ (z >> np.uint64(27))) * np.uint64(0x94D049BB133111EB)
        return z ^ (z >> np.uint64(31))
    z = (z + 0x9E3779B97F4A7C15) & _M64
    z = ((z ^ (z >> 30)) * 0xBF58476D1CE4E5B9) & _M64
    z = ((z ^ (z >> 27)) * 0x94D049BB133111EB) & _M64
    return z ^ (z >> 31)


def uniform(seed: int, stream: int, i) -> np.ndarray:
    """The counter-based generator the library's K-means draws from (DESIGN.md 4.7):
    u(seed, stream, i) = (mix(mix(mix(seed) ^ stream) ^ i) >> 11) * 2^-53 in [0, 1), for an integer array i."""
    base = _mix(_mix(int(seed) & _M64) ^ int(stream))
    z = _mix(np.uint64(base) ^ np.asarray(i, dtype=np.uint64))
    return (z >> np.uint64(11)).astype(np.float64) * 2.0 ** -53


def kfold_assignment(n: int, num_folds: int, seed: int, offset: int = 0) -> np.ndarray:
    """CrossValidator's default split: point i goes to fold floor(u(seed, 200, i) * numFolds) (int32), for the n points
    i in [offset, offset + n) (a rank's shard of a data-parallel selection numbers its rows globally)."""
    i = np.arange(int(offset), int(offset) + int(n))
    return np.floor(uniform(seed, 200, i) * int(num_folds)).astype(np.int32)


def train_validation_assignment(n: int, train_ratio: float, seed: int, offset: int = 0) -> np.ndarray:
    """TrainValidationSplit's default split: row i trains iff u(seed, 201, i) < trainRatio (bool mask), for the n rows
    i in [offset, offset + n)."""
    return uniform(seed, 201, np.arange(int(offset), int(offset) + int(n))) < float(train_ratio)
