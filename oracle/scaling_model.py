"""The device rule of feature standardisation (TEST INFRASTRUCTURE -- see oracle/__init__.py).

`commons/util/Scaling.scala:10-25` with exactly rounded sums: the column sums S by `math.fsum`, mean = S / n, the
reference formula's centred squares (x - mean)^2 (one fp64 rounding for the subtraction, one for the square) summed by
`math.fsum`, variance = Q / n, a variance that is not > 0 taken as 1, and (x - mean) / sqrt(variance).

`sum_bound` is the error bound of the library's fixed-order sum (csrc/scale.cu): rows in blocks of ROWS_PER_BLOCK, one
fp64 partial per block and column (each thread sums its rows of the block in order, its lane sums are then added in
lane order), and the partials added in block order.  A term passes through at most (rows per block / L - 1) + (L - 1)
+ (blocks - 1) < rows per block + blocks - 1 roundings for any L lanes, so the sum is within
(rows per block + blocks) 2^-53 sum |terms| of the exact sum.
"""
import math

import numpy as np

ROWS_PER_BLOCK = 2048      # kScaleRows, csrc/sgp_internal.h
U = 2.0 ** -53


def exact_sums(T) -> np.ndarray:
    """math.fsum of every column of T (n x d): the exact sum, rounded once."""
    T = np.asarray(T, dtype=np.float64)
    return np.array([math.fsum(T[:, k]) for k in range(T.shape[1])])


def centred_squares(X, center) -> np.ndarray:
    """The terms (x_ik - c_k)^2 of the variance as the reference formula rounds them: x converted exactly to fp64, then
    one rounding for the subtraction and one for the square."""
    t = np.asarray(X, dtype=np.float64) - np.asarray(center, dtype=np.float64)
    return t * t


def moments(X):
    """(mean, sd) of the rule: exact sums, the reference's formula."""
    X = np.asarray(X, dtype=np.float64)
    n = float(len(X))
    mean = exact_sums(X) / n
    variance = exact_sums(centred_squares(X, mean)) / n
    return mean, np.sqrt(np.where(variance > 0.0, variance, 1.0))


def scale(X) -> np.ndarray:
    """Scaling.scale by the rule: (x - mean) / sd, subtraction then division, each rounded once."""
    mean, sd = moments(X)
    return (np.asarray(X, dtype=np.float64) - mean) / sd


def blocks(n: int) -> int:
    return -(-int(n) // ROWS_PER_BLOCK)


def sum_bound(n: int, abs_sums) -> np.ndarray:
    """The largest distance of the library's sum of n terms per column from the exact sum, given sum |terms| per
    column."""
    return (ROWS_PER_BLOCK + blocks(n)) * U * np.asarray(abs_sums, dtype=np.float64)
