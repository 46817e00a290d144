"""Projected-process statistics, m x m tail, predictor, expert grouping
(TEST INFRASTRUCTURE -- see oracle/__init__.py).

Follows `commons/ProjectedGaussianProcessHelper.scala` (PGPH) and
`commons/GaussianProcessCommons.scala` (GPC) of the reference.
"""
from __future__ import annotations

import numpy as np
import scipy.linalg as sla

from .kernels import Kernel, EyeKernel, const


class NotPositiveDefiniteException(Exception):
    """PGPH:9-11."""

    def __init__(self):
        super().__init__("Some matrix which is supposed to be positive definite is not. This probably "
                         "happened due to `sigma2` parameter being too small. Try to gradually increase it.")


def get_kernel(user_kernel_factory, sigma2: float):
    """GPC:18  `() => $(kernel)() + $(sigma2).const * new EyeKernel`."""
    return lambda: user_kernel_factory() + const(sigma2) * EyeKernel()


def group_for_experts(n_points: int, dataset_size_for_expert: int):
    """GPC:26-31.  E = Math.round(N / n_e) (round-half-up on a positive double); point i (zipWithIndex
    order) goes to expert i % E.  Returns the list of index arrays, one per expert, each in ascending
    point order (what `groupByKey` yields for an ordered input partition; order inside an expert does
    not affect G or b, which are sums over points)."""
    n_experts = int(np.floor(n_points / dataset_size_for_expert + 0.5))
    if n_experts <= 0:
        raise ZeroDivisionError("numberOfExperts == 0 (N < n_e/2): the reference fails with / by zero")
    return [np.arange(e, n_points, n_experts) for e in range(n_experts)]


def get_expert_labels_and_kernels(X, y, kernel_factory, dataset_size_for_expert: int):
    """GPC:33-38: per expert (BDV(labels), getKernel().setTrainingVectors(X_e))."""
    X = np.asarray(X, dtype=np.float64)
    y = np.asarray(y, dtype=np.float64)
    return [(y[idx], kernel_factory().set_training_vectors(X[idx]))
            for idx in group_for_experts(len(X), dataset_size_for_expert)]


def get_matrix_kmn_knm_and_vector_kmny(expert_labels_and_kernels, active_set):
    """PGPH:20-36 -- THE hot path.  For every expert (y_e, k_e): K_mn = k_e.crossKernel(activeSet)
    (m x n_e), G += K_mn K_mn^T (full dgemm, PGPH:28), b += K_mn y_e (PGPH:29); the treeAggregate
    combOp is a plain sum (PGPH:31-35)."""
    active_set = np.asarray(active_set, dtype=np.float64)
    m = len(active_set)
    G = np.zeros((m, m))
    b = np.zeros(m)
    for y, k in expert_labels_and_kernels:
        kmn = k.cross_kernel(active_set)
        G += kmn @ kmn.T
        b += kmn @ y
    return G, b


def assert_sym_positive_definite(matrix: np.ndarray):
    """PGPH:62-65: throws iff any eigSym eigenvalue < 0 (semi-definite passes)."""
    ev = sla.eigvalsh(matrix, driver="evd")
    if np.any(ev < 0.0):
        raise NotPositiveDefiniteException()


def get_magic_vector(kernel: Kernel, matrix_kmn_knm: np.ndarray, vector_kmny: np.ndarray):
    """PGPH:49-60.  `kernel` has the optimal hyperparameters and the active set as training vectors.
    K_mm = kernel.trainingKernel() INCLUDES the Eye terms on its diagonal; whiteNoiseVar is the sum of
    all Eye coefficients.  Returns (magicVector, magicMatrix)."""
    train_kernel = kernel.training_kernel()
    pdm = kernel.white_noise_var * train_kernel          # sigma^2 K_mm           PGPH:55
    pdm = pdm + matrix_kmn_knm                           # + K_mn K_nm            PGPH:56
    assert_sym_positive_definite(pdm)                    #                        PGPH:58
    lu, piv = sla.lu_factor(pdm)                         # `\` = dgesv            PGPH:59
    magic_vector = sla.lu_solve((lu, piv), vector_kmny)
    magic_matrix = sla.inv(pdm) * kernel.white_noise_var - sla.inv(train_kernel)   # dgetrf+dgetri x2
    return magic_vector, magic_matrix


def tail_errors(kernel: Kernel, matrix_kmn_knm: np.ndarray, vector_kmny: np.ndarray, magic_vector: np.ndarray,
                magic_matrix: np.ndarray) -> dict:
    """How far a computed pair (v, M) is from `get_magic_vector`'s, in units of the fp64 unit roundoff u = 2^-53.
    `kernel` has the active set as training vectors; A0 = whiteNoiseVar K0 + G is built here in fp64.
      omega : componentwise backward error of v, max_i |A0 v - b|_i / (|A0| |v| + |b|)_i, over u;
      fwd_v : |v - v0|_inf / |v0|_inf over kappa_inf(A0) u, v0 the LU solution;
      fwd_M : max |M - M0| over u (wn kappa_inf(A0) max|inv A0| + kappa_inf(K0) max|inv K0|),
              M0 = wn inv(A0) - inv(K0).
    A backward-stable tail keeps each of them at a small multiple of 1 whatever the conditioning."""
    u = np.finfo(np.float64).eps / 2
    K0 = kernel.training_kernel()
    wn = kernel.white_noise_var
    A0 = wn * K0 + matrix_kmn_knm
    b = np.asarray(vector_kmny, dtype=np.float64)
    v = np.asarray(magic_vector, dtype=np.float64)
    M = np.asarray(magic_matrix, dtype=np.float64)
    r = np.abs(A0 @ v - b)
    den = np.abs(A0) @ np.abs(v) + np.abs(b)
    with np.errstate(divide="ignore", invalid="ignore"):
        omega = float(np.max(np.where(r == 0, 0.0, r / den)))      # r > 0 over den = 0 counts as infinite
    v0 = sla.lu_solve(sla.lu_factor(A0), b)
    inv_a, inv_k = sla.inv(A0), sla.inv(K0)
    kappa_a = np.linalg.norm(A0, np.inf) * np.linalg.norm(inv_a, np.inf)
    kappa_k = np.linalg.norm(K0, np.inf) * np.linalg.norm(inv_k, np.inf)
    v_scale = max(float(np.max(np.abs(v0))), np.finfo(np.float64).tiny)
    M0 = inv_a * wn - inv_k
    m_scale = u * (wn * kappa_a * np.max(np.abs(inv_a)) + kappa_k * np.max(np.abs(inv_k)))
    return {"omega": omega / u,
            "fwd_v": float(np.max(np.abs(v - v0))) / v_scale / (kappa_a * u),
            "fwd_M": float(np.max(np.abs(M - M0))) / m_scale,
            "kappa_A": float(kappa_a), "kappa_K": float(kappa_k)}


class GaussianProjectedProcessRawPredictor:
    """GPC:118-126."""

    def __init__(self, magic_vector, magic_matrix, kernel: Kernel):
        self.magic_vector, self.magic_matrix, self.kernel = magic_vector, magic_matrix, kernel

    def predict(self, features):
        """GPC:121-125 for one vector: (mean, variance)."""
        cross = self.kernel.cross_kernel_vec(features)
        self_k = self.kernel.self_kernel(features)
        return float(cross @ self.magic_vector), float(self_k + cross @ self.magic_matrix @ cross)

    def predict_many(self, X):
        """Row-wise `predict` for a block of test vectors (same arithmetic, vectorised)."""
        cross = self.kernel.cross_kernel(np.asarray(X, dtype=np.float64))        # T x m
        self_k = self.kernel.self_kernel(None)
        mean = cross @ self.magic_vector
        var = self_k + np.einsum("ti,ij,tj->t", cross, self.magic_matrix, cross)
        return mean, var


def projected_process(expert_labels_and_kernels, active_set, kernel_factory, optimal_hyperparameters):
    """GPC:40-59 with the active set passed in explicitly (the provider's sampling is unpinned)."""
    for _, k in expert_labels_and_kernels:               # GPR:50
        k.set_hyperparameters(optimal_hyperparameters)
    G, b = get_matrix_kmn_knm_and_vector_kmny(expert_labels_and_kernels, active_set)
    optimal_kernel = kernel_factory().set_hyperparameters(optimal_hyperparameters) \
                                     .set_training_vectors(active_set)            # GPC:52
    mv, mm = get_magic_vector(optimal_kernel, G, b)
    return GaussianProjectedProcessRawPredictor(mv, mm, optimal_kernel), G, b
