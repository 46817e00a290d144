"""CPU restatement (test infrastructure) of commons/ActiveSetProvider.scala:58-139, GreedilyOptimizingActiveSetProvider
("Fast Forward Selection to Speed Up Sparse Gaussian Process Regression", Seeger et al. 2003, as the reference codes it).

Parity notes (SURVEY.md 8c): the FIRST point comes from Spark's `takeSample(…, 1, seed)` (ASP:70), whose RNG stream is
unpinned -- here it is an explicit index.  Everything after it is deterministic arithmetic and is restated verbatim,
including the quirks:
  * `getNext` is handed `kernelInstance.whiteNoiseVar` as its `sigma2` (ASP:76): with the default kernel that is
    1 + sigma2, not the sigma2 parameter;
  * per expert the candidates are folded left to right with `(max(delta, oldMax), if (oldMax > delta) oldIdx else i)`
    (ASP:108-127): on ties the LATER point wins, and one NaN delta poisons the expert's maximum (math.max(NaN, x) = NaN),
    after which the expert is dropped by `.filter(!_._1.isNaN)` (ASP:131);
  * across experts `max()` keeps the FIRST of equal scores (Ordering.max: `if (gteq(x, y)) x else y`);
  * points already in the active set are not excluded.
"""
from __future__ import annotations

import math
from typing import NamedTuple

import numpy as np
import scipy.linalg as sla

from .ppa import assert_sym_positive_definite

DOUBLE_MIN_VALUE = -1.7976931348623157e308


def _delta_formula(p, q, mu, y, kii, sigma2):
    """ASP:114-124 from the quadratic forms p_i = k_i' inv(K_mm) k_i, q_i = k_i' inv(A) k_i, mu_i = k_i' magicVector."""
    with np.errstate(all="ignore"):
        sigma = math.sqrt(sigma2)
        li = np.sqrt(kii - p)
        ksi = 1.0 / ((sigma / li) ** 2 + 1.0 - q)
        kappa = ksi * (1.0 + 2.0 * (sigma / li) ** 2)
        return -np.log(sigma / li) - (np.log(ksi) + ksi * (1.0 - kappa) / sigma2 * (y - mu) ** 2 - kappa + 2.0) / 2.0


def _fold_expert(deltas: np.ndarray):
    """ASP:108-127: returns (maxDelta, maxIndex) of one expert's candidates."""
    old_max, old_idx = -1.7976931348623157e308, -1          # Double.MinValue
    for i, delta in enumerate(deltas):
        new_idx = old_idx if old_max > delta else i         # a NaN on either side compares false -> i
        old_max = float("nan") if (math.isnan(delta) or math.isnan(old_max)) else max(delta, old_max)   # math.max
        old_idx = new_idx
    return old_max, old_idx


def candidate_deltas(cross: np.ndarray, y: np.ndarray, kii: np.ndarray, k_inv: np.ndarray, pdm_inv: np.ndarray,
                     magic_vector: np.ndarray, sigma2: float) -> np.ndarray:
    """ASP:109-124 for all points of an expert at once.  cross: m x n_e (column i = k(activeSet, x_i))."""
    with np.errstate(all="ignore"):
        p = np.einsum("ji,jk,ki->i", cross, k_inv, cross)
        q = np.einsum("ji,jk,ki->i", cross, pdm_inv, cross)
        mu = cross.T @ magic_vector
    return _delta_formula(p, q, mu, y, kii, sigma2)


def get_next(kmm: np.ndarray, experts, active_set: np.ndarray, sigma2: float):
    """ASP:83-137.  experts: list of (y_e, kernel_e with training vectors X_e and hyper-parameters set)."""
    k_inv = np.linalg.inv(kmm)
    crosses = [(y, k.cross_kernel(active_set), k) for y, k in experts]
    g = sum(c @ c.T for _, c, _ in crosses)
    b = sum(c @ y for y, c, _ in crosses)
    pdm = sigma2 * kmm + g
    assert_sym_positive_definite(pdm)
    pdm_inv = np.linalg.inv(pdm)
    magic_vector = np.linalg.solve(pdm, b)
    best = None
    for y, c, k in crosses:
        d = candidate_deltas(c, y, k.training_kernel_diag(), k_inv, pdm_inv, magic_vector, sigma2)
        md, mi = _fold_expert(d)
        if math.isnan(md):
            continue
        if best is None or not (best[0] >= md):              # Ordering.max keeps the earlier of equal scores
            best = (md, k.get_training_vectors()[mi])
    if best is None:
        raise ValueError("empty.max")                        # what RDD.max() throws on an empty RDD
    return best[1]


def greedy_active_set(active_set_size: int, experts, kernel_factory, hyperparameters, first_point) -> np.ndarray:
    """ASP:63-81 with the takeSample'd first point given explicitly."""
    active = np.asarray(first_point, dtype=np.float64).reshape(1, -1)
    theta = np.asarray(hyperparameters, dtype=np.float64)
    while len(active) < active_set_size:
        inst = kernel_factory().set_hyperparameters(theta).set_training_vectors(active)
        nxt = get_next(inst.training_kernel(), experts, active, inst.white_noise_var)
        active = np.vstack([active, nxt])
    return active


class RoundScores(NamedTuple):
    delta: np.ndarray       # [N] ASP:109-124 with the reference's algebra: inv(K_mm), inv(A), A \ b by LU (NaN everywhere
                            #     when K_mm or A is exactly singular)
    delta_chol: np.ndarray  # [N] the same through Cholesky solves (NaN everywhere when A or K_mm does not factor)
    best: np.ndarray        # [E] per-expert fold maximum (NaN: poisoned expert)
    best_idx: np.ndarray    # [E] per-expert fold index, a point index (-1: no candidate above Double.MinValue)
    pick: int               # the selected point; -1 when every expert is poisoned (RDD.max throws empty.max)
    min_eig_a: float        # smallest eigenvalue of A = s2 K_mm + G (the reference throws NotPositiveDefinite when < 0)


def fold_experts(delta: np.ndarray, E: int):
    """ASP:108-135 for every expert at once (point i belongs to expert i % E): returns (best [E], best_idx [E], pick).
    Same results as `_fold_expert` per expert followed by `filter(!isNaN).max()`: within an expert the LATER of equal
    scores wins and one NaN poisons it (its index is then its last point, as the fold leaves it); the FIRST expert with
    the maximal score wins; pick = -1 when every expert is poisoned."""
    delta = np.asarray(delta, dtype=np.float64)
    n = len(delta)
    rows = -(-n // E)
    D = np.full(rows * E, -np.inf)
    D[:n] = delta
    D = D.reshape(rows, E)                                    # D[k, e] = delta[k E + e]
    valid = (np.arange(rows * E) < n).reshape(rows, E)
    nan = np.isnan(D)
    poisoned = nan.any(axis=0)
    Dm = np.where(nan, -np.inf, D)
    best = np.maximum(Dm.max(axis=0), DOUBLE_MIN_VALUE)       # the fold starts from Double.MinValue
    hits = (Dm == best) & valid
    k_last = rows - 1 - np.argmax(hits[::-1], axis=0)
    e = np.arange(E)
    best_idx = np.where(hits.any(axis=0), k_last * E + e, -1)
    last_point = np.where(e < n, ((n - 1 - e) // E) * E + e, -1)
    best_idx = np.where(poisoned, last_point, best_idx)
    best = np.where(poisoned, np.nan, best)
    if poisoned.all():
        return best, best_idx, -1
    e_star = int(np.argmax(np.where(poisoned, -np.inf, best) == np.nanmax(best)))   # the first maximal expert
    return best, best_idx, int(best_idx[e_star])


def round_scores(X, y, active_idx, kernel_factory, theta, E: int, cross=None) -> RoundScores:
    """One round of `getNext` (ASP:83-137) for the active set X[active_idx], vectorised over all N points in fp64.

    The deltas come in two formulations: `delta` with the reference's algebra (explicit inv(K_mm) and inv(A), the magic
    vector by an LU solve) and `delta_chol` through Cholesky factors of K_mm and A; their difference measures how many
    digits the round's conditioning leaves.  O(N r^2) with BLAS-3 only.  `cross` (N x r) is the cross kernel of X
    against the active set when the caller already has it.  The kernel is stationary: every point's diagonal is the
    active points' diagonal."""
    X = np.asarray(X, dtype=np.float64)
    y = np.asarray(y, dtype=np.float64)
    inst = kernel_factory().set_hyperparameters(np.asarray(theta, dtype=np.float64))
    inst.set_training_vectors(X[np.asarray(active_idx, dtype=np.int64)])
    Kc = inst.cross_kernel(X) if cross is None else np.asarray(cross, dtype=np.float64)      # N x r
    kmm = inst.training_kernel()
    kii = float(inst.training_kernel_diag()[0])
    s2 = inst.white_noise_var
    G = Kc.T @ Kc
    b = Kc.T @ y
    pdm = s2 * kmm + G
    min_eig = float(sla.eigvalsh(pdm, driver="evd", check_finite=False)[0])
    try:
        with np.errstate(all="ignore"):
            p = ((Kc @ np.linalg.inv(kmm)) * Kc).sum(axis=1)
            q = ((Kc @ np.linalg.inv(pdm)) * Kc).sum(axis=1)
            mu = Kc @ np.linalg.solve(pdm, b)
    except np.linalg.LinAlgError:                             # breeze throws MatrixSingularException here
        delta = np.full(len(X), np.nan)
    else:
        delta = _delta_formula(p, q, mu, y, kii, s2)
    try:
        Lk = np.linalg.cholesky(kmm)
        La = np.linalg.cholesky(pdm)
    except np.linalg.LinAlgError:
        delta_chol = np.full(len(X), np.nan)
    else:
        with np.errstate(all="ignore"):
            Vk = sla.solve_triangular(Lk, Kc.T, lower=True, check_finite=False)
            Va = sla.solve_triangular(La, Kc.T, lower=True, check_finite=False)
            mv = sla.cho_solve((La, True), b, check_finite=False)
            delta_chol = _delta_formula((Vk * Vk).sum(axis=0), (Va * Va).sum(axis=0), Kc @ mv, y, kii, s2)
    best, best_idx, pick = fold_experts(delta, E)
    return RoundScores(delta, delta_chol, best, best_idx, pick, min_eig)
