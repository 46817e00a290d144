"""CPU restatement (test infrastructure) of the K-means the reference's KMeansActiveSetProvider calls
(commons/ActiveSetProvider.scala:22-46: `new KMeans().setK(activeSetSize).setSeed(seed).setMaxIter(maxIter)`, Spark 3.1
defaults otherwise: initMode "k-means||", initSteps 2, tol 1e-4, Euclidean distance, unit weights).

Spark's source is not part of this project: the steps are restated from Spark 3.1's
`mllib/clustering/KMeans.scala` (`initKMeansParallel`, `runAlgorithmWithWeight`) and `LocalKMeans.scala`
(`kMeansPlusPlus`) from memory; DESIGN.md 4.7 lists them.  Spark's XORShift / java.util.Random streams depend on the
partitioning and are not reproduced: every draw comes from the counter-based generator `u` below, which the library
(csrc/kmeans.cu) shares, so that this restatement replays every draw.

"nearest" is the smallest squared Euclidean distance, ties to the lowest centre index.  Distances are summed over the
coordinates in order; running sums the algorithm compares are sequential (np.cumsum), as on Spark's driver.
"""
from __future__ import annotations

import numpy as np

_M64 = (1 << 64) - 1


def _mix(z: int) -> int:
    z = (z + 0x9E3779B97F4A7C15) & _M64
    z = ((z ^ (z >> 30)) * 0xBF58476D1CE4E5B9) & _M64
    z = ((z ^ (z >> 27)) * 0x94D049BB133111EB) & _M64
    return z ^ (z >> 31)


def _mix_vec(z: np.ndarray) -> np.ndarray:
    with np.errstate(over="ignore"):
        z = z + np.uint64(0x9E3779B97F4A7C15)
        z = (z ^ (z >> np.uint64(30))) * np.uint64(0xBF58476D1CE4E5B9)
        z = (z ^ (z >> np.uint64(27))) * np.uint64(0x94D049BB133111EB)
    return z ^ (z >> np.uint64(31))


def u(seed: int, stream: int, i) -> np.ndarray | float:
    """u(seed, stream, i) = (mix(mix(mix(seed) ^ stream) ^ i) >> 11) * 2^-53, in [0, 1).  i: int or integer array."""
    base = _mix(_mix(int(seed) & _M64) ^ stream)
    if np.isscalar(i):
        return (_mix(base ^ int(i)) >> 11) * 2.0 ** -53
    z = _mix_vec(np.uint64(base) ^ np.asarray(i, dtype=np.uint64))
    return (z >> np.uint64(11)).astype(np.float64) * 2.0 ** -53


def sq_dist(P: np.ndarray, c: np.ndarray) -> np.ndarray:
    """|p - c|^2 for every row p of P, summed over the coordinates in order."""
    acc = np.zeros(len(P))
    for j in range(P.shape[1]):
        df = P[:, j] - c[j]
        acc = acc + df * df
    return acc


def assign(P: np.ndarray, C: np.ndarray, block: int = 4096):
    """(labels, min d^2, margin): nearest centre of every row of P (ties -> lowest index); margin = second smallest d^2
    minus the smallest (inf with one centre)."""
    n = len(P)
    labels = np.empty(n, dtype=np.int64)
    best = np.empty(n)
    margin = np.full(n, np.inf)
    for s in range(0, n, block):
        Pb = P[s:s + block]
        D = np.stack([sq_dist(Pb, c) for c in C], axis=1)
        lab = np.argmin(D, axis=1)                       # first minimum: the lowest index wins ties
        labels[s:s + block] = lab
        best[s:s + block] = D[np.arange(len(Pb)), lab]
        if len(C) > 1:
            part = np.partition(D, 1, axis=1)
            margin[s:s + block] = part[:, 1] - part[:, 0]
    return labels, best, margin


def kmeans_parallel_candidates(X: np.ndarray, k: int, seed: int):
    """KMeans.initKMeansParallel up to the distinct candidates: first centre, two k-means|| steps, distinct rows in first-
    occurrence order.  Returns (candidates, chosen indices in order incl. the first centre)."""
    n = len(X)
    i0 = min(n - 1, int(np.floor(u(seed, 0, 0) * n)))            # step 1: c0 = X[floor(u(seed, 0, 0) n)]
    cost = np.full(n, np.inf)
    new = [i0]
    chosen = [i0]
    idx = np.arange(n)
    for step in range(2):                                         # step 2: initSteps = 2
        for c in new:
            cost = np.minimum(cost, sq_dist(X, X[c]))
        S = float(np.sum(cost))
        with np.errstate(invalid="ignore", divide="ignore"):
            thr = (2.0 * k * cost) / S
        pick = u(seed, 1 + step, idx) < thr                      # a NaN threshold chooses nothing
        new = list(idx[pick])
        chosen += new
    seen, cand = set(), []
    for i in chosen:                                              # step 3: distinct, first occurrence kept
        key = tuple(float(v) + 0.0 for v in X[i])
        if key not in seen:
            seen.add(key)
            cand.append(X[i])
    return np.array(cand, dtype=np.float64).reshape(-1, X.shape[1]), chosen


def _walk(v: np.ndarray, r: float) -> int:
    """`while (j < C && cum < r) { cum += v(j); j += 1 }` and take max(j - 1, 0)."""
    if not (r > 0.0):
        return 0
    cum = np.cumsum(v)
    hit = np.nonzero(cum >= r)[0]
    return int(hit[0]) if len(hit) else len(v) - 1


def local_kmeans_pp(cand: np.ndarray, w: np.ndarray, k: int, seed: int, max_iterations: int = 30) -> np.ndarray:
    """LocalKMeans.kMeansPlusPlus(candidates, weights, k, 30): weighted k-means++ seeding, then up to 30 weighted Lloyd
    iterations over the candidates.  Draws: stream 100 (seeding, counter = centre index), stream 101 (empty clusters)."""
    Cn, d = cand.shape
    w = np.asarray(w, dtype=np.float64)
    centres = np.empty((k, d))
    cost = np.full(Cn, np.inf)
    for i in range(k):
        v = w if i == 0 else w * cost
        r = u(seed, 100, i) * float(np.cumsum(v)[-1])            # pickWeighted / r = u * sum_j w_j cost_j
        p = _walk(v, r)
        centres[i] = cand[p]
        cost = np.minimum(cost, sq_dist(cand, cand[p]))
    old = np.full(Cn, -1)
    draws = 0
    for _ in range(max_iterations):
        lab, _, _ = assign(cand, centres)
        moved = bool(np.any(lab != old))                          # the first pass counts as a change
        old = lab
        sums = np.zeros((k, d))
        cnt = np.zeros(k)
        np.add.at(sums, lab, w[:, None] * cand)                   # axpy(w_i, p_i, sums(index)), in point order
        np.add.at(cnt, lab, w)
        for j in range(k):
            if cnt[j] == 0.0:
                p = min(Cn - 1, int(np.floor(u(seed, 101, draws) * Cn)))
                draws += 1
                centres[j] = cand[p]
            else:
                centres[j] = sums[j] * (1.0 / cnt[j])
        if not moved:
            break
    return centres


def init_centres(X: np.ndarray, k: int, seed: int) -> np.ndarray:
    """Steps 1-4: the k-means|| initial centres (k_out <= k rows)."""
    cand, _ = kmeans_parallel_candidates(X, k, seed)
    if len(cand) <= k:
        return cand
    lab, _, _ = assign(X, cand)
    w = np.bincount(lab, minlength=len(cand)).astype(np.float64)
    return local_kmeans_pp(cand, w, k, seed, 30)


def lloyd(X: np.ndarray, centres: np.ndarray, max_iter: int, tol: float):
    """KMeans.runAlgorithmWithWeight: (centres, labels, iterations, cost).  Labels and cost are those of the last
    assignment pass (against the centres before the last update, as trainingCost); max_iter = 0 runs one pass."""
    C = np.array(centres, dtype=np.float64, copy=True)
    k, d = C.shape
    iteration, converged = 0, False
    while True:
        lab, best, _ = assign(X, C)
        cost = float(np.sum(best))
        if max_iter == 0:
            break
        sums = np.zeros((k, d))
        np.add.at(sums, lab, X)
        cnt = np.bincount(lab, minlength=k).astype(np.float64)
        converged = True
        for j in range(k):
            if cnt[j] == 0.0:                                     # an empty cluster keeps its centre
                continue
            nc = sums[j] * (1.0 / cnt[j])
            if not (float(np.sum((nc - C[j]) ** 2)) <= tol * tol):
                converged = False
            C[j] = nc
        iteration += 1
        if iteration >= max_iter or converged:
            break
    return C, lab, iteration, cost


def kmeans(X, k: int, max_iter: int = 20, tol: float = 1e-4, seed: int = 0, init_centers=None):
    """The whole of Spark 3.1 MLlib KMeans.fit with the reference's settings: (centres, labels, iterations, cost)."""
    X = np.asarray(X, dtype=np.float64)
    C0 = init_centres(X, k, seed) if init_centers is None else np.asarray(init_centers, dtype=np.float64)
    return lloyd(X, C0, max_iter, tol)
