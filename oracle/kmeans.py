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

Every step that computes (nearest centres, the running k-means|| cost, the sums the algorithm branches on, the k-means++
pick, the per-cluster sums, the moved test) goes through an arithmetic object, `Fp64` by default: the restatement's own
fp64 arithmetic.  oracle/kmeans_model.py supplies the library's fp32 arithmetic to the same algorithm.
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


class Fp64:
    """The restatement's arithmetic: fp64 distances summed over the coordinates in order, NumPy sums, sequential walks."""

    def start(self, X: np.ndarray) -> None:
        """Called once with all the points before the first step."""

    def nearest(self, P: np.ndarray, C: np.ndarray):
        """(labels, min d^2) of every row of P over the centres C, ties to the lowest index."""
        lab, best, _ = assign(P, C)
        return lab, best

    def running_min(self, cost: np.ndarray, P: np.ndarray, new: np.ndarray) -> np.ndarray:
        """The k-means|| cost: min(cost_i, d^2 to each new centre)."""
        for c in new:
            cost = np.minimum(cost, sq_dist(P, c))
        return cost

    def total(self, v: np.ndarray) -> float:
        """The sum of a point-sized vector (the k-means|| S, the training cost)."""
        return float(np.sum(v))

    def pick(self, v: np.ndarray, seed: int, i: int) -> int:
        """k-means++ centre i: r = u(seed, 100, i) * sum(v), then the walk."""
        return _walk(v, u(seed, 100, i) * float(np.cumsum(v)[-1]))

    def changed(self, lab: np.ndarray, old: np.ndarray, it: int) -> bool:
        """Whether a local Lloyd pass moved a label (the first pass, against -1, always does)."""
        return bool(np.any(lab != old))

    def draws_at(self, draws: int) -> int:
        """The empty-cluster draw counter at the start of a local Lloyd iteration (it persists)."""
        return draws

    def cluster_sums(self, X: np.ndarray, lab: np.ndarray, k: int) -> np.ndarray:
        """Per-cluster coordinate sums, in point order."""
        sums = np.zeros((k, X.shape[1]))
        np.add.at(sums, lab, X)
        return sums

    def moved(self, nc: np.ndarray, c: np.ndarray, tol: float) -> bool:
        """Whether a cluster's move |nc - c|^2 is above tol^2."""
        return not (float(np.sum((nc - c) ** 2)) <= tol * tol)

    def note(self, key: str, value) -> None:
        """Instrumentation: what the run reached (candidate count, iterations, draws, ...)."""


FP64 = Fp64()


def kmeans_parallel_candidates(X: np.ndarray, k: int, seed: int, ar: Fp64 = FP64):
    """KMeans.initKMeansParallel up to the distinct candidates: first centre, two k-means|| steps, distinct rows in first-
    occurrence order.  Returns (candidates, chosen indices in order incl. the first centre)."""
    n = len(X)
    i0 = min(n - 1, int(np.floor(u(seed, 0, 0) * n)))            # step 1: c0 = X[floor(u(seed, 0, 0) n)]
    cost = np.full(n, np.inf)
    new = [i0]
    chosen = [i0]
    idx = np.arange(n)
    for step in range(2):                                         # step 2: initSteps = 2
        if new:
            cost = ar.running_min(cost, X, X[new])
        S = ar.total(cost)
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


def local_kmeans_pp(cand: np.ndarray, w: np.ndarray, k: int, seed: int, max_iterations: int = 30,
                    ar: Fp64 = FP64) -> np.ndarray:
    """LocalKMeans.kMeansPlusPlus(candidates, weights, k, 30): weighted k-means++ seeding, then up to 30 weighted Lloyd
    iterations over the candidates.  Draws: stream 100 (seeding, counter = centre index), stream 101 (empty clusters)."""
    Cn, d = cand.shape
    w = np.asarray(w, dtype=np.float64)
    centres = np.empty((k, d))
    cost = np.full(Cn, np.inf)
    for i in range(k):
        v = w if i == 0 else w * cost
        p = ar.pick(v, seed, i)                                   # pickWeighted / r = u * sum_j w_j cost_j
        centres[i] = cand[p]
        cost = np.minimum(cost, sq_dist(cand, cand[p]))
    old = np.full(Cn, -1)
    draws = 0
    its = 0
    for it in range(max_iterations):
        its += 1
        draws = ar.draws_at(draws)
        lab, _ = ar.nearest(cand, centres)
        moved = ar.changed(lab, old, it)                          # the first pass counts as a change
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
    ar.note("local_iterations", its)
    ar.note("draws101", draws)
    return centres


def init_centres(X: np.ndarray, k: int, seed: int, ar: Fp64 = FP64) -> np.ndarray:
    """Steps 1-4: the k-means|| initial centres (k_out <= k rows)."""
    cand, _ = kmeans_parallel_candidates(X, k, seed, ar)
    ar.note("C", len(cand))
    if len(cand) <= k:
        return cand
    lab, _ = ar.nearest(X, cand)
    w = np.bincount(lab, minlength=len(cand)).astype(np.float64)
    return local_kmeans_pp(cand, w, k, seed, 30, ar)


def lloyd(X: np.ndarray, centres: np.ndarray, max_iter: int, tol: float, ar: Fp64 = FP64):
    """KMeans.runAlgorithmWithWeight: (centres, labels, iterations, cost).  Labels and cost are those of the last
    assignment pass (against the centres before the last update, as trainingCost); max_iter = 0 runs one pass."""
    C = np.array(centres, dtype=np.float64, copy=True)
    k, d = C.shape
    iteration, converged = 0, False
    while True:
        lab, best = ar.nearest(X, C)
        cost = ar.total(best)
        if max_iter == 0:
            break
        sums = ar.cluster_sums(X, lab, k)
        cnt = np.bincount(lab, minlength=k).astype(np.float64)
        converged = True
        for j in range(k):
            if cnt[j] == 0.0:                                     # an empty cluster keeps its centre
                ar.note("empty", 1)
                continue
            nc = sums[j] * (1.0 / cnt[j])
            if ar.moved(nc, C[j], tol):
                converged = False
            C[j] = nc
        iteration += 1
        ar.note("lloyd_iteration", iteration)
        if iteration >= max_iter or converged:
            break
    return C, lab, iteration, cost


def kmeans(X, k: int, max_iter: int = 20, tol: float = 1e-4, seed: int = 0, init_centers=None, ar: Fp64 = FP64):
    """The whole of Spark 3.1 MLlib KMeans.fit with the reference's settings: (centres, labels, iterations, cost)."""
    ar.start(X)
    X = np.asarray(X, dtype=np.float64)
    C0 = init_centres(X, k, seed, ar) if init_centers is None else np.asarray(init_centers, dtype=np.float64)
    return lloyd(X, C0, max_iter, tol, ar)
