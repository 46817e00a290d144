"""The exact arithmetic model of `sgp_kmeans` (csrc/kmeans.cu): the algorithm of oracle/kmeans.py run with the library's
own operations, in the library's order, so that its outputs equal the GPU's bit for bit on any finite data.

`Fp32Model` replaces each place where the fp64 restatement's arithmetic differs from the kernels':
  * origin -- `kmeans_colstats_kernel`'s slices and row lanes (sequential `a += v`, `b = fma(v, v, b)`), the lanes and
    then the slices folded in order, the host's `mean`, `sd` and `o = rint(mean / q) q`, `q = 2^ilogb(sd)`;
  * prescale -- `2^s` with s = 0 while the largest column sd is in [2^-16, 2^16], else the s that brings it into [1, 2),
    refused beyond |s| = 511 or where a column's sum of squares overflows fp64;
  * images -- `fp32((x - o) 2^s)` for points and centres (fp64 arithmetic, one rounding to fp32);
  * distance -- `acc = fmaf(a, a, acc)` over the coordinates in order, `a = fp32(xs - cs)`, returned as fp64 times
    2^-2s; the argmin by strict `<` over the centres in index order from (+inf, 0);
  * fixed-order sums -- `kmeans_sum_kernel` (264 blocks, 256-thread strided sums, a tree, the blocks added in order);
  * the k-means++ pick -- `kmeans_pp_kernel`'s segments, warp scans and walk;
  * the moved test -- per-lane `fma(df, df, .)` over coordinates lane, lane + 32, ..., then the shuffle-down tree;
  * shards -- each rank's fixed-order partial sums added over the ranks (exact at two ranks: one addition each).

fmaf and fma are emulated exactly in NumPy.  The fp32 distance of every (point, centre) pair is screened in fp64 with a
proven bound, and emulated exactly for the centres that can be nearest (`nearest` below).
"""
from __future__ import annotations

import math

import numpy as np

from oracle import kmeans as okm

F32, F64 = np.float32, np.float64
U32, U64 = 2.0 ** -24, 2.0 ** -53
SUM_BLOCKS, SUM_THREADS, PP_THREADS = 264, 256, 1024
M32 = 2.0 ** 128 - 2.0 ** 103                      # the fp32 rounding boundary to +inf
SD_LO, SD_HI = 2.0 ** -16, 2.0 ** 16                # the prescale leaves s = 0 while the largest sd is inside
S_MAX = 511                                          # |s| beyond it: refused (2^s and 2^-2s stay normal fp64 numbers)


# ---- exact fused multiply-adds ----------------------------------------------------------------------------------------
def _two_sum(a, b):
    s = a + b
    bb = s - a
    return s, (a - (s - bb)) + (b - bb)


def fmaf(a, b, c):
    """fp32 fmaf(a, b, c), correctly rounded, elementwise: the fp64 product is exact, TwoSum gives the fp64 sum s and its
    error e, and the one double-rounding case (s exactly an fp32 midpoint with e != 0) is rounded towards e."""
    a64, b64, c64 = (np.asarray(x, F32).astype(F64) for x in (a, b, c))
    with np.errstate(all="ignore"):
        p = a64 * b64
        s, e = _two_sum(p, c64)
        r = s.astype(F32)
        r64 = r.astype(F64)
        dlt = s - r64
        nb = np.nextafter(r, np.where(dlt > 0, F32(np.inf), F32(-np.inf)).astype(F32))
        gap = np.abs(nb.astype(F64) - r64)
        fin = np.isfinite(r)
        mid = fin & (dlt != 0) & (2.0 * np.abs(dlt) == gap) & (e != 0) & (np.sign(e) == np.sign(dlt))
        r = np.where(mid, nb, r)
        back = ~fin & np.isfinite(s) & (np.abs(s) == M32) & (e * np.sign(s) < 0)     # just below the overflow midpoint
        r = np.where(back, (np.sign(s) * np.finfo(F32).max).astype(F32), r)
    return r.astype(F32)


def _split(x):
    t = 134217729.0 * x
    hi = t - (t - x)
    return hi, x - hi


def fma64(a, b, c):
    """fp64 fma(a, b, c), correctly rounded, elementwise (no overflow or underflow in the partial products): the exact
    product as a pair, then the correctly rounded sum of three by rounding to odd (Boldo and Melquiond)."""
    a, b, c = (np.asarray(x, F64) for x in (a, b, c))
    with np.errstate(all="ignore"):
        ph = a * b
        ah, al = _split(a)
        bh, bl = _split(b)
        pl = ((ah * bh - ph) + ah * bl + al * bh) + al * bl
        th, tl = _two_sum(c, pl)
        vh, vl = _two_sum(ph, th)
        w, we = _two_sum(tl, vl)
        even = (np.atleast_1d(w).view(np.int64) & 1) == 0
        w = np.where((we != 0) & even.reshape(np.shape(w)), np.nextafter(w, np.where(we > 0, np.inf, -np.inf)), w)
        return vh + w


# ---- fixed-order reductions --------------------------------------------------------------------------------------------
def fixed_sum(v) -> float:
    """`kmeans_sum_kernel` then the host: 264 blocks of ceil(m / 264), each a 256-thread strided sequential sum and a tree,
    the block results added in order."""
    v = np.asarray(v, F64)
    m = len(v)
    per = -(-m // SUM_BLOCKS)
    pad = np.zeros(SUM_BLOCKS * max(per, 1))
    pad[:m] = v
    blk = pad.reshape(SUM_BLOCKS, max(per, 1))
    lanes = -(-max(per, 1) // SUM_THREADS)
    grid = np.zeros((SUM_BLOCKS, lanes * SUM_THREADS))
    grid[:, :blk.shape[1]] = blk
    grid = grid.reshape(SUM_BLOCKS, lanes, SUM_THREADS)
    sh = np.zeros((SUM_BLOCKS, SUM_THREADS))
    for q in range(lanes):                                       # a += v[i], i = b0 + t, b0 + t + 256, ...
        sh = sh + grid[:, q, :]
    s = SUM_THREADS // 2
    while s > 0:
        sh[:, :s] = sh[:, :s] + sh[:, s:2 * s]
        s //= 2
    t = 0.0
    for x in sh[:, 0]:
        t += x
    return t


def warp_scan(x):
    """Hillis-Steele inclusive scan over the last axis (32 lanes): offsets 1, 2, 4, 8, 16, every lane reading the values
    before the round."""
    x = np.array(x, F64)
    for o in (1, 2, 4, 8, 16):
        x[..., o:] = x[..., o:] + x[..., :-o].copy()
    return x


def pp_scan(v, C, seq_scan=False):
    """`kmeans_pp_kernel`'s scan of one centre's pick: per-thread segment sums (seg = ceil(C / 1024) entries each), the
    Hillis-Steele scan within each warp and over the 32 warp totals.  Returns (pre, total, j0, j1, vv): each thread's
    exclusive prefix, the total, its segment [j0, j1) and its entries vv[thread][q].  seq_scan: a mutant (a sequential
    cumsum over the thread sums)."""
    seg = -(-C // PP_THREADS)
    tid = np.arange(PP_THREADS)
    j0 = np.minimum(C, tid * seg)
    j1 = np.minimum(C, j0 + seg)
    vv = np.zeros(PP_THREADS * seg)
    vv[:C] = v
    vv = vv.reshape(PP_THREADS, seg)
    loc = np.zeros(PP_THREADS)
    for q in range(seg):
        loc = loc + np.where(q < j1 - j0, vv[:, q], 0.0)
    if seq_scan:
        incl = np.cumsum(loc)
        pre = np.concatenate([[0.0], incl[:-1]])
        total = float(incl[-1])
    else:
        incl = warp_scan(loc.reshape(32, 32))
        excl = np.zeros_like(incl)
        excl[:, 1:] = incl[:, :-1]
        wt = warp_scan(incl[:, 31])
        total = float(wt[31])
        pre = (np.concatenate([[0.0], wt[:-1]])[:, None] + excl).reshape(-1)
    return pre, total, j0, j1, vv


def pp_walk(pre, j0, j1, vv, r, C):
    """The walk: every thread adds its entries to its prefix and stops at the first cum >= r; the pick is the smallest
    such index over the threads, C - 1 if there is none, and 0 unless r > 0."""
    if not (r > 0.0):
        return 0
    cum = pre.copy()
    n = j1 - j0
    hit = np.full(PP_THREADS, C)
    done = np.zeros(PP_THREADS, bool)
    for q in range(vv.shape[1]):
        live = (q < n) & ~done
        cum = np.where(live, cum + vv[:, q], cum)
        h = live & (cum >= r)
        hit = np.where(h, j0 + q, hit)
        done |= h
    found = int(hit.min())
    return found if found < C else C - 1


# ---- the origin --------------------------------------------------------------------------------------------------------
def colstats(X):
    """Per column [sum; sum of squares] as `kmeans_colstats_kernel` and the host fold compute them on one rank's rows."""
    X = np.asarray(X)
    n, d = X.shape
    slices = min(SUM_BLOCKS, max(1, -(-n // 1024)))
    rps = -(-n // slices) if n else 0
    a_tot, b_tot = np.zeros(d), np.zeros(d)
    if n == 0:
        return a_tot, b_tot
    X64 = X.astype(F64)
    L = -(-rps // 8)
    pad = np.zeros((slices * rps, d))
    pad[:n] = X64
    blk = pad.reshape(slices, rps, d)
    lanes = np.zeros((slices, L * 8, d))
    lanes[:, :rps] = blk
    lanes = lanes.reshape(slices, L, 8, d)                      # row r0 + rl + 8 q -> [q][rl]
    a = np.zeros((slices, 8, d))
    b = np.zeros((slices, 8, d))
    for q in range(L):
        v = lanes[:, q]
        a = a + v
        b = fma64(v, v, b)
    ta, tb = np.zeros((slices, d)), np.zeros((slices, d))
    for q in range(8):
        ta = ta + a[:, q]
        tb = tb + b[:, q]
    for q in range(slices):
        a_tot = a_tot + ta[q]
        b_tot = b_tot + tb[q]
    return a_tot, b_tot


def origin_and_scale(shards, x0, unrounded=False):
    """(o, s, sd): the host's origin from the ranks' column statistics (summed over the ranks), and the prescale."""
    N = sum(len(X) for X in shards)
    d = len(x0)
    a, b = np.zeros(d), np.zeros(d)
    for X in shards:
        sa, sb = colstats(X)
        a, b = a + sa, b + sb
    o = np.empty(d)
    sds = np.empty(d)
    for j in range(d):
        mean = a[j] / float(N)
        sd = math.sqrt(max(b[j] / float(N) - mean * mean, 0.0))
        sds[j] = sd
        if sd > 0.0 and math.isfinite(sd):
            q = math.ldexp(1.0, math.frexp(sd)[1] - 1)
            o[j] = mean if unrounded else float(np.rint(mean / q)) * q
        else:
            o[j] = x0[j]
    return o, prescale(sds), sds


def prescale(sds) -> int:
    """s of the prescale 2^s from the column sds; OverflowError where the library refuses (a column's sum of squares
    beyond fp64, or |s| > 511)."""
    if not all(math.isfinite(s) for s in sds):
        raise OverflowError("a column's sum of squares is beyond fp64")
    fin = [s for s in sds if s > 0.0]
    if not fin or SD_LO <= max(fin) <= SD_HI:
        return 0
    s = -(math.frexp(max(fin))[1] - 1)
    if abs(s) > S_MAX:
        raise OverflowError("the prescale 2^%d is beyond 2^+-%d" % (s, S_MAX))
    return s


# ---- the model ---------------------------------------------------------------------------------------------------------
class Fp32Model(okm.Fp64):
    """The library's arithmetic for oracle/kmeans.py.  sizes: the ranks' row counts (sharded form), None for one GPU.
    Mutants (CPU tests only): ties_high (ties to the highest index), seq_scan (a sequential cumsum for the k-means++
    scan), prefix_shift (each k-means++ thread walks from the previous thread's exclusive prefix), drop_chunk (the last
    d > 32 chunk dropped), unrounded (o = mean), replace_cost (the k-means|| cost replaced, not min-ed), first_not_moved,
    reset_draws (the stream-101 counter reset every local iteration)."""

    def __init__(self, sizes=None, flips=False, **mutant):
        self.sizes = sizes
        self.want_flips = flips
        self.mut = mutant
        self.info = dict(C=None, seg=None, local_iterations=0, draws101=0, empty=0, ties=0, flips=0, s=0, inf=False,
                         moved_first=None)
        self._moves = []

    # -- set-up
    def start(self, X):
        X = np.asarray(X)
        self.n, self.d = X.shape
        cuts = np.cumsum([0] + list(self.sizes)) if self.sizes else np.array([0, self.n])
        self.cuts = cuts
        shards = [X[cuts[r]:cuts[r + 1]] for r in range(len(cuts) - 1)]
        self.o, self.s, self.sds = origin_and_scale(shards, X[0].astype(F64), self.mut.get("unrounded", False))
        self.scale = math.ldexp(1.0, self.s)
        self.inv2 = math.ldexp(1.0, -2 * self.s)
        d = self.d
        dch = 4 if d <= 4 else 8 if d <= 8 else 16 if d <= 16 else 32
        slices = min(SUM_BLOCKS, max(1, -(-self.n // 1024)))
        self.info.update(s=self.s, sds=self.sds, TC=64 if d <= 16 else 32, DCH=dch, chunks=-(-d // dch),
                         slices=slices, rows_per_slice=-(-self.n // slices),            # kmeans_colstats_kernel
                         sum_per=-(-self.n // SUM_BLOCKS),                              # kmeans_sum_kernel
                         assign_blocks=-(-self.n // 128), last_block_rows=self.n - 128 * (-(-self.n // 128) - 1))

    def note(self, key, value):
        if key == "lloyd_iteration":                              # the largest move the first Lloyd step compared
            if value == 1:
                self.info["moved_first"] = max(self._moves, default=None)
            self._moves = []
        elif key == "empty":
            self.info["empty"] += value
        else:
            self.info[key] = value
        if key == "C":
            self.info["seg"] = -(-value // PP_THREADS)

    def images(self, P):
        with np.errstate(over="ignore"):
            return ((np.asarray(P, F64) - self.o) * self.scale).astype(F32)

    def dims(self):
        d = self.d
        if self.mut.get("drop_chunk") and d > 32:
            return 32 * ((d + 31) // 32 - 1)
        return d

    # -- distances
    def _exact(self, Pi, Ci, i, c):
        acc = np.zeros(len(i), F32)
        for j in range(self.dims()):
            a = Pi[i, j] - Ci[c, j]                              # fp32 subtraction, correctly rounded
            acc = fmaf(a, a, acc)
        return acc

    def _d32(self, P, C):
        """(labels, fp32 minima) over the centres, with the ties and the fp64 minima's disagreements counted."""
        Pi, Ci = self.images(P)[:, :self.dims()], self.images(C)[:, :self.dims()]
        n, k = len(Pi), len(Ci)
        dd = Pi.shape[1]
        P64, C64 = Pi.astype(F64), Ci.astype(F64)
        pn, cn = (P64 * P64).sum(1), (C64 * C64).sum(1)
        lab = np.zeros(n, np.int64)
        best = np.full(n, np.inf, F32)
        step = max(1, 4_000_000 // max(k, 1))
        for s0 in range(0, n, step):
            sl = slice(s0, s0 + step)
            with np.errstate(over="ignore", invalid="ignore"):
                D = pn[sl, None] - 2.0 * (P64[sl] @ C64.T) + cn[None, :]
                E64 = 2.0 * (dd + 8) * U64 * (pn[sl, None] + cn[None, :])
                B = 1.01 * ((dd + 3) * U32 * (np.maximum(D, 0.0) + E64) + E64) + (dd + 2) * 2.0 ** -149
                hi = (D + B).min(1)
                cont = (D - B) <= hi[:, None]
                cont |= ~np.isfinite(hi)[:, None]
            ii, cc = np.nonzero(cont)
            vals = self._exact(Pi, Ci, ii + s0, cc)
            rowmin = np.full(len(D), np.inf, F32)
            np.minimum.at(rowmin, ii, vals)
            eq = (vals == rowmin[ii]) & np.isfinite(vals)
            cnt = np.bincount(ii[eq], minlength=len(D))
            self.info["ties"] += int((cnt >= 2).sum())
            first = np.full(len(D), k, np.int64)
            if self.mut.get("ties_high"):
                first[:] = -1
                np.maximum.at(first, ii[eq], cc[eq])
                first[first < 0] = 0
            else:
                np.minimum.at(first, ii[eq], cc[eq])
                first[first >= k] = 0                             # every distance inf: label 0
            lab[sl] = first
            best[sl] = rowmin
        if self.want_flips and n * k * self.d <= 5e7:
            l64, _, _ = okm.assign(np.asarray(P, F64), np.asarray(C, F64))
            self.info["flips"] += int((l64 != lab).sum())
        if not np.all(np.isfinite(best)):
            self.info["inf"] = True
        return lab, best

    def nearest(self, P, C):
        lab, best = self._d32(P, C)
        return lab, best.astype(F64) * self.inv2

    def running_min(self, cost, P, new):
        _, best = self._d32(P, new)
        b = best.astype(F64) * self.inv2
        return b if self.mut.get("replace_cost") else np.fmin(cost, b)

    # -- sums and the walk
    def total(self, v):
        return sum_over(v, self.cuts)

    def pick(self, v, seed, i):
        C = len(v)
        pre, total, j0, j1, vv = pp_scan(v, C, self.mut.get("seq_scan", False))
        if self.mut.get("prefix_shift"):
            pre = np.concatenate([[0.0], pre[:-1]])
        return pp_walk(pre, j0, j1, vv, okm.u(seed, 100, i) * total, C)

    def changed(self, lab, old, it):
        if self.mut.get("first_not_moved") and it == 0:
            return False
        return bool(np.any(lab != old))

    def draws_at(self, draws):
        return 0 if self.mut.get("reset_draws") else draws

    def cluster_sums(self, X, lab, k):
        out = np.zeros((k, X.shape[1]))
        for r in range(len(self.cuts) - 1):                       # each rank's sums in point order, then added
            sl = slice(self.cuts[r], self.cuts[r + 1])
            part = np.zeros((k, X.shape[1]))
            np.add.at(part, lab[sl], X[sl])
            out = out + part
        return out

    def moved(self, nc, c, tol):
        df = np.asarray(nc, F64) - np.asarray(c, F64)
        lanes = -(-len(df) // 32) * 32
        pad = np.zeros(lanes)
        pad[:len(df)] = df
        pad = pad.reshape(-1, 32)
        m = np.zeros(32)
        for row in pad:                                         # coordinates lane, lane + 32, ...
            m = fma64(row, row, m)
        off = 16
        while off > 0:
            m[:off] = m[:off] + m[off:2 * off]
            off //= 2
        self._moves.append(float(m[0]))
        return not (m[0] <= tol * tol)


def sum_over(v, cuts) -> float:
    """Each rank's fixed-order sum of its part of v, then their sum in rank order."""
    v = np.asarray(v)
    parts = [fixed_sum(v[cuts[r]:cuts[r + 1]]) for r in range(len(cuts) - 1)]
    t = parts[0]
    for p in parts[1:]:
        t = t + p
    return t


def run(X, k, max_iter=20, tol=1e-4, seed=0, init_centers=None, sizes=None, flips=False, **mutant):
    """The model's (centres, labels, iterations, cost) and its instrumentation.  Raises OverflowError where the library
    returns SGP_E_RANGE: the prescale out of range, or a nearest-centre distance beyond the fp32 range after it."""
    ar = Fp32Model(sizes=sizes, flips=flips, **mutant)
    C, lab, it, cost = okm.kmeans(X, k, max_iter=max_iter, tol=tol, seed=seed, init_centers=init_centers, ar=ar)
    ar.info["iterations"] = it
    if ar.info["inf"]:
        raise OverflowError("a nearest-centre distance is beyond the fp32 range")
    return (C, lab, it, cost), ar.info
