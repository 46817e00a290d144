"""CPU checks of the exact model of `sgp_kmeans` (oracle/kmeans_model.py): its emulated fmaf / fma against correctly
rounded rational arithmetic, its sum, scan and column-statistics mirrors against Python loops, its screened distances
against exhaustive emulation, its agreement with the fp64 restatement where both are exact, and mutants of the kernels'
arithmetic, each of which changes an output on the GPU case catalogue (oracle/kmeans_cases.py)."""
from fractions import Fraction as Fr

import numpy as np
import pytest

from oracle import kmeans as okm
from oracle import kmeans_cases as kc
from oracle import kmeans_model as km

F32 = np.float32


def round_f32(q: Fr) -> np.float32:
    """q correctly rounded to fp32 (ties to even, overflow to inf)."""
    if abs(q) >= Fr(2) ** 128 - Fr(2) ** 103:
        return F32(np.inf if q > 0 else -np.inf)
    f = F32(float(q))
    best = None
    for c in (np.nextafter(f, F32(-np.inf)), f, np.nextafter(f, F32(np.inf))):
        if not np.isfinite(c):
            continue
        key = (abs(Fr(float(c)) - q), int(np.array(c).view(np.int32)) & 1)
        if best is None or key < best[0]:
            best = (key, c)
    return best[1]


def exact(*xs):
    return [Fr(float(x)) for x in xs]


# ---- fmaf / fma ------------------------------------------------------------------------------------------------------
def test_fmaf_is_correctly_rounded():
    rng = np.random.default_rng(0)
    N = 20000
    a = (rng.standard_normal(N) * 2.0 ** rng.integers(-70, 60, N)).astype(F32)
    b = (rng.standard_normal(N) * 2.0 ** rng.integers(-70, 60, N)).astype(F32)
    c = (rng.standard_normal(N) * 2.0 ** rng.integers(-140, 120, N)).astype(F32)
    c[:4000] = (-(a[:4000].astype(np.float64) * b[:4000])).astype(F32)          # cancellation
    a[4000:4100], b[4000:4100] = F32(2.0 ** -75), F32(2.0 ** -75)               # subnormal and zero products
    c[4000:4050] = 0
    a[4100:4200] = F32(0.0)
    a[4200:4300], b[4200:4300], c[4200:4300] = F32(2.0 ** 64), F32(2.0 ** 64), F32(3.0e38)   # overflow to inf
    r = km.fmaf(a, b, c)
    for i in range(N):
        pa, pb, pc = exact(a[i], b[i], c[i])
        want = round_f32(pa * pb + pc)
        assert r[i] == want or (np.isnan(r[i]) and np.isnan(want)), (i, a[i], b[i], c[i], r[i], want)
    assert np.isinf(r[4200:4300]).all() and np.all(r[4100:4200] == c[4100:4200])


@pytest.mark.parametrize("sign", [1.0, -1.0])
def test_fmaf_rounds_the_double_rounding_midpoints_the_right_way(sign):
    # a b = 2^24 - 2^-22: the fp64 sum with 2^48 + 2^25 is the fp32 midpoint 2^48 + 2^25 + 2^24 (ties to even: up), the
    # exact sum lies below it (correct: down); and the mirror case with the error above the midpoint
    a, b = F32(2.0 ** 12 * (1 + 2.0 ** -23)), F32(2.0 ** 12 * (1 - 2.0 ** -23))
    c = F32(sign * (2.0 ** 48 + 2.0 ** 25))
    naive = F32(np.float64(sign * a) * np.float64(b) + np.float64(c))
    r = km.fmaf(F32(sign * a), b, c)
    assert r == F32(sign * (2.0 ** 48 + 2.0 ** 25)) != naive
    assert r == round_f32(Fr(float(sign * a)) * Fr(float(b)) + Fr(float(c)))


def test_fma64_is_correctly_rounded():
    rng = np.random.default_rng(1)
    N = 20000
    a = rng.standard_normal(N) * 2.0 ** rng.integers(-60, 60, N)
    b = rng.standard_normal(N) * 2.0 ** rng.integers(-60, 60, N)
    c = rng.standard_normal(N) * 2.0 ** rng.integers(-120, 120, N)
    c[:6000] = -(a[:6000] * b[:6000]) * (1 + rng.integers(-4, 5, 6000) * 2.0 ** -52)
    b[6000:8000] = a[6000:8000]                                                 # squares, as the column statistics use
    r = km.fma64(a, b, c)
    for i in range(N):
        pa, pb, pc = exact(a[i], b[i], c[i])
        assert r[i] == float(pa * pb + pc), i


# ---- mirrors -----------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("m", [0, 1, 263, 264, 265, 256 * 264, 256 * 264 + 1, 100_003])
def test_fixed_sum_mirrors_the_sum_kernel(m):
    v = np.random.default_rng(m).standard_normal(m) * 10.0 ** np.random.default_rng(m + 1).integers(-8, 8, m)
    per = -(-m // 264)
    t = 0.0
    for blk in range(264):
        sh = [0.0] * 256
        for th in range(256):
            a = 0.0
            i = blk * per + th
            while i < min(m, blk * per + per):
                a += float(v[i])
                i += 256
            sh[th] = a
        s = 128
        while s:
            for th in range(s):
                sh[th] += sh[th + s]
            s //= 2
        t += sh[0]
    assert km.fixed_sum(v) == t
    assert km.sum_over(v, [0, m]) == t


def _pp_loop(v, r, C):
    """kmeans_pp_kernel's scan and walk, thread by thread and lane by lane."""
    seg = -(-C // 1024)
    loc = []
    for tid in range(1024):
        j0, j1 = min(C, tid * seg), min(C, min(C, tid * seg) + seg)
        a = 0.0
        for j in range(j0, j1):
            a += v[j]
        loc.append(a)
    incl = list(loc)
    for w in range(32):
        for o in (1, 2, 4, 8, 16):
            old = incl[w * 32:(w + 1) * 32]
            for lane in range(o, 32):
                incl[w * 32 + lane] = old[lane] + old[lane - o]
    wt = [incl[w * 32 + 31] for w in range(32)]
    for o in (1, 2, 4, 8, 16):
        old = list(wt)
        for lane in range(o, 32):
            wt[lane] = old[lane] + old[lane - o]
    total = wt[31]
    rr = r * total
    if not (rr > 0.0):
        return 0, total
    found = C
    for tid in range(1024):
        w, lane = divmod(tid, 32)
        cum = (wt[w - 1] if w else 0.0) + (incl[tid - 1] if lane else 0.0)
        j0, j1 = min(C, tid * seg), min(C, min(C, tid * seg) + seg)
        for j in range(j0, j1):
            cum += v[j]
            if cum >= rr:
                found = min(found, j)
                break
    return (found if found < C else C - 1), total


@pytest.mark.parametrize("C", [5, 1024, 1025, 2048, 2049, 4000])
def test_pp_scan_and_walk_mirror_the_kernel_loop(C):
    rng = np.random.default_rng(C)
    v = rng.random(C) * 10.0 ** rng.integers(-6, 6, C)
    v[rng.random(C) < 0.2] = 0.0
    for u in (0.0, 1e-9, 0.3, 0.77, 0.999999):
        pre, total, j0, j1, vv = km.pp_scan(v, C)
        assert (km.pp_walk(pre, j0, j1, vv, u * total, C), total) == _pp_loop(list(v), u, C)
    # the block scan's rounding differs from a sequential cumsum's: the mirror keeps the kernel's, not the oracle's
    if C >= 1025:
        blk, seq = km.pp_scan(v, C), km.pp_scan(v, C, seq_scan=True)
        assert blk[1] != seq[1] or not np.array_equal(blk[0], seq[0])


@pytest.mark.parametrize("n", [1, 9, 1024, 1025, 3000])
def test_colstats_mirror_the_kernel_lanes(n):
    rng = np.random.default_rng(n)
    X = rng.standard_normal((n, 3)) * 1e3 + 1e6
    a, b = km.colstats(X)
    slices = min(264, max(1, -(-n // 1024)))
    rps = -(-n // slices)
    for j in range(3):
        ta, tb = 0.0, 0.0
        for q in range(slices):
            la, lb = 0.0, 0.0
            for rl in range(8):
                xa, xb = 0.0, Fr(0)
                for r in range(q * rps + rl, min(n, q * rps + rps), 8):
                    xa += float(X[r, j])
                    xb = Fr(float(Fr(float(X[r, j])) ** 2 + xb))             # fma(v, v, b): one rounding
                la += xa
                lb += float(xb)
            ta += la
            tb += lb
        assert a[j] == ta and b[j] == tb


def test_screened_distances_equal_exhaustive_emulation():
    rng = np.random.default_rng(3)
    for d, n, k in ((1, 300, 7), (5, 200, 40), (33, 150, 20)):
        X = kc._lattice_mixture(n, d, d)
        C = X[rng.permutation(n)[:k]] + rng.standard_normal((k, d)) * 1e-3
        ar = km.Fp32Model()
        ar.start(X)
        lab, best = ar.nearest(X, C)
        Pi, Ci = ar.images(X), ar.images(C)
        ii, cc = np.meshgrid(np.arange(n), np.arange(k), indexing="ij")
        full = ar._exact(Pi, Ci, ii.ravel(), cc.ravel()).reshape(n, k)
        want = np.full(n, 0)
        wbest = np.full(n, np.inf, F32)
        for i in range(n):
            for c in range(k):
                if full[i, c] < wbest[i]:
                    wbest[i], want[i] = full[i, c], c
        assert np.array_equal(lab, want) and np.array_equal(best, wbest.astype(np.float64))


# ---- the model against the restatement -------------------------------------------------------------------------------
def _int_blobs(d, seed=5, n_blobs=64, per=50):
    rng = np.random.default_rng(seed)
    centres = 1000.0 * rng.choice(np.arange(-40, 41), size=(n_blobs, d))
    X = np.concatenate([c + rng.integers(-2, 3, (per, d)) for c in centres]).astype(np.float64)
    return X[rng.permutation(len(X))]


@pytest.mark.parametrize("d", [2, 16, 33])
def test_model_equals_the_restatement_on_integer_blobs(d):
    X = _int_blobs(d)
    (C0, lab0, it0, cost0), _ = km.run(X, 64, max_iter=0, seed=3)
    o = okm.kmeans(X, 64, max_iter=0, seed=3)
    assert np.array_equal(C0, o[0]) and np.array_equal(lab0, o[1]) and it0 == o[2]
    assert abs(cost0 - o[3]) <= 1e-4 * o[3]                 # fp32 distances to the local Lloyd's weighted means
    (C, lab, it, cost), info = km.run(X, 64, max_iter=20, seed=3)
    o = okm.kmeans(X, 64, max_iter=20, seed=3)
    assert np.array_equal(C, o[0]) and np.array_equal(lab, o[1]) and it == o[2]
    assert abs(cost - o[3]) <= 1e-4 * o[3]                  # fp32 distances to non-integer means
    assert info["s"] == 0


def test_two_rank_model_equals_one_rank_on_integer_blobs():
    X = _int_blobs(5)
    one, _ = km.run(X, 40, max_iter=20, seed=2)
    for sizes in ([0, len(X)], [7, len(X) - 7], [1600, len(X) - 1600]):
        two, _ = km.run(X, 40, max_iter=20, seed=2, sizes=sizes)
        # every sum is exact but the final cost (fp32 distances to non-integer means), which splits at the shard edge
        assert all(np.array_equal(a, b) for a, b in zip(one[:3], two[:3]))
        assert abs(two[3] - one[3]) <= 1e-12 * one[3]


def test_ordinary_cases_have_no_prescale():
    for name in ("near_tie_d4", "d33", "k129", "offset1e6", "n1025"):
        _, info = kc.run_model(kc.catalogue()[name]())
        assert info["s"] == 0, name


# ---- mutants ----------------------------------------------------------------------------------------------------------
MUTANTS = {
    "ties_high": ("exact_ties",),
    "prefix_shift": ("C1077",),                 # two entries per k-means++ thread
    "drop_chunk": ("d33",),
    "unrounded": ("pow2_sd",),
    "replace_cost": ("d3",),
    "first_not_moved": ("d3",),
    "reset_draws": ("local_empty",),
}


def _outs(o):
    if o is None:
        return None
    C, lab, it, cost = o
    return C.tobytes(), lab.tobytes(), it, np.float64(cost).tobytes()


@pytest.mark.parametrize("mutant", list(MUTANTS))
def test_every_mutant_changes_an_output_on_the_catalogue(mutant):
    cat = kc.catalogue()
    for name in MUTANTS[mutant]:
        case = cat[name]()
        base, _ = kc.run_model(case)
        mut, _ = kc.run_model(case, **{mutant: True})
        if _outs(base) != _outs(mut):
            return
    pytest.fail("mutant %s changes no output on %s" % (mutant, MUTANTS[mutant]))


def test_fp64_distances_change_outputs_on_the_near_tie_cases():
    """The fp64 restatement itself is a mutant of the model: on the near-tie cases the two pick different centres."""
    for name in ("near_tie_d4", "near_tie_d9"):
        case = kc.catalogue()[name]()
        got, info = kc.run_model(case)
        assert info["flips"] > 0
        o = okm.kmeans(case["X"], case["k"], max_iter=case["max_iter"], tol=case["tol"], seed=case["seed"])
        assert _outs(o) != _outs(got), name
