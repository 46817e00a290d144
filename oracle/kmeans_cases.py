"""The case catalogue on which `sgp_kmeans` is pinned to its exact model (oracle/kmeans_model.py): each case names the
edge it reaches, and `claims` states what the model's instrumentation must show for the case to reach it.

A case is a dict: X, k, max_iter, tol, seed, init (or None), f32 (whether the fp32-X form runs too), claims (key ->
(op, value) on the model's instrumentation), refused (the library must return SGP_E_RANGE)."""
from __future__ import annotations

import numpy as np


def _lattice_mixture(n, d, seed, parts=6, sep=0.6, step=0.1):
    """Overlapping Gaussian blobs rounded to a decimal lattice: real-valued coordinates (0.1 is not dyadic) with many
    points equidistant in exact arithmetic from two candidates, so fp32 and fp64 pick different nearest centres."""
    rng = np.random.default_rng(seed)
    X = np.concatenate([rng.standard_normal((n // parts + (i < n % parts), d)) + sep * rng.standard_normal(d)
                        for i in range(parts)])
    return np.round(X[rng.permutation(len(X))] * 3.0 / step) * step


def _case(X, k, max_iter=20, tol=1e-4, seed=0, init=None, f32=True, claims=None, refused=False):
    return dict(X=X, k=k, max_iter=max_iter, tol=tol, seed=seed, init=init, f32=f32, claims=claims or {}, refused=refused)


def _near_tie():
    return _case(_lattice_mixture(6000, 4, 1), 40, max_iter=200, seed=2,
                 claims=dict(flips=(">", 0), C=(">", 40), local_iterations=(">=", 2), iterations=("<", 200)))


def _near_tie_d9():
    return _case(_lattice_mixture(4000, 9, 2), 25, max_iter=200, seed=5,
                 claims=dict(flips=(">", 0), C=(">", 25), iterations=("<", 200)))


def _d(d):
    dch = 4 if d <= 4 else 8 if d <= 8 else 16 if d <= 16 else 32
    return _case(_lattice_mixture(2000, d, 10 + d), 12, max_iter=4, seed=d,
                 claims=dict(DCH=("==", dch), TC=("==", 64 if d <= 16 else 32), chunks=("==", -(-d // dch)),
                             C=(">", 12)))


def _k(k):
    n = max(3000, 12 * k)
    return _case(_lattice_mixture(n, 3, 100 + k), k, max_iter=3, seed=k, f32=k <= 129,
                 claims=dict(C=(">", k), seg=(">=", 3) if k == 1000 else ("==", 1)))


# C -> (k, seed) giving exactly C candidates on _lattice_mixture(12000, 3, 1): one k-means++ segment per thread at
# C = 1024, two at 1077, three at 2085 and 2106 (k = 1000 reaches four)
C_EDGES = {1024: (244, 10), 1077: (253, 4), 2085: (510, 4), 2106: (520, 6)}


def _C(C):
    k, seed = C_EDGES[C]
    return _case(_lattice_mixture(12000, 3, 1), k, max_iter=2, seed=seed, f32=False,
                 claims=dict(C=("==", C), seg=("==", -(-C // 1024))))


# n -> the launch geometry it reaches: the assignment's 128-thread blocks (blocks, rows in the last), the column
# statistics' slices of 1024 rows (at most 264 slices), and the sum kernel's 264 blocks of ceil(n / 264) elements
N_EDGES = {127: dict(assign_blocks=1, last_block_rows=127), 128: dict(assign_blocks=1, last_block_rows=128),
           129: dict(assign_blocks=2, last_block_rows=1), 1024: dict(slices=1, rows_per_slice=1024),
           1025: dict(slices=2, rows_per_slice=513), 67584: dict(sum_per=256), 67585: dict(sum_per=257),
           270336: dict(slices=264, rows_per_slice=1024), 270337: dict(slices=264, rows_per_slice=1025)}


def _n(n, d=2, k=8):
    X = _lattice_mixture(n, d, n % 1000 + 7)
    return _case(X, k, max_iter=3, seed=n % 97, f32=n < 100_000,
                 claims={key: ("==", v) for key, v in N_EDGES[n].items()})


def _local_empty():
    """Ten sites, each a cloud of points that differ from the site by 1e-13 relative: distinct fp64 rows, one fp32 image
    per site.  Only the first candidate of each image gets weight, so the k-means++ repeats candidate 0 once the ten
    are taken and the local Lloyd reseeds its empty clusters from stream 101."""
    rng = np.random.default_rng(31)
    sites = rng.integers(-50, 51, (10, 3)).astype(np.float64) + 0.5
    X = np.concatenate([s * (1.0 + 1e-13 * rng.standard_normal((60, 3))) for s in sites])
    return _case(X[rng.permutation(len(X))], 30, max_iter=10, seed=3, f32=False,
                 claims=dict(draws101=(">", 0), C=(">", 30), local_iterations=(">=", 2)))


def _global_empty():
    rng = np.random.default_rng(8)
    X = np.round(rng.standard_normal((3000, 3)) * 30) / 10
    init = X[:12].copy()
    init[3] = init[0]                                         # a duplicate: the tie goes to centre 0, 3 stays empty
    init[7] = 1e3 + np.arange(3)                              # far from the data: empty throughout
    return _case(X, 12, max_iter=30, init=init, claims=dict(empty=(">", 0), ties=(">", 0)))


def _exact_ties():
    g = np.arange(-6, 7, dtype=np.float64)
    X = np.stack(np.meshgrid(g, g, g), -1).reshape(-1, 3)
    init = np.array([[x, y, 0.0] for x in (-4, -2, 0, 2, 4) for y in (-3, 1, 5)])
    return _case(X, len(init), max_iter=1, init=init, claims=dict(ties=(">", 100)))


def _tol(tol, max_iter, iterations):
    """Cluster 0 = {0, 1} from centre 0 moves by exactly 0.5, so moved = 0.25 = 0.5^2: converged at iteration 1 with
    tol = 0.5, not with the next double below (then at iteration 2, where nothing moves)."""
    X = np.array([[0.0, 0.0], [1.0, 0.0], [10.0, 4.0], [10.0, 4.0]] * 50)
    claims = dict(iterations=("==", iterations))
    if max_iter:
        claims["moved_first"] = ("==", 0.25)
    return _case(X, 2, max_iter=max_iter, tol=tol, init=np.array([[0.0, 0.0], [10.0, 4.0]]), claims=claims)


def _offset(off):
    rng = np.random.default_rng(int(np.log10(off)))
    X = rng.standard_normal((3000, 4)) + off
    return _case(X, 16, max_iter=10, seed=1, f32=False, claims=dict(C=(">", 16)))


def _constant_column():
    X = _lattice_mixture(3000, 4, 41)
    X[:, 2] = 3.0
    return _case(X, 16, max_iter=10, seed=4, claims=dict(constant=("==", 1)))


def _pow2_sd():
    """Column 1 is 5 +- 2 in equal halves: its mean is 5 and its sd exactly 2 (a power of two)."""
    X = _lattice_mixture(4000, 3, 43)
    X[:, 1] = 5.0 + 2.0 * np.where(np.arange(4000) % 2 == 0, 1.0, -1.0)
    return _case(X, 16, max_iter=10, seed=6, claims=dict(pow2sd=("==", 1)))


def _scale(spread, n=4000):
    """Data scaled by `spread`; below fp32's range (about 1e-45) only the fp64 form keeps the data."""
    X = _lattice_mixture(n, 4, 3) * spread
    return _case(X, 20, max_iter=20, seed=1, f32=spread > 1e-40, claims=dict(s=("!=", 0), C=(">", 20)))


def _outlier():
    X = _lattice_mixture(4000, 4, 3)
    X[17, 2] = 2.0 ** 70
    return _case(X, 20, max_iter=20, seed=1, claims=dict(s=("!=", 0), C=(">", 20)))


def _far_init():
    X = _lattice_mixture(2000, 3, 5)
    return _case(X, 4, max_iter=5, init=np.full((4, 3), 1e25), refused=True)


def _tiny():
    """sd about 3e-160: the prescale would need 2^529, beyond 2^511."""
    return _case(_lattice_mixture(2000, 3, 7) * 1e-160, 8, max_iter=5, seed=1, f32=False, refused=True)


def _huge():
    X = _lattice_mixture(2000, 3, 6) * 1e200                  # squares overflow fp64 (and fp32 X cannot hold it)
    return _case(X, 8, max_iter=5, seed=1, f32=False, refused=True)


def catalogue():
    """name -> builder (called lazily: the builders cost milliseconds, the model seconds)."""
    cat = {"near_tie_d4": _near_tie, "near_tie_d9": _near_tie_d9}
    for d in (1, 3, 4, 5, 8, 9, 16, 17, 31, 32, 33, 64, 65, 100):
        cat["d%d" % d] = (lambda d=d: _d(d))
    for k in (2, 31, 32, 33, 63, 64, 65, 128, 129, 1000):
        cat["k%d" % k] = (lambda k=k: _k(k))
    for C in C_EDGES:
        cat["C%d" % C] = (lambda C=C: _C(C))
    for n in (127, 128, 129, 1024, 1025, 67584, 67585, 270336, 270337):
        cat["n%d" % n] = (lambda n=n: _n(n, d=1 if n > 100_000 else 2, k=4 if n > 100_000 else 8))
    cat.update(local_empty=_local_empty, global_empty=_global_empty, exact_ties=_exact_ties,
               tol_equal=lambda: _tol(0.5, 50, 1), tol_ulp_above=lambda: _tol(np.nextafter(0.5, 0.0), 50, 2),
               max_iter0=lambda: _tol(0.5, 0, 0), max_iter1=lambda: _tol(np.nextafter(0.5, 0.0), 1, 1),
               offset1e6=lambda: _offset(1e6), offset1e12=lambda: _offset(1e12), constant_column=_constant_column,
               pow2_sd=_pow2_sd, spread1e_30=lambda: _scale(1e-30), spread1e_21=lambda: _scale(1e-21),
               spread1e17=lambda: _scale(1e17), spread1e21=lambda: _scale(1e21), outlier2_70=_outlier,
               spread1e_146=lambda: _scale(1e-146, 1500), spread1e_150=lambda: _scale(1e-150, 1500),
               far_init_refused=_far_init, tiny_refused=_tiny, huge_refused=_huge)
    return cat


def run_model(case, f32=False, sizes=None, **mutant):
    """The model on a case: ((centres, labels, iterations, cost), info), or (None, info) where the library refuses."""
    from oracle import kmeans_model as km
    X = case["X"].astype(np.float32) if f32 else case["X"]
    try:
        with np.errstate(over="ignore", invalid="ignore"):
            out, info = km.run(X, case["k"], max_iter=case["max_iter"], tol=case["tol"], seed=case["seed"],
                               init_centers=case["init"], sizes=sizes, flips=True, **mutant)
    except OverflowError:
        return None, {}
    info = dict(info, n=len(X), constant=int(np.sum(info["sds"] == 0.0)),
                pow2sd=int(np.sum([s > 0 and np.frexp(s)[0] == 0.5 for s in info["sds"]])))
    return out, info


def check_claims(case, info):
    ops = {">": np.greater, ">=": np.greater_equal, "==": np.equal, "<": np.less, "!=": np.not_equal}
    bad = ["%s %s %s (got %r)" % (key, op, val, info.get(key)) for key, (op, val) in case["claims"].items()
           if info.get(key) is None or not ops[op](info[key], val)]
    assert not bad, "the case does not reach its edge: " + "; ".join(bad)
