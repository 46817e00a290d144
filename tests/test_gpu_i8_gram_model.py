"""The int8 Gram on the H100 against its exact integer model (run on an H100: `pytest -m gpu`).

tests/test_host_i8_gram_model.py writes the model down: from the kernel values kappa, the digit planes of their fixed-point
words, the exact integer products A4, A3, A2, G* = C^2 / (4 C0^2) (2^32 A4 + 2^24 A3 + 2^16 A2) and its majorant G+.  The
kernel's G must stay within R 2^-53 G+ of G* element by element (R counted from the launch geometry: about 1e-14 of
G+), and be exactly 0 where G+ is; b within C (17 2^-24 + R_b 2^-53) sum |kappa y32| of C sum kappa y32.

The premise: sgp_kmn_sweep runs the same operand images, the same fp16 distance contraction and the same fragment layout
as the digit-plane producer and stores scale * ex2f(T), so with scale 1 it returns the producer's fp32 kappa bit for bit.
Every case asserts it on the device: the producer's words of its first tile and unit (sgp_debug_i8_tile, the words of
the first unit of the last launch) equal fixed_word(kappa from the sweep) on every valid element.

Every case: force the int8 mode (AUTO where stated) and assert the path, run the statistics, sweep the same X in the same
dtype on a second context begun with C = 1 (same beta, same Z), build G*, G+ and b* with torch fp64 on the device, apply
both gates, check the premise and G == G' bitwise, and print the worst ratio |G - G*| / (2^-53 G+) against R.  Shards
made of B shuffled copies of a block are modelled as B times the block (the words depend on the point only).  The direct
distance mode cannot be swept; there the shard is B copies of one 64-point block placed first, so the debug tile IS the
block's word matrix and G is modelled from it (m <= 128), its b is left to the oracle tests."""
import numpy as np
import pytest
import torch

import spark_gp_b200 as sg
from spark_gp_b200 import _native as N
from test_gpu_entry_points import bench_shard
from test_host_i8_gram_model import (GramModel, b_gate, b_model, b_rounding_budget, entry_launches, gram_gate,
                                     launch_geometry, rounding_budget)
from test_host_logic import TILE, UNIT_POINTS, fixed_word, i8_slices, points_for_units

pytestmark = pytest.mark.gpu

SIGMA2 = 1e-4
GATE = 4096.0                 # kI8TensorR2Max
MODES = {"i8": N.SGP_PREC_I8, "auto": N.SGP_PREC_AUTO, "direct": N.SGP_PREC_I8_DIRECT}


@pytest.fixture(scope="module")
def eng():
    e = sg.ProjectedProcessEngine(0)
    e.debug_i8_tile()                              # arm the dump: every int8 launch writes its first tile and unit
    yield e
    e.close()


@pytest.fixture(scope="module")
def sweeper():
    e = sg.ProjectedProcessEngine(0)
    yield e
    e.close()


@pytest.fixture(scope="module")
def num_sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


def to_device(a):
    t = torch.from_numpy(np.ascontiguousarray(a)).cuda()
    torch.cuda.synchronize()
    return t


def kernel_factory(kind, d, eyes=0, rng=None):
    """mk(C): C * k for k = ARD (uniform beta sqrt(18 / d)), ARD with non-uniform beta, RBF, or the nested 2 * (0.5 C * ARD),
    with `eyes` Eye terms added; mk(1.0) is the kernel the sweep runs."""
    beta = np.full(d, np.sqrt(18.0 / d))
    if kind == "ard-nonuniform":
        u = rng.uniform(0.5, 1.5, d)
        beta = u * np.sqrt(18.0 / (u ** 2).sum())
    if kind == "rbf":
        base = lambda: sg.RBFKernel(1.0 / (np.sqrt(2.0) * np.sqrt(18.0 / d)))
    else:
        base = lambda: sg.ARDRBFKernel(beta)

    def mk(C):
        k = 2.0 * ((0.5 * C) * base()) if kind == "nested" else C * base()
        for e in range(eyes):
            k = k + sg.const(0.3 + e) * sg.EyeKernel()
        return k
    return mk


def bench_like(n, d, m, seed, dtype=np.float32, offset=0.0):
    """X ~ U[0,1)^d + offset (stored in dtype), y = sin(sum x) + 0.1 eps, Z = m of the points (or fresh ones if n < m)."""
    rng = np.random.default_rng(seed)
    X = (rng.random((n, d)) + offset).astype(dtype)
    y = np.sin(X.astype(np.float64).sum(1)) + 0.1 * rng.standard_normal(n)
    Z = X[rng.permutation(n)[:m]].astype(np.float64) if n >= m else rng.random((m, d)) + offset
    return X, y, Z


def sweep_chunks(sweeper, mk, Z, Xd, is_f32):
    """kappa of the points Xd (device), in chunks of (cn x m) fp32 on the device, from the sweep with C = 1."""
    m = len(Z)
    sweeper.begin(mk(1.0), Z)
    step = max(UNIT_POINTS, min(65536, (1 << 24) // m))
    for p0 in range(0, len(Xd), step):
        cn = min(step, len(Xd) - p0)
        K = torch.empty((cn, m), dtype=torch.float32, device="cuda")
        # the sweep writes on its context's stream: torch's products of the previous chunk, whose memory the caching
        # allocator may have handed out again, must be done first
        torch.cuda.synchronize()
        sweeper.kmn_sweep_device(Xd[p0:p0 + cn].data_ptr(), is_f32, cn, K.data_ptr())
        sweeper.sync()
        yield p0, cn, K


def run_case(eng, sweeper, num_sms, name, Xb, yb, Z, mk, C, mode="i8", calls=None, reps=1, seed=0):
    """Statistics of the shard of `reps` shuffled copies of (Xb, yb) (the block itself for reps = 1) through `calls`
    [(entry, points), ...] in one begin..finish window (default: one device call), against the model.  Returns G, b."""
    n, (nb, d), m = len(Xb) * reps, Xb.shape, len(Z)
    is_f32 = Xb.dtype == np.float32
    src = np.random.default_rng(seed).permutation(n) % nb if reps > 1 else np.arange(n)
    X, y = (Xb[src], yb[src]) if reps > 1 else (Xb, yb)
    calls = calls or [("device", n)]
    assert sum(cn for _, cn in calls) == n
    Xd = yd = None
    if any(entry == "device" for entry, _ in calls):
        Xd, yd = to_device(X), to_device(y)
    # 1-2. the statistics
    eng.set_precision(MODES[mode])
    eng.begin(mk(C), Z)
    launches, p0, last = [], 0, 0
    for entry, cn in calls:
        before = eng.launch_count()
        if entry == "device":
            eng.accumulate_ptr(Xd[p0:p0 + cn].data_ptr(), is_f32, yd[p0:p0 + cn].data_ptr(), cn, device=True)
            windows = launch_geometry(cn, m, num_sms)["windows"]
            assert eng.launch_count() - before == 1 + 2 * windows + 1          # prep, (planes, Gram) per window, reduce
        else:
            eng.accumulate(X[p0:p0 + cn], y[p0:p0 + cn])
        assert eng.last_path() == N.SGP_PREC_I8
        chunks = entry_launches(entry, cn, d, is_f32)
        last = p0 + sum(chunks[:-1])
        launches += chunks
        p0 += cn
    _, words = eng.debug_i8_tile()
    G, b = eng.finish()
    del Xd, yd
    # 3-4. the sweep with C = 1, and the model on the device
    model = GramModel(m, device="cuda")
    bstar = torch.zeros(m, dtype=torch.float64, device="cuda")
    bplus = torch.zeros(m, dtype=torch.float64, device="cuda")
    Xbd, ybd = to_device(Xb), to_device(yb)
    for q0, cn, K in sweep_chunks(sweeper, mk, Z, Xbd, is_f32):
        model.add_kappa(K)
        bs, bp = b_model(K, ybd[q0:q0 + cn], C)
        bstar += bs
        bplus += bp
    del Xbd, ybd
    # 5. the premise, before the gates: the words of the last launch's first unit are fixed_word(swept kappa)
    rows, pts = min(m, TILE), min(UNIT_POINTS, launches[-1])
    kappa = sweeper.kmn_sweep(X[last:last + pts])
    want = (fixed_word(kappa[:, :rows]) >> np.uint64(1)).astype(np.uint32).T
    assert np.array_equal(words[:rows, :pts], want), "producer words != fixed_word(sweep kappa): %d of %d differ" % (
        int((words[:rows, :pts] != want).sum()), want.size)
    Gs, Gp = model.times(reps).gram(C)
    bstar, bplus = (reps * bstar).cpu().numpy(), (reps * bplus).cpu().numpy()
    R = rounding_budget(launches, m, num_sms)
    ratio = gram_gate(G, Gs, Gp, R)
    bratio = b_gate(b, bstar, bplus, C, b_rounding_budget(launches, num_sms))
    # 6. symmetry
    assert np.array_equal(G, G.T)
    windows = sum(launch_geometry(cn, m, num_sms)["windows"] for cn in launches)
    print("%s: n=%d m=%d d=%d %s, %d launch(es), %d window(s): G worst %.2f of R = %d roundings of G+; b %.2e of its "
          "bound; premise %d words equal" % (name, n, m, d, np.dtype(Xb.dtype).name, len(launches), windows, ratio, R,
                                             bratio, want.size))
    return G, b


# ---- producer variants: KS = 4 (d <= 16, one K chunk) and KS = 7 (d 17..32, two chunks), fp32 and fp64 X ------------------
@pytest.mark.parametrize("dtype", [np.float32, np.float64], ids=["fp32", "fp64"])
@pytest.mark.parametrize("d", [1, 2, 3, 8, 15, 16, 17, 20, 31, 32])
def test_producer_variants(eng, sweeper, num_sms, d, dtype):
    X, y, Z = bench_like(30001, d, 300, seed=d, dtype=dtype)
    run_case(eng, sweeper, num_sms, "d=%d" % d, X, y, Z, kernel_factory("ard", d, eyes=1), 1.0)


# ---- the tile triangle: 1 to 32 active tiles, up to 528 tile pairs, diagonal tiles, padded rows ----------------------------
@pytest.mark.parametrize("m", [1, 2, 127, 128, 129, 255, 256, 257, 1000, 1300, 2000, 4000])
def test_tile_triangle(eng, sweeper, num_sms, m):
    X, y, Z = bench_like(40000, 8, m, seed=m)
    run_case(eng, sweeper, num_sms, "m=%d" % m, X, y, Z, kernel_factory("ard", 8, eyes=1), 1.0)


# ---- units: padded points in the last (or only) unit ---------------------------------------------------------------------
@pytest.mark.parametrize("n", [1, 63, 64, 65])
def test_unit_edges(eng, sweeper, num_sms, n):
    X, y, Z = bench_like(n, 5, 200, seed=n)
    run_case(eng, sweeper, num_sms, "n=%d" % n, X, y, Z, kernel_factory("ard", 5), 1.0)


def test_empty_slices(eng, sweeper, num_sms):
    """300 units on one tile: the Gram takes 16 slices of 19 units (the last one shorter), the producer 132 or 264
    slices of 3 or 2 units, so its last slices get no units."""
    n, m = 300 * UNIT_POINTS - 7, 128
    assert i8_slices(TILE, num_sms, 300) == 16
    for per_sm in (1, 2):
        s = min(num_sms * per_sm, 300)
        assert -(-300 // s) * (s - 1) >= 300                     # at least one empty producer slice
    X, y, Z = bench_like(n, 6, m, seed=300)
    run_case(eng, sweeper, num_sms, "300 units", X, y, Z, kernel_factory("ard", 6), 1.0)


# ---- folds: one slice of 399 .. 1201 units, the int32 accumulators folded every 400 ------------------------------------
@pytest.mark.parametrize("units,jag", [(399, 0), (400, 17), (401, 0), (800, 0), (801, 5), (1201, 63)])
def test_fold_boundaries(eng, sweeper, num_sms, units, jag):
    m, d = 1300, 16
    n = points_for_units(m, units, num_sms, jag)
    g = launch_geometry(n, m, num_sms)
    assert g["windows"] == 1 and -(-g["units"] // g["g_slices"]) == units
    X, y, Z = bench_like(n, d, m, seed=units)
    run_case(eng, sweeper, num_sms, "%d units per slice" % units, X, y, Z, kernel_factory("ard", d, eyes=1), 1.0)


# ---- launch windows: the planes of one launch split into windows of <= 4 GiB -------------------------------------------
WINDOW_CASES = {           # block points, copies, d, m, dtype, windows
    "m4000-2-windows": (10001, 69, 8, 4000, np.float32, 2),
    "m4000-3-windows": (13001, 54, 8, 4000, np.float32, 3),
    "configs3": (20480, 61, 32, 2000, np.float32, 2),
}


@pytest.mark.parametrize("name", list(WINDOW_CASES))
def test_launch_windows(eng, sweeper, num_sms, name):
    """Device entry; the window count is checked through launch_count() (1 + 2 windows + 1 launches).  configs3 is
    bench.py's configs3 shard shape (1.25M x 32, m = 2000) as 61 shuffled copies of a 20480-point block."""
    nb, reps, d, m, dtype, windows = WINDOW_CASES[name]
    g = launch_geometry(nb * reps, m, num_sms)
    assert g["windows"] == windows
    if name != "configs3":
        assert g["units"] - (windows - 1) * g["win_units"] < g["win_units"]          # a shorter last window
    X, y, Z = bench_like(nb, d, m, seed=nb)
    run_case(eng, sweeper, num_sms, name, X, y, Z, kernel_factory("ard", d, eyes=1), 1.0, reps=reps, seed=reps)


# ---- entries and windows of calls ------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", ["host-fp32", "host-fp64", "device+host+device"])
def test_entries(eng, sweeper, num_sms, name):
    """The host entry (its chunk plan: several launches) and a begin..finish window mixing device and host calls."""
    if name == "host-fp32":
        X, y, Z = bench_like(300_000, 16, 512, seed=1)
        calls = [("host", len(X))]
    elif name == "host-fp64":
        X, y, Z = bench_like(300_001, 16, 300, seed=2, dtype=np.float64)
        calls = [("host", len(X))]
    else:
        X, y, Z = bench_like(350_001, 12, 700, seed=3)
        calls = [("device", 100_000), ("host", 200_000), ("device", 50_001)]
    assert sum(len(entry_launches(e, cn, X.shape[1], X.dtype == np.float32)) for e, cn in calls) >= 3
    run_case(eng, sweeper, num_sms, name, X, y, Z, kernel_factory("ard", X.shape[1], eyes=1), 1.0, calls=calls)


# ---- bench.py's configs1 shard on the device entry, forced and as AUTO picks it ------------------------------------------
@pytest.mark.parametrize("mode", ["i8", "auto"])
def test_configs1_device_entry(eng, sweeper, num_sms, mode):
    """1M x 16, m = 1000: 11 slices of 1421 units, four folds of which three add."""
    X, y, Z = bench_shard("configs1")
    g = launch_geometry(len(X), 1000, num_sms)
    assert g["windows"] == 1
    if num_sms == 132:
        assert (g["g_slices"], g["folds"]) == (11, 4)
    run_case(eng, sweeper, num_sms, "configs1 [%s]" % mode, X, y, Z, kernel_factory("ard", 16, eyes=2), 1.0, mode=mode)


# ---- kernel forms ----------------------------------------------------------------------------------------------------
FORMS = [("ard-nonuniform", 0.37, 1), ("rbf", 17.0, 2), ("nested", 1.0, 0), ("ard", 0.25, 1), ("ard", 1.0, 2),
         ("rbf", 0.25, 0), ("nested", 0.25, 2)]


@pytest.mark.parametrize("kind,C,eyes", FORMS)
def test_kernel_forms(eng, sweeper, num_sms, kind, C, eyes):
    d = 7
    X, y, Z = bench_like(50_000, d, 300, seed=int(C * 100) + eyes)
    mk = kernel_factory(kind, d, eyes=eyes, rng=np.random.default_rng(11))
    run_case(eng, sweeper, num_sms, "%s C=%g eyes=%d" % (kind, C, eyes), X, y, Z, mk, C)


def test_eye_terms_leave_the_statistics_alone(eng, num_sms):
    """Zero, one and two Eye terms: G and b bit for bit the same."""
    d = 7
    X, y, Z = bench_like(50_000, d, 300, seed=77)
    out = []
    for eyes in (0, 1, 2):
        eng.set_precision(N.SGP_PREC_I8)
        eng.begin(kernel_factory("ard", d, eyes=eyes)(0.37), Z)
        eng.accumulate(X, y)
        assert eng.last_path() == N.SGP_PREC_I8
        out.append(eng.finish())
    for G, b in out[1:]:
        assert np.array_equal(G, out[0][0]) and np.array_equal(b, out[0][1])


# ---- placement and margins -------------------------------------------------------------------------------------------
def clustered(level, n, d, m, seed):
    """Points in 8 clusters whose scaled squared norms reach `level` (at most 0.99 of the operand gate); X contains Z,
    so the first tile holds coinciding pairs, where kappa can exceed 1."""
    rng = np.random.default_rng(seed)
    signs = rng.choice([-1.0, 1.0], (8, d))
    L = np.sqrt(level / (np.log2(np.e) * d))
    X = L * signs[rng.integers(0, 8, n)] + 0.3 * rng.standard_normal((n, d))
    norms = np.log2(np.e) * ((X - X[:m].mean(0)) ** 2).sum(1)
    X *= min(1.0, np.sqrt(0.99 * GATE / norms.max()))
    y = rng.standard_normal(n)
    return X, y, X[:m].copy()


@pytest.mark.parametrize("name", ["offset-1e3", "norms-512", "norms-4000"])
def test_placement_and_margins(eng, sweeper, num_sms, name):
    d, m = 16, 256
    if name == "offset-1e3":
        X, y, Z = bench_like(40_000, d, m, seed=5, offset=1e3)
        mk = kernel_factory("ard", d, eyes=1)
    else:
        X, y, Z = clustered(float(name.split("-")[1]), 16384, d, m, seed=6)
        mk = lambda C: C * sg.ARDRBFKernel(np.ones(d)) + sg.const(1e-3) * sg.EyeKernel()
    run_case(eng, sweeper, num_sms, name, X, y, Z, mk, 1.0)


# ---- exact zeros -----------------------------------------------------------------------------------------------------
def test_exact_zero_blocks(eng, sweeper, num_sms):
    """Two clusters 60 length scales apart, active tile 0 from one and tile 1 from the other: every kernel value between
    them is 0, so the off-diagonal block of G* is exactly 0 and G must be too (a misrouted tile shows).  y = 0 gives
    b == 0 exactly."""
    rng = np.random.default_rng(8)
    d, n = 4, 40_000
    centre = np.full(d, 30.0 / np.sqrt(d))
    lab = rng.integers(0, 2, n)
    X = np.where(lab[:, None] == 0, -centre, centre) + 0.5 * rng.standard_normal((n, d))
    y = rng.standard_normal(n)
    Z = np.vstack([X[lab == 0][:TILE], X[lab == 1][:TILE]])
    mk = lambda C: C * sg.ARDRBFKernel(np.ones(d)) + sg.const(1e-3) * sg.EyeKernel()
    G, _ = run_case(eng, sweeper, num_sms, "two clusters", X, y, Z, mk, 1.0)
    assert np.all(G[:TILE, TILE:] == 0.0) and np.all(G[TILE:, :TILE] == 0.0)
    assert np.all(np.diag(G) > 0.0)
    _, b = run_case(eng, sweeper, num_sms, "two clusters, y = 0", X, np.zeros(n), Z, mk, 1.0)
    assert np.array_equal(b, np.zeros(len(Z)))


# ---- the direct-distance mode, Gram half only ---------------------------------------------------------------------------
DIRECT_CASES = [   # terms, d, m, copies of the 64-point block
    (1, 72, 128, 1),
    (1, 5, 1, 300),
    (2, 36, 100, 6400),
    (3, 24, 128, 16 * 1201),
    (4, 16, 77, 16 * 1201),
    (4, 3, 128, 801),
]


@pytest.mark.parametrize("terms,d,m,reps", DIRECT_CASES, ids=lambda v: str(v))
def test_direct_mode_gram(eng, num_sms, terms, d, m, reps):
    """SGP_PREC_I8_DIRECT with 1 to 4 terms up to the width limit n_terms * roundup(d, 4) <= 72.  The shard is `reps`
    copies of one 64-point block placed first, so the producer's debug tile is the block's whole word matrix and
    G* = reps x the block's products."""
    rng = np.random.default_rng(terms * 1000 + d)
    Xb = rng.random((UNIT_POINTS, d), dtype=np.float32)
    yb = rng.standard_normal(UNIT_POINTS)
    Z = rng.random((m, d))
    scales = [1.3, 0.6, 0.25, 2.0][:terms]
    terms_k = [s * (sg.ARDRBFKernel(rng.uniform(0.5, 1.5, d) * np.sqrt(3.0 / d)) if t % 2 == 0
                    else sg.RBFKernel(np.sqrt(d / 6.0))) for t, s in enumerate(scales)]
    k = terms_k[0]
    for t in terms_k[1:]:
        k = k + t
    k = k + sg.const(SIGMA2) * sg.EyeKernel()
    C = 0.0
    for t in k.flatten():
        if t["type"] != N.SGP_TERM_EYE:
            C += t["scale"]                                   # the mode's fixed-point scale: sum of the term scales
    n = UNIT_POINTS * reps
    X, y = np.tile(Xb, (reps, 1)), np.tile(yb, reps)
    Xd, yd = to_device(X), to_device(y)
    eng.set_precision(N.SGP_PREC_I8_DIRECT)
    eng.begin(k, Z)
    eng.accumulate_ptr(Xd.data_ptr(), True, yd.data_ptr(), n, device=True)
    assert eng.last_path() == N.SGP_PREC_I8_DIRECT
    _, words = eng.debug_i8_tile()
    G, _ = eng.finish()
    del Xd, yd
    w = torch.from_numpy((words[:m].astype(np.int64) << 1).T.copy()).cuda()     # 64 points x m, the producer's words
    assert torch.all((w >> 24) & 0xFF == 150)                     # no word overflowed the encoding
    Gs, Gp = GramModel(m, device="cuda").add_words(w).times(reps).gram(C)
    g = launch_geometry(n, m, num_sms)
    R = rounding_budget([n], m, num_sms)
    ratio = gram_gate(G, Gs, Gp, R)
    assert np.array_equal(G, G.T)
    print("direct, %d terms, d=%d, m=%d, %d units (%d slices, %d folds): G worst %.2f of R = %d roundings of G+" % (
        terms, d, m, g["units"], g["g_slices"], g["folds"], ratio, R))
