"""The exact integer model of the int8 Gram (kmn_i8_planes_kernel + gram_i8_kernel, csrc/gram_i8_wgmma.cu), checked on
the CPU; tests/test_gpu_i8_gram_model.py applies it to the kernel on an H100.

The int8 path's error has two halves.  The distance half (fp16 hi/lo contraction, ex2.approx, the 23-bit fixed point) is
inexact by design and pinned element by element by the sweep-vs-oracle tests.  The Gram half is exact: every kernel
value kappa becomes the word fixed_word(kappa) (test_host_logic.py), whose bytes are the digit planes P0, P1 (signed) and
P2 (unsigned), and the kernel keeps six int8 products of them:
    A4 = P2'P2,  A3 = P2'P1 + P1'P2,  A2 = P2'P0 + P0'P2 + P1'P1,
    G* = C^2 / (4 C0^2) (2^32 A4 + 2^24 A3 + 2^16 A2).
Every partial sum of A4, A3, A2 is an integer below 255^2 * 2 n < 2^53, so an fp64 matmul computes them exactly in any
order.  The device adds fp64 roundings only: the three-term sum and the product with C^2 / (4 C0^2) of each fold, one
per fold add, one per Gram slice in gram_reduce_upper_kernel, one per launch's G +=.  Each is bounded by 2^-53 times
G+, the same formula on |P0|, |P1|, P2, which majorises every partial sum, so G is pinned element by element:
    |G - G*| <= R 2^-53 G+,
with R counted from the launch geometry (rounding_budget).  Where G+ is 0 the gate demands exact zeros.  b stays inexact
by design: 16 fp32 FMAs per lane and unit, then fp64:
    |b - C sum_n kappa y32| <= C (17 2^-24 + R_b 2^-53) sum_n |kappa y32|,
with y32 = fp32(y), the values the producer reads.

A CPU emulation of the kernel's folds, slices and reduction on bench.py's data family passes the gate; each mutant of
it fails the gate by a factor of 1e6 or more -- and the mutant that drops the P2'P0 + P0'P2 product class passes the
oracle gates of the existing int8 tests (TOL_I8, TOL_STATS)."""
import os
import re
from fractions import Fraction

import numpy as np
import pytest
import torch

from test_host_logic import (FIXED_C0, FIXED_MAGIC, FLUSH_UNITS, H100_SXM_SMS, TILE, UNIT_POINTS, digit_planes,
                             fixed_word, host_chunks, i8_slices, points_for_units)

U53, U24 = 2.0 ** -53, 2.0 ** -24
TOL_I8, TOL_STATS = 3e-6, 1e-6            # the oracle gates of test_gpu_entry_points.py / test_gpu_parity.py
B_FP32_ULPS = 17                          # 16 FMAs per lane and unit, and one to spare
R_CONST = 12                              # per fold: 2 in the three-term sum, 1 in the scale, 2 in the scale itself;
                                          # the model's own G*: the same 5; and 2 to spare
I8_PLANE_BYTES = 3 * TILE * UNIT_POINTS   # kI8PlaneBytes: three 128 x 64 planes per (unit, active tile)
I8_PLANE_CAP_BYTES = 4 << 30              # kI8PlaneCapBytes: digit planes of one launch window
CSRC = os.path.join(os.path.dirname(os.path.abspath(__file__)), "..", "spark_gp_b200", "csrc")


# ---- the model ------------------------------------------------------------------------------------------------------
def fixed_word_t(kappa):
    """torch port of test_host_logic.fixed_word: bits(fmaf(kappa, C0, MAGIC)) << 1 as int64, for an fp32 tensor on any
    device.  kappa * C0 is exact in fp64; torch.round rounds half to even, like the FMA's single rounding."""
    p = kappa.to(torch.float32).to(torch.float64) * float(FIXED_C0)
    magic = float(FIXED_MAGIC)
    below = magic + torch.round(p)
    above = 2.0 * torch.round((magic + p) * 0.5)
    f = torch.where(below < 2.0 ** 24, below, above).to(torch.float32)
    return (f.view(torch.int32).to(torch.int64) << 1) & 0xFFFFFFFF


def digit_planes_t(word):
    """torch port of test_host_logic.digit_planes: (P0, P1, P2) of int64 words, as fp64 tensors."""
    return tuple(((((word >> (8 * i)) & 0xFF) - (128 if i < 2 else 0)).to(torch.float64)) for i in range(3))


def gram_scale(C):
    """gscale of launch_gram_i8: C^2 / (4 C0^2), in the same operation order."""
    return C * C / (4.0 * float(FIXED_C0) * float(FIXED_C0))


class GramModel:
    """The exact integer products of the digit planes of a set of points (rows: points, columns: active points), summed
    in fp64 over chunks of points, with their majorants on |P0| and |P1|."""

    def __init__(self, m, device="cpu"):
        self.S = {k: torch.zeros((m, m), dtype=torch.float64, device=device)
                  for k in ("22", "21", "20", "11", "21+", "20+", "11+")}

    def add_planes(self, P0, P1, P2):
        a0, a1 = P0.abs(), P1.abs()
        for k, (a, b) in {"22": (P2, P2), "21": (P2, P1), "20": (P2, P0), "11": (P1, P1),
                          "21+": (P2, a1), "20+": (P2, a0), "11+": (a1, a1)}.items():
            self.S[k] += a.T @ b
        return self

    def add_kappa(self, kappa):
        return self.add_planes(*digit_planes_t(fixed_word_t(kappa)))

    def add_words(self, word):
        return self.add_planes(*digit_planes_t(word))

    def times(self, B):
        """The products of B copies of the points (exact: integers below 2^53)."""
        for k in self.S:
            self.S[k] *= B
        return self

    def products(self):
        """(A4, A3, A2, A3+, A2+)."""
        S = self.S
        return (S["22"], S["21"] + S["21"].T, S["20"] + S["20"].T + S["11"],
                S["21+"] + S["21+"].T, S["20+"] + S["20+"].T + S["11+"])

    def gram(self, C):
        """(G*, G+) as fp64 numpy arrays."""
        A4, A3, A2, A3p, A2p = self.products()
        c = gram_scale(C)
        G = c * (2.0 ** 32 * A4 + 2.0 ** 24 * A3 + 2.0 ** 16 * A2)
        Gp = c * (2.0 ** 32 * A4 + 2.0 ** 24 * A3p + 2.0 ** 16 * A2p)
        return G.cpu().numpy(), Gp.cpu().numpy()


def b_model(kappa, y, C):
    """(b*, b+) of one set of points: C sum_n kappa_nj y32_n and C sum_n |kappa_nj y32_n| (fp64, any device)."""
    k = kappa.to(torch.float64)
    y32 = y.to(torch.float32).to(torch.float64)
    return C * (k.T @ y32), C * (k.abs().T @ y32.abs())


def gram_gate(G, Gstar, Gplus, R):
    """Worst |G - G*| / (2^-53 G+) over the elements, asserted <= R; where G+ is 0, G must be exactly 0."""
    G = np.asarray(G)
    zero = Gplus == 0
    assert np.all(G[zero] == 0.0) and np.all(Gstar[zero] == 0.0), "a block the model holds at exact 0 is not 0"
    ratio = float((np.abs(G[~zero] - Gstar[~zero]) / (U53 * Gplus[~zero])).max()) if (~zero).any() else 0.0
    assert ratio <= R, "G is %.3g roundings off its exact integer model (budget %d)" % (ratio, R)
    return ratio


def b_gate(b, bstar, bplus, C, R_b):
    """Worst |b - b*| / (C (17 2^-24 + R_b 2^-53) sum |kappa y32|) over the elements, asserted <= 1; where the sum is 0, b
    must be exactly 0."""
    b, bstar, bplus = np.asarray(b), np.asarray(bstar), np.asarray(bplus)
    zero = bplus == 0
    assert np.all(b[zero] == 0.0)
    tol = (B_FP32_ULPS * U24 + R_b * U53) * bplus[~zero]        # bplus carries the factor C already
    ratio = float((np.abs(b[~zero] - bstar[~zero]) / tol).max()) if (~zero).any() else 0.0
    assert ratio <= 1.0, "b is %.3g of its bound off the model" % ratio
    return ratio


# ---- launch geometry: the mirrors the GPU cases are built from -----------------------------------------------------
def launch_windows(n_units, m_pad):
    """(windows, units per window) of one int8 launch (launch_stats_i8, csrc/api.cu): the planes of a window take
    kI8PlaneBytes per unit and active tile and at most kI8PlaneCapBytes; larger launches split into equal windows."""
    nt = m_pad // TILE
    cap_units = max(1, I8_PLANE_CAP_BYTES // (I8_PLANE_BYTES * nt))
    windows = -(-n_units // cap_units)
    return windows, -(-n_units // windows)


def launch_geometry(n, m, num_sms):
    """One launch over n points: windows, Gram slices, and the folds the fullest slice makes over all windows."""
    m_pad = -(-m // TILE) * TILE
    n_units = -(-n // UNIT_POINTS)
    windows, win_units = launch_windows(n_units, m_pad)
    g_slices = i8_slices(m_pad, num_sms, win_units)           # every window runs with the first window's slices
    folds = 0
    for w in range(windows):
        nu = min(win_units, n_units - w * win_units)
        folds += -(-(-(-nu // g_slices)) // FLUSH_UNITS)
    return dict(units=n_units, windows=windows, win_units=win_units, g_slices=g_slices, folds=folds)


def rounding_budget(launch_points, m, num_sms):
    """R of the G gate for a begin..finish window whose int8 launches cover launch_points points each: per launch,
    every fold add of the fullest slice, every Gram slice of the reduction and the G +=; plus R_CONST."""
    R = R_CONST
    for n in launch_points:
        g = launch_geometry(n, m, num_sms)
        R += g["folds"] + g["g_slices"] + 1
    return R


def b_rounding_budget(launch_points, num_sms):
    """R_b of the b gate: per launch, the fp64 adds across the units of a producer slice (at most all of them), the
    quad reduction, the producer slices (at most two per SM and tile), the windows and the b +=."""
    R = R_CONST
    for n in launch_points:
        R += -(-n // UNIT_POINTS) + 2 + 2 * num_sms + 1
    return R


def entry_launches(entry, n, d, x_is_f32):
    """Points of each launch one accumulate call makes: the device entry one launch, the host entry its chunk plan."""
    return [n] if entry == "device" else host_chunks(n, d, x_is_f32)


# ---- CPU emulation of one launch of the int8 Gram, and its mutants -----------------------------------------------
MUTANTS = ["drop P2'P2", "drop P2'P1", "drop P1'P2", "drop P2'P0", "drop P0'P2", "drop P1'P1", "weight P1'P1 2^17",
           "lost point", "lost unit", "fold stores", "slice missing", "tile misplaced"]


def emulate_gram(P, m, slices, C=1.0, mutant=None, flush=FLUSH_UNITS):
    """G of one launch over the points whose planes are P = (P0, P1, P2) (n x m, fp64), as gram_i8_kernel and
    gram_reduce_upper_kernel compute it: per slice of ceil(units / slices) units, the exact int32 accumulators of each
    fold of `flush` units go into the fp64 partial tile (the first fold stores, later ones add) at the mirror position
    (row from tile J, column from tile I); the reduction adds the slices in order and mirrors the upper triangle."""
    P0, P1, P2 = (np.array(p, dtype=np.float64) for p in P)
    n = len(P0)
    if mutant == "lost point":
        for p in (P0, P1, P2):
            p[n // 3] = 0.0
    if mutant == "lost unit":
        u = (n // UNIT_POINTS) // 2
        for p in (P0, P1, P2):
            p[u * UNIT_POINTS:(u + 1) * UNIT_POINTS] = 0.0
    units = -(-n // UNIT_POINTS)
    ups = -(-units // slices)
    gscale = gram_scale(C)
    w22, w21, w12, w20, w02, w11 = (0.0 if mutant == "drop " + k else 1.0 for k in ("P2'P2", "P2'P1", "P1'P2", "P2'P0",
                                                                                   "P0'P2", "P1'P1"))
    s11 = 2.0 if mutant == "weight P1'P1 2^17" else 1.0
    G = np.zeros((m, m))
    for s in range(slices):
        tile = np.zeros((m, m))
        for f, u0 in enumerate(range(s * ups, min((s + 1) * ups, units), flush)):
            a, b = u0 * UNIT_POINTS, min(u0 + flush, (s + 1) * ups, units) * UNIT_POINTS
            q0, q1, q2 = P0[a:b], P1[a:b], P2[a:b]
            # element [I row i, J column j]: the A operand is tile I's planes, the B operand tile J's
            acc4 = w22 * (q2.T @ q2)
            acc3 = w21 * (q2.T @ q1) + w12 * (q1.T @ q2)
            acc2 = w20 * (q2.T @ q0) + w02 * (q0.T @ q2) + s11 * w11 * (q1.T @ q1)
            v = gscale * (4294967296.0 * acc4 + 16777216.0 * acc3 + 65536.0 * acc2)
            tile = v.T if (f == 0 or mutant == "fold stores") else tile + v.T      # stored transposed
        if not (mutant == "slice missing" and s == 1):
            G = G + tile
    if mutant == "tile misplaced":                     # tile pair (I = 1, J = 0) written transposed inside its block
        G[:TILE, TILE:2 * TILE] = G[:TILE, TILE:2 * TILE].T.copy()
    U = np.triu(G)
    return U + np.triu(U, 1).T


def bench_family(n, m):
    """bench.py's data (make_shard, active_set) at n points: X ~ U[0,1)^16 in fp32, beta = sqrt(18 / 16), Z = m of the
    points; kappa rounded to fp32 from the fp64 kernel values (what the kernel computes, up to the distance half)."""
    d = 16
    X = np.random.default_rng(13).random((n, d), dtype=np.float32).astype(np.float64)
    Z = X[np.random.default_rng(7).permutation(n)[:m]]
    beta = np.sqrt(18.0 / d)
    q = (X ** 2).sum(1)[:, None] + (Z ** 2).sum(1)[None, :] - 2.0 * X @ Z.T
    K = np.exp(-beta ** 2 * np.maximum(q, 0.0))
    return K, K.astype(np.float32)


# ---- tests ----------------------------------------------------------------------------------------------------------
def test_mirror_constants_match_source():
    """kI8PlaneBytes, kI8PlaneCapBytes and the window split of launch_stats_i8, read from the sources."""
    internal = open(os.path.join(CSRC, "sgp_internal.h")).read()
    api = open(os.path.join(CSRC, "api.cu")).read()
    gram = open(os.path.join(CSRC, "gram_i8_wgmma.cu")).read()
    m = re.search(r"constexpr size_t kI8PlaneBytes = (\d+) \* kTile \* (\d+);", internal)
    assert int(m.group(1)) * TILE * int(m.group(2)) == I8_PLANE_BYTES
    m = re.search(r"constexpr size_t kI8PlaneCapBytes = size_t\((\d+)\) << (\d+);", internal)
    assert int(m.group(1)) << int(m.group(2)) == I8_PLANE_CAP_BYTES
    assert "const long long cap_units = std::max<long long>(1, kI8PlaneCapBytes / (kI8PlaneBytes * nt1));" in api
    assert "const long long n_windows = (n_units + cap_units - 1) / cap_units;" in api
    assert "const long long win_units = (n_units + n_windows - 1) / n_windows;" in api
    assert "const int g_slices = i8_slices(c->m_pad, c->num_sms, win_units);" in api
    assert "p.gscale = C * C / (4.0 * static_cast<double>(C0) * static_cast<double>(C0));" in gram
    # the kept products and their weights, in the order emulate_gram adds them
    body = re.search(r"wgmma_uu\(acc4, A2, B2, acc\);(.*?)\}", gram, re.S).group(0)
    assert re.findall(r"wgmma_(\w\w)\((acc\d), (A\d), (B\d)", body) == [
        ("uu", "acc4", "A2", "B2"), ("us", "acc3", "A2", "B1"), ("su", "acc3", "A1", "B2"), ("us", "acc2", "A2", "B0"),
        ("su", "acc2", "A0", "B2"), ("ss", "acc2", "A1", "B1")]
    assert ("p.gscale * (4294967296.0 * static_cast<double>(acc4[e]) + 16777216.0 * static_cast<double>(acc3[e]) +"
            in gram)


def test_launch_windows_mirror():
    # m = 4000: 32 tiles, 5461 units (349504 points) per window
    assert launch_windows(5461, 4096) == (1, 5461) and launch_windows(5462, 4096) == (2, 2731)
    g = launch_geometry(700_000, 4000, H100_SXM_SMS)
    assert g["windows"] == 3 and g["units"] == 10938
    # bench.py's configs3 shard on the device entry: two windows
    assert launch_geometry(1_250_000, 2000, H100_SXM_SMS)["windows"] == 2
    assert launch_geometry(1_000_000, 1000, H100_SXM_SMS) == dict(units=15625, windows=1, win_units=15625, g_slices=11,
                                                                  folds=4)
    for n, m in ((1, 1), (64, 128), (65, 4000), (10 ** 7, 4000), (123_457, 1300)):
        g = launch_geometry(n, m, H100_SXM_SMS)
        assert (g["windows"] - 1) * g["win_units"] < g["units"] <= g["windows"] * g["win_units"]
        assert g["win_units"] * (-(-m // TILE)) * I8_PLANE_BYTES <= I8_PLANE_CAP_BYTES or g["win_units"] == 1
    # every GPU case stays far inside 1e-12 relative
    assert rounding_budget([1_250_000], 2000, H100_SXM_SMS) * U53 < 1e-13
    assert rounding_budget(host_chunks(1_000_000, 16, True), 1000, H100_SXM_SMS) * U53 < 1e-13


def _kappa_grid():
    kappa = np.unique(np.concatenate([np.linspace(0.0, 1.0 + 2e-3, 2_000_001, dtype=np.float32),
                                      np.float32(1.0) + np.arange(-4096, 4097, dtype=np.float32) * np.float32(2 ** -23),
                                      np.float32(2.0) ** -np.arange(0, 150, dtype=np.float32)]))
    return kappa[kappa <= np.float32(1.0 + 2e-3)]


def test_torch_port_matches_numpy_bit_for_bit():
    """On the grid of test_fixed_point_digits_exact_in_range and past the encoding's margin (1 + 2.05e-3 up to 2)."""
    past = np.concatenate([np.float32(1.0) + np.arange(0, 40000, dtype=np.float32) * np.float32(2 ** -23),
                           np.linspace(1.0 + 2.05e-3, 2.0, 100_001, dtype=np.float32)])
    for kappa in (_kappa_grid(), past):
        w_np = fixed_word(kappa)
        w_t = fixed_word_t(torch.from_numpy(kappa))
        assert np.array_equal(w_t.numpy(), w_np.astype(np.int64))
        for a, b in zip(digit_planes_t(w_t), digit_planes(w_np)):
            assert np.array_equal(a.numpy(), b.astype(np.float64))
    # the words past the margin overflow into the exponent: the port keeps those words too
    assert np.any(((fixed_word(past) >> np.uint64(24)) & np.uint64(0xFF)) != 150)


def test_model_against_python_integers():
    """On small random word matrices (any 32-bit word whose low bit is 0, overflowed or not): the integer products equal
    the per-point sums in Python ints, and G* the exact rational C^2 / (4 C0^2) (...) to within a few roundings."""
    rng = np.random.default_rng(1)
    for n, m, C in ((1, 1, 1.0), (7, 3, 0.37), (130, 5, 17.0), (64, 9, 0.25)):
        words = rng.integers(0, 2 ** 31, (n, m), dtype=np.int64) << 1
        model = GramModel(m).add_words(torch.from_numpy(words))
        A4, A3, A2 = (a.numpy() for a in model.products()[:3])
        G, Gp = model.gram(C)
        P0, P1, P2 = (np.array(p, dtype=object) for p in digit_planes(words.astype(np.uint64)))
        c = Fraction(C) ** 2 / (4 * Fraction(float(FIXED_C0)) ** 2)
        for i in range(m):
            for j in range(m):
                a4 = sum(P2[:, i] * P2[:, j])
                a3 = sum(P2[:, i] * P1[:, j] + P1[:, i] * P2[:, j])
                a2 = sum(P2[:, i] * P0[:, j] + P0[:, i] * P2[:, j] + P1[:, i] * P1[:, j])
                assert (A4[i, j], A3[i, j], A2[i, j]) == (a4, a3, a2)
                exact = c * (2 ** 32 * a4 + 2 ** 24 * a3 + 2 ** 16 * a2)
                plus = c * (2 ** 32 * a4 + 2 ** 24 * sum(abs(P2[:, i] * P1[:, j]) + abs(P1[:, i] * P2[:, j]))
                            + 2 ** 16 * sum(abs(P2[:, i] * P0[:, j]) + abs(P0[:, i] * P2[:, j]) + abs(P1[:, i] * P1[:, j])))
                assert abs(Fraction(G[i, j]) - exact) <= 6 * U53 * plus
                assert abs(Fraction(Gp[i, j]) - plus) <= 6 * U53 * plus


def test_fp64_products_exact_at_the_largest_totals():
    """The digits that maximise every product (P2 = 255, P1 = -128, P0 = -128 or 126), summed in chunks of 65536 points up
    to 2^21 points -- more than any GPU case models -- in fp64 matmuls: equal to the closed form in integers, and the
    largest total, 81664 * 2^21 per element, is far below 2^53."""
    npts, chunks, m = 65536, 32, 4
    P2 = torch.full((npts, m), 255.0, dtype=torch.float64)
    P1 = torch.full((npts, m), -128.0, dtype=torch.float64)
    P0 = torch.tensor([-128.0, 126.0, -128.0, 126.0], dtype=torch.float64).repeat(npts, 1)
    model = GramModel(m)
    for _ in range(chunks):
        model.add_planes(P0, P1, P2)
    N = npts * chunks
    A4, A3, A2, A3p, A2p = (a.numpy() for a in model.products())
    p0 = np.array([-128, 126, -128, 126], dtype=object)
    for i in range(m):
        for j in range(m):
            assert A4[i, j] == 255 * 255 * N and A3[i, j] == 2 * 255 * -128 * N and A3p[i, j] == 2 * 255 * 128 * N
            assert A2[i, j] == (255 * (p0[i] + p0[j]) + 128 * 128) * N
            assert A2p[i, j] == (255 * (abs(p0[i]) + abs(p0[j])) + 128 * 128) * N
    assert A2p.max() == 81664 * N and 81664 * N < 2 ** 53 / 1000


@pytest.fixture(scope="module")
def family():
    n, m = 40960, 256
    K, kappa = bench_family(n, m)
    P = digit_planes(fixed_word(kappa))
    model = GramModel(m).add_kappa(torch.from_numpy(kappa))
    Gs, Gp = model.gram(1.0)
    return dict(n=n, m=m, K=K, P=P, Gs=Gs, Gp=Gp, G0=K.T @ K)


def rel(a, b):
    return float(np.abs(a - b).max() / np.abs(b).max())


@pytest.mark.parametrize("slices", [1, 16])
def test_emulated_kernel_passes_the_gate(family, slices):
    """The kernel as written, at the geometry the launch mirror gives this shape (16 slices of 40 units) and at one slice
    (two folds: 400 units, then 240)."""
    f = family
    units = -(-f["n"] // UNIT_POINTS)
    if slices == 16:
        assert i8_slices(f["m"], H100_SXM_SMS, units) == 16
    G = emulate_gram(f["P"], f["m"], slices)
    R = R_CONST + -(-(-(-units // slices)) // FLUSH_UNITS) + slices + 1
    ratio = gram_gate(G, f["Gs"], f["Gp"], R)
    print("emulated kernel, %d slices: worst %.2f roundings of G+ (budget %d); oracle gap %.1e" % (
        slices, ratio, R, rel(G, f["G0"])))
    assert np.array_equal(G, G.T)
    assert rel(G, f["G0"]) < 1e-7


@pytest.mark.parametrize("mutant", MUTANTS)
def test_mutants_fail_the_gate(family, mutant):
    """Each mutant of the emulated kernel misses the model by at least 1e6 times the rounding budget.  The fold mutant
    needs two folds in a slice, so every mutant runs on one slice but the missing-slice one (16 slices)."""
    f = family
    slices = 16 if mutant == "slice missing" else 1
    units = -(-f["n"] // UNIT_POINTS)
    R = R_CONST + -(-(-(-units // slices)) // FLUSH_UNITS) + slices + 1
    G = emulate_gram(f["P"], f["m"], slices, mutant=mutant)
    nz = f["Gp"] > 0
    ratio = float((np.abs(G - f["Gs"])[nz] / (U53 * f["Gp"][nz])).max())
    print("%-18s worst %.1e roundings of G+ (budget %d); oracle gap %.1e" % (mutant, ratio, R, rel(G, f["G0"])))
    assert ratio >= 1e6 * R
    with pytest.raises(AssertionError):
        gram_gate(G, f["Gs"], f["Gp"], R)


def test_a_dropped_product_class_passes_the_oracle_gates(family):
    """Why the model is needed: on bench.py's own data, dropping the whole P2'P0 + P0'P2 class stays inside the oracle
    gates of the existing int8 tests (measured against max |G|: 8.0e-7 here; 8e-7 to 1.6e-6 over other active sets of
    the same data), while the model rejects it by about nine orders of magnitude."""
    f = family
    G = emulate_gram(f["P"], f["m"], 16, mutant=None)
    P0, P1, P2 = f["P"]
    zero = np.zeros_like(P0)
    # P2'P0 + P0'P2 dropped: the planes without P0 keep the other four products
    G_mut = emulate_gram((zero, P1, P2), f["m"], 16)
    G_p1 = emulate_gram(f["P"], f["m"], 16, mutant="drop P1'P1")
    G_pt = emulate_gram(f["P"], f["m"], 16, mutant="lost point")
    gaps = [rel(g, f["G0"]) for g in (G, G_mut, G_p1, G_pt)]
    nz = f["Gp"] > 0
    model_gap = float((np.abs(G_mut - f["Gs"]) / np.abs(f["Gs"]).max()).max())
    elementwise = float((np.abs(G_mut - f["Gs"])[nz] / np.abs(f["Gs"])[nz]).max())
    print("oracle gap: as written %.1e, no P2'P0 class %.1e, no P1'P1 %.1e, one point lost %.1e; "
          "no P2'P0 class vs the model %.1e of max|G|, %.1e elementwise" % (*gaps, model_gap, elementwise))
    assert gaps[0] < 1e-7
    assert gaps[1] < TOL_STATS and gaps[1] < TOL_I8                  # passes both oracle gates ...
    assert gaps[2] > TOL_I8 and gaps[3] > TOL_I8
    with pytest.raises(AssertionError):                              # ... and fails the model's
        gram_gate(G_mut, f["Gs"], f["Gp"], R_CONST + 1 + 16 + 1)


def test_b_gate_on_emulated_producer():
    """The producer's b: per unit and lane, an fp32 FMA chain over 16 points, then fp64 across units and lanes.  The
    emulation passes the b gate; without one unit's contribution it does not."""
    rng = np.random.default_rng(5)
    n, m = 64 * 300, 40
    _, kappa = bench_family(n, m)
    y = np.sin(rng.random(n) * 6.0) + 0.1 * rng.standard_normal(n)
    y32 = y.astype(np.float32)
    C = 0.37
    f32 = np.float32
    lanes = np.zeros(m)
    lost = np.zeros(m)
    for u in range(n // 64):
        for lane in range(4):                 # points 8j + 2 lane + {0, 1}
            b0 = np.zeros(m, dtype=f32)
            for j in range(8):
                p = u * 64 + 8 * j + 2 * lane
                # fmaf(T0, y0, fmaf(T1, y1, b0)): each FMA rounds once (emulated in fp64, exact before the rounding)
                b0 = (kappa[p + 1].astype(np.float64) * y32[p + 1] + b0).astype(f32)
                b0 = (kappa[p].astype(np.float64) * y32[p] + b0).astype(f32)
            lanes += b0.astype(np.float64)
            if u != 150:
                lost += b0.astype(np.float64)
    bstar, bplus = (t.numpy() for t in b_model(torch.from_numpy(kappa), torch.from_numpy(y), C))
    R_b = b_rounding_budget([n], H100_SXM_SMS)
    ratio = b_gate(C * lanes, bstar, bplus, C, R_b)
    print("emulated producer b: %.1e of the bound" % ratio)
    with pytest.raises(AssertionError):
        b_gate(C * lost, bstar, bplus, C, R_b)


def test_points_for_units_reaches_the_fold_cases():
    """The fold cases of the GPU file: one slice of exactly 399 .. 1201 units at m = 1300 on this SM count."""
    for units in (399, 400, 401, 800, 801, 1201):
        n = points_for_units(1300, units, H100_SXM_SMS)
        g = launch_geometry(n, 1300, H100_SXM_SMS)
        assert g["windows"] == 1 and -(-g["units"] // g["g_slices"]) == units
        assert g["folds"] == -(-units // FLUSH_UNITS)
