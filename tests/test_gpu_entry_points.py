"""The entry points bench.py times, against the fp64 oracle (run on an H100: `pytest -m gpu`).

`sgp_stats_accumulate_device` (one launch over a device-resident shard) and `sgp_kmn_sweep_device` are what the
benchmark measures; the rest of the suite calls their host forms.  The device entry gives every point slice of the int8
Gram far more 64-point units than the host entry's chunks do (1421 on bench.py's configs1 shape against at most 367
anywhere else), so the kernel folds its exact int32 accumulators into the fp64 partial tile several times: the first
fold stores, every later one adds.  The shapes below are picked with the launch-geometry mirror of test_host_logic.py
from the SM count of the device, so that one slice runs through 399, 400, 401, 800, 801 and more than 1200 units.

Inputs are torch CUDA tensors, as in bench.py.  Oracles:
  * statistics: oracle.cpu_baseline.stats_parallel (configs1), or sums of the oracle's statistics of a base block for
    shards built by repeating it (G and b are sums over points), or the closed form N k k' for identical points;
  * the K_nm sweep: the oracle's cross_kernel, element by element;
  * prediction: the oracle's GaussianProjectedProcessRawPredictor with its own magic vector and matrix.

Tolerances: G, b 1e-6 of their largest element (TOL_STATS), posterior mean / variance 1e-5 (TOL_PRED), as in
test_gpu_parity.py; TOL_I8 = 3e-6 where no averaging over points happens; two entries or two call splits on the same
data differ in the fp64 summation order only (1e-12); prediction on the oracle's magic vector and matrix is all-fp64
(1e-11 of the sum of the magnitudes it adds up).  The sweep's elements are checked one by one against a relative bound
that grows with the scaled squared norms s = |x^|^2 + |z^|^2 of the pair (x^ = sqrt(log2 e) beta (x - centre)):
    |K - K0| / K0 <= 3e-7 + ln 2 * SWEEP_ULPS * 2^-24 * s.
3e-7 covers ex2.approx and the fp32 product with C.  The exponent T carries the 22-bit hi/lo fp16 split of x^ and z^
(|dT| <= 2^-21 |x^ - z^| (|x^| + |z^|) <= 16 * 2^-24 s) and the fp32 accumulation of terms as large as s.  Measured on
an H100: slopes up to 12.9 in use, element errors up to 5.2e-6 (d = 1, s ~ 13), so a flat 2.5e-6 does not hold.
"""
import numpy as np
import pytest
import torch

import oracle
import spark_gp_b200 as sg
from oracle.cpu_baseline import stats_parallel
from spark_gp_b200 import _native as N
from test_host_logic import points_for_units, units_per_slice

pytestmark = pytest.mark.gpu

TOL_STATS, TOL_PRED, TOL_I8, TOL_ORDER, TOL_PREDICT_F64 = 1e-6, 1e-5, 3e-6, 1e-12, 1e-11
SWEEP_ULPS = 24
LOG2E = np.log2(np.e)
SIGMA2 = 1e-4
MODES = {"auto": N.SGP_PREC_AUTO, "i8": N.SGP_PREC_I8, "i8_direct": N.SGP_PREC_I8_DIRECT, "f64": N.SGP_PREC_F64,
         "f64_strict": N.SGP_PREC_F64_STRICT}


@pytest.fixture(scope="module")
def eng():
    e = sg.ProjectedProcessEngine(0)
    yield e
    e.close()


@pytest.fixture(scope="module")
def num_sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


def rel(a, b):
    return float(np.abs(np.asarray(a) - np.asarray(b)).max() / max(np.abs(np.asarray(b)).max(), 1e-300))


def to_device(a):
    t = torch.from_numpy(np.ascontiguousarray(a)).cuda()
    torch.cuda.synchronize()
    return t


def stats_device(eng, kernel, Xd, yd, Z, precision):
    eng.set_precision(precision)
    eng.begin(kernel, Z)
    eng.accumulate_ptr(Xd.data_ptr(), Xd.dtype == torch.float32, yd.data_ptr(), len(Xd), device=True)
    path = eng.last_path()
    G, b = eng.finish()
    return G, b, path


def stats_host(eng, kernel, X, y, Z, precision):
    eng.set_precision(precision)
    eng.begin(kernel, Z)
    eng.accumulate(X, y)
    path = eng.last_path()
    G, b = eng.finish()
    return G, b, path


def ard_pair(beta, C=1.0, eye=1.0):
    """(library kernel, oracle kernel factory): C * ARD(beta) + eye.const * Eye + sigma2.const * Eye."""
    k = C * sg.ARDRBFKernel(beta) + sg.const(eye) * sg.EyeKernel() + sg.const(SIGMA2) * sg.EyeKernel()
    ok = lambda: C * oracle.ARDRBFKernel(beta) + oracle.const(eye) * oracle.EyeKernel() + oracle.const(SIGMA2) * oracle.EyeKernel()
    return k, ok


def oracle_rows(ok, Z, X):
    """The oracle's crossKernel of the points X against the active set Z: len(X) x m, fp64."""
    return ok().set_hyperparameters(ok().get_hyperparameters()).set_training_vectors(Z).cross_kernel(
        np.asarray(X, dtype=np.float64))


class TiledOracle:
    """Statistics of shards built from copies of one base block: G(n) = r K'K + K[:s]'K[:s] for n = r * len(base) + s,
    with K the oracle's cross kernel of the base block against Z (PGPH:28-29 summed over points)."""

    def __init__(self, ok, Xb, yb, Z):
        self.K = oracle_rows(ok, Z, Xb)
        self.y = yb
        self.G1, self.b1 = self.K.T @ self.K, self.K.T @ yb

    def stats(self, n):
        r, s = divmod(n, len(self.K))
        Ks = self.K[:s]
        return r * self.G1 + Ks.T @ Ks, r * self.b1 + Ks.T @ self.y[:s]


def tiled(a, n):
    reps = -(-n // len(a))
    return np.concatenate([a] * reps)[:n]


# ---------------- a. device-resident statistics against the oracle ------------------------------------------------------
def bench_shard(name):
    """bench.py's make_shard(name, rank 0) and active_set(name): X ~ U[0,1)^d in fp32, y = sin(sum x) + 0.1 eps."""
    n, d, m = {"configs1": (1_000_000, 16, 1000), "configs3": (1_250_000, 32, 2000)}[name]
    rng = np.random.default_rng(13)
    X = rng.random((n, d), dtype=np.float32)
    y = np.sin(X.astype(np.float64).sum(1)) + 0.1 * rng.standard_normal(n)
    Z = X[np.random.default_rng(7).permutation(n)[:m]].astype(np.float64)
    return X, y, Z


@pytest.fixture(scope="module")
def configs1():
    X, y, Z = bench_shard("configs1")
    d = X.shape[1]
    k, ok = ard_pair(np.full(d, np.sqrt(18.0 / d)))
    theta = ok().get_hyperparameters()
    G0, b0, _ = stats_parallel(X.astype(np.float64), y, Z, ok, theta, 100)
    kernel0 = ok().set_hyperparameters(theta).set_training_vectors(Z)
    mv0, mm0 = oracle.get_magic_vector(kernel0, G0, b0)
    Xt = np.random.default_rng(99).random((1000, d))
    m0, v0 = oracle.GaussianProjectedProcessRawPredictor(mv0, mm0, kernel0).predict_many(Xt)
    return dict(X=X, y=y, Z=Z, k=k, G0=G0, b0=b0, Xt=Xt, m0=m0, v0=v0,
                Xd={np.float32: to_device(X), np.float64: to_device(X.astype(np.float64))}, yd=to_device(y))


@pytest.mark.parametrize("dtype", [np.float32, np.float64], ids=["fp32", "fp64"])
@pytest.mark.parametrize("mode", list(MODES))
def test_device_stats_configs1_vs_oracle(eng, configs1, mode, dtype):
    """bench.py's configs1 shard (1M x 16, m = 1000) through the device entry in every mode, against the oracle: G, b to
    1e-6, posterior mean and variance at 1000 held-out points to 1e-5.  The host entry on the same data differs in the
    slicing only, so in the fp64 summation order: 1e-12."""
    c = configs1
    G, b, path = stats_device(eng, c["k"], c["Xd"][dtype], c["yd"], c["Z"], MODES[mode])
    if mode == "auto":
        assert path in (N.SGP_PREC_I8, N.SGP_PREC_I8_DIRECT)
    else:
        assert path == MODES[mode]
    eng.magic()
    mean, var = eng.predict(c["Xt"])
    eg, eb, em, ev = rel(G, c["G0"]), rel(b, c["b0"]), rel(mean, c["m0"]), float(np.abs(var / c["v0"] - 1).max())
    Gh, bh, path_h = stats_host(eng, c["k"], c["X"].astype(dtype), c["y"], c["Z"], MODES[mode])
    print("configs1 device [%s, %s]: dG=%.2e db=%.2e dmean=%.2e dvar=%.2e; host vs device dG=%.1e db=%.1e" % (
        mode, dtype.__name__, eg, eb, em, ev, rel(Gh, G), rel(bh, b)))
    assert eg < TOL_STATS and eb < TOL_STATS
    assert em < TOL_PRED and ev < TOL_PRED
    assert np.array_equal(G, G.T)
    assert path_h == path
    assert rel(Gh, G) < TOL_ORDER and rel(bh, b) < TOL_ORDER


def test_device_and_host_calls_share_one_window(eng, configs1):
    """A device call and a host call in one begin..finish window add up to the single call over the whole shard."""
    c = configs1
    G1, b1, _ = stats_device(eng, c["k"], c["Xd"][np.float32], c["yd"], c["Z"], N.SGP_PREC_I8)
    cut = 400_000
    eng.begin(c["k"], c["Z"])
    eng.accumulate_ptr(c["Xd"][np.float32].data_ptr(), True, c["yd"].data_ptr(), cut, device=True)
    eng.accumulate(c["X"][cut:], c["y"][cut:])
    G2, b2 = eng.finish()
    print("device(400k) + host(600k) vs one device call: dG=%.1e db=%.1e" % (rel(G2, G1), rel(b2, b1)))
    assert rel(G2, G1) < TOL_ORDER and rel(b2, b1) < TOL_ORDER


@pytest.fixture(scope="module")
def configs3():
    """bench.py's configs3 shape (1.25M x 32, m = 2000) as 61 shuffled copies of a 20480-point block: the oracle is 61
    times the block's statistics (the block alone holds 1e-6 in test_i8_config_shapes_vs_oracle)."""
    rng = np.random.default_rng(103)
    nb, d, m, reps = 20480, 32, 2000, 61
    Xb = rng.random((nb, d), dtype=np.float32)
    yb = np.sin(Xb.astype(np.float64).sum(1)) + 0.1 * rng.standard_normal(nb)
    Z = Xb[rng.permutation(nb)[:m]].astype(np.float64)
    k, ok = ard_pair(np.full(d, np.sqrt(18.0 / d)))
    G0, b0 = TiledOracle(ok, Xb, yb, Z).stats(nb * reps)
    order = rng.permutation(nb * reps)
    X, y = np.tile(Xb, (reps, 1))[order], np.tile(yb, reps)[order]
    return dict(Z=Z, k=k, G0=G0, b0=b0, yd=to_device(y),
                Xd={np.float32: to_device(X), np.float64: to_device(X.astype(np.float64))})


@pytest.mark.parametrize("mode,dtype", [("auto", np.float32), ("i8", np.float32), ("i8_direct", np.float32),
                                        ("f64", np.float32), ("i8", np.float64)])
def test_device_stats_configs3_vs_oracle(eng, num_sms, configs3, mode, dtype):
    """configs3 through the device entry: a slice runs through 1220 units, past three folds that add."""
    c = configs3
    Z, k, G0, b0, Xd = c["Z"], c["k"], c["G0"], c["b0"], c["Xd"][dtype]
    m, d = Z.shape
    assert max(units_per_slice(len(Xd), m, d, device=True, num_sms=num_sms)) > 1200
    G, b, path = stats_device(eng, k, Xd, c["yd"], Z, MODES[mode])
    assert path in ((N.SGP_PREC_I8, N.SGP_PREC_I8_DIRECT) if mode == "auto" else (MODES[mode],))
    eg, eb = rel(G, G0), rel(b, b0)
    print("configs3 device [%s, %s]: dG=%.2e db=%.2e" % (mode, np.dtype(dtype).name, eg, eb))
    assert eg < TOL_STATS and eb < TOL_STATS
    assert np.array_equal(G, G.T)


@pytest.fixture(scope="module")
def fold_block():
    """A 12288-point block of bench-like data (d = 16) and m = 1300 active points: m_pad = 1408 is 11 tiles, 132 CTAs
    per slice."""
    rng = np.random.default_rng(211)
    nb, d, m = 12288, 16, 1300
    Xb = rng.random((nb, d), dtype=np.float32)
    yb = np.sin(Xb.astype(np.float64).sum(1)) + 0.1 * rng.standard_normal(nb)
    Z = Xb[rng.permutation(nb)[:m]].astype(np.float64)
    k, ok = ard_pair(np.full(d, np.sqrt(18.0 / d)))
    return dict(Xb=Xb, yb=yb, Z=Z, k=k, oracle=TiledOracle(ok, Xb, yb, Z))


@pytest.mark.parametrize("units,jag", [(399, 0), (400, 17), (401, 0), (800, 0), (801, 5), (1201, 63)])
def test_device_stats_across_fold_boundaries(eng, num_sms, fold_block, units, jag):
    """One point slice runs exactly `units` units: the int32 accumulators are folded into the fp64 tile after 400 units
    and at the end of the slice.  Tensor-core and direct distances, against the tiled oracle at 1e-6."""
    c = fold_block
    m, d = c["Z"].shape
    n = points_for_units(m, units, num_sms, jag)
    assert units_per_slice(n, m, d, device=True, num_sms=num_sms) == [units]
    X, y = tiled(c["Xb"], n), tiled(c["yb"], n)
    G0, b0 = c["oracle"].stats(n)
    Xd, yd = to_device(X), to_device(y)
    for mode in ("i8", "i8_direct"):
        G, b, path = stats_device(eng, c["k"], Xd, yd, c["Z"], MODES[mode])
        assert path == MODES[mode]
        eg, eb = rel(G, G0), rel(b, b0)
        print("fold boundary: %d units per slice (n=%d, %d SMs) [%s]: dG=%.2e db=%.2e" % (units, n, num_sms, mode, eg, eb))
        assert eg < TOL_STATS and eb < TOL_STATS


def test_host_stats_one_chunk_across_folds(eng, num_sms):
    """d <= 2: the host entry's ~16 MB chunk holds all 1.3M points, so one launch's slice runs through 20313 units
    (132 SMs) -- the host entry's own way past the fold."""
    rng = np.random.default_rng(307)
    nb, d, m, n = 8192, 2, 1300, 1_300_000
    Xb = rng.random((nb, d), dtype=np.float32)
    yb = np.sin(Xb.astype(np.float64).sum(1)) + 0.1 * rng.standard_normal(nb)
    Z = Xb[rng.permutation(nb)[:m]].astype(np.float64)
    k, ok = ard_pair(np.full(d, np.sqrt(18.0 / d)))
    G0, b0 = TiledOracle(ok, Xb, yb, Z).stats(n)
    X, y = tiled(Xb, n), tiled(yb, n)
    assert max(units_per_slice(n, m, d, True, device=False, num_sms=num_sms)) > 1200
    for mode in ("i8", "i8_direct"):
        G, b, path = stats_host(eng, k, X, y, Z, MODES[mode])
        assert path == MODES[mode]
        print("host entry, 1.3M x 2 in one chunk [%s]: dG=%.2e db=%.2e" % (mode, rel(G, G0), rel(b, b0)))
        assert rel(G, G0) < TOL_STATS and rel(b, b0) < TOL_STATS


def test_auto_gate_on_device_entry(eng):
    """AUTO's magnitude gate runs on the device entry too: large scaled norms take the fp64 kernel (and match the
    oracle); forced I8 on coordinates outside the fp16 operand range raises OperandRangeError at finish."""
    rng = np.random.default_rng(401)
    n, d, m = 100_000, 8, 256
    X = rng.random((n, d), dtype=np.float32) * np.float32(6.0)          # scaled squared norms x 36: over the budget
    y = rng.standard_normal(n)
    Z = X[:m].astype(np.float64)
    k, ok = ard_pair(np.full(d, np.sqrt(18.0 / d)))
    G, b, path = stats_device(eng, k, to_device(X), to_device(y), Z, N.SGP_PREC_AUTO)
    assert path == N.SGP_PREC_F64
    G0, b0 = TiledOracle(ok, X, y, Z).stats(n)
    assert rel(G, G0) < TOL_STATS and rel(b, b0) < TOL_STATS
    Xf = rng.standard_normal((n, d)) * 1e4
    eng.set_precision(N.SGP_PREC_I8)
    eng.begin(k, Xf[:m])
    Xfd, yd = to_device(Xf), to_device(y)
    eng.accumulate_ptr(Xfd.data_ptr(), False, yd.data_ptr(), n, device=True)
    with pytest.raises(sg.OperandRangeError):
        eng.finish()
    eng.set_precision(N.SGP_PREC_AUTO)


# ---------------- b. the int32 accumulator bound, in closed form ---------------------------------------------------------
# all N points are x0; active point j sits where k(x0, z_j) = kappa_j, so G = N k k' and b = k sum(y) exactly.  u_worst
# has the digits s2 = 255, s1 = -128, s0 = 63: the largest 2^16-class product (80644 per point, test_host_logic.py).
FIXED_C0 = 8355000.0
GATE = 4096.0                      # kI8TensorR2Max: largest scaled squared norm the tensor-core distance mode takes
U_WORST = 255 * 2 ** 15 - 128 * 2 ** 7 + 63
KAPPAS = [1.0, U_WORST / FIXED_C0, (254 * 2 ** 15 + 127 * 2 ** 7 + 63) / FIXED_C0, (128 * 2 ** 15 - 128 * 2 ** 7 - 64) / FIXED_C0,
          0.75, 0.5, 0.25, 0.1]


@pytest.mark.parametrize("units", [400, 1201])
def test_accumulator_bound_closed_form(eng, num_sms, units):
    d, C = 4, 1.7
    beta = np.array([1.3, 0.7, 1.1, 0.9])
    x0 = np.array([0.25, 0.5, 0.375, 0.75], dtype=np.float32)
    Z = np.tile(x0.astype(np.float64), (len(KAPPAS), 1))
    Z[:, 0] += np.sqrt(-np.log(KAPPAS)) / beta[0]
    k, ok = ard_pair(beta, C=C, eye=0.3)
    kvec = oracle_rows(ok, Z, x0[None, :])[0]
    assert np.allclose(kvec / C, KAPPAS, rtol=1e-12)
    n = points_for_units(len(KAPPAS), units, num_sms)
    assert units_per_slice(n, len(KAPPAS), d, device=True, num_sms=num_sms) == [units]
    X = np.tile(x0, (n, 1))
    y = 1.0 + (np.arange(n) % 3)
    G0, b0 = n * np.outer(kvec, kvec), kvec * y.sum()
    Xd, yd = to_device(X), to_device(y)
    for mode in ("i8", "i8_direct"):
        for entry in ("device", "host"):
            if entry == "device":
                G, b, path = stats_device(eng, k, Xd, yd, Z, MODES[mode])
            else:
                G, b, path = stats_host(eng, k, X, y, Z, MODES[mode])
            assert path == MODES[mode]
            print("closed form, N=%d identical points (%d units per slice) [%s, %s]: dG=%.2e db=%.2e" % (
                n, units, mode, entry, rel(G, G0), rel(b, b0)))
            assert rel(G, G0) < TOL_I8 and rel(b, b0) < TOL_I8


# ---------------- c. the K_nm sweep against the oracle's cross kernel ----------------------------------------------------
def sweep_data(family, n, m, d, rng):
    if family == "standardised":
        X = rng.standard_normal((n, d))
        target = 1.5                                                   # sum_k beta_k^2 var(x_k)
    else:
        X = rng.random((n, d)) + (1e3 if family == "offset" else 0.0)
        target = 18.0 / 12.0
    Z = X[rng.permutation(n)[:m]] if n >= m else np.vstack([X, X[rng.integers(0, n, m - n)] + 0.1 * rng.random((m - n, d))])
    var = 1.0 if family == "standardised" else 1.0 / 12.0
    return X, Z.copy(), target / var


SWEEP_CASES = [   # d, m, n, data family, X dtype, kernel, entry
    (1, 1, 1, "cube", "fp32", "ard", "host"),
    (2, 64, 63, "offset", "fp64", "rbf", "host"),
    (15, 127, 64, "standardised", "fp32", "ard", "host"),
    (16, 128, 65, "cube", "fp64", "rbf", "host"),
    (17, 129, 65535, "offset", "fp32", "ard", "host"),
    (31, 4000, 65, "standardised", "fp64", "ard", "host"),
    (32, 129, 65536, "cube", "fp32", "rbf", "host"),
    (16, 127, 65537, "standardised", "fp64", "ard", "host"),
    (2, 128, 131073, "cube", "fp32", "ard", "host"),
    (1, 4000, 63, "offset", "fp64", "rbf", "host"),
    (32, 64, 131073, "standardised", "fp32", "ard", "device"),
    (17, 1, 65537, "cube", "fp64", "rbf", "device"),
    (15, 129, 1, "offset", "fp32", "rbf", "device"),
    (31, 128, 65536, "standardised", "fp32", "ard", "device"),
    (1, 127, 65535, "cube", "fp64", "ard", "device"),
    (16, 64, 64, "offset", "fp32", "ard", "device"),
]


def sweep_kernel(kind, d, sum_beta2, rng):
    """ARD with non-uniform beta (C = 2.5) or RBF (C = 0.7), each with Eye terms, which must contribute nothing."""
    if kind == "ard":
        u = rng.uniform(0.5, 1.5, d)
        beta = u * np.sqrt(sum_beta2 / (u ** 2).sum())
        return (2.5 * sg.ARDRBFKernel(beta) + sg.const(0.3) * sg.EyeKernel() + sg.const(SIGMA2) * sg.EyeKernel(),
                lambda: 2.5 * oracle.ARDRBFKernel(beta) + oracle.const(0.3) * oracle.EyeKernel() + oracle.const(SIGMA2) * oracle.EyeKernel(),
                2.5, beta)
    sigma = 1.0 / (np.sqrt(2.0) * np.sqrt(sum_beta2 / d))
    return (0.7 * sg.RBFKernel(sigma) + sg.const(1e-3) * sg.EyeKernel(),
            lambda: 0.7 * oracle.RBFKernel(sigma) + oracle.const(1e-3) * oracle.EyeKernel(), 0.7,
            np.full(d, 1.0 / (np.sqrt(2.0) * sigma)))


def sweep_check(K, X, Z, ok, C, beta):
    """Asserts the element-wise bound of the module docstring on the sweep's K (rows X) against the oracle; returns
    (max relative error, max of (error - 3e-7) / (ln 2 * 2^-24 * s): the bound's slope in use, in units of 2^-24)."""
    K = np.asarray(K, dtype=np.float64)
    K0 = oracle_rows(ok, Z, X)
    scale = np.sqrt(LOG2E) * beta
    centre = Z.mean(0)
    s = (((np.asarray(X, dtype=np.float64) - centre) * scale) ** 2).sum(1)[:, None] + (((Z - centre) * scale) ** 2).sum(1)[None, :]
    big = K0 > 1e-30 * C                       # fp32 flushes smaller values: those only have to be tiny
    assert np.all(np.abs(K[~big]) <= 1e-29 * C)
    if not big.any():
        return 0.0, 0.0
    err = np.abs(K[big] - K0[big]) / K0[big]
    excess = np.maximum(err - 3e-7, 0.0)
    slope = np.divide(excess, np.log(2.0) * 2.0 ** -24 * s[big], out=np.where(excess > 0, np.inf, 0.0), where=s[big] > 0)
    assert slope.max() <= SWEEP_ULPS, (float(err.max()), float(slope.max()))
    return float(err.max()), float(slope.max())


def sample_rows(n, rng, extra=512):
    """The first and last 64-point unit and a random sample of the rest."""
    rows = np.concatenate([np.arange(min(64, n)), np.arange(max(0, n - 64), n), rng.integers(0, n, min(extra, n))])
    return np.unique(rows)


@pytest.mark.parametrize("case", SWEEP_CASES, ids=lambda c: "d%d-m%d-n%d-%s-%s-%s-%s" % c)
def test_kmn_sweep_vs_oracle(eng, case):
    d, m, n, family, dt, kind, entry = case
    rng = np.random.default_rng(d * 1_000_003 + m * 1009 + n)
    X, Z, sum_beta2 = sweep_data(family, n, m, d, rng)
    k, ok, C, beta = sweep_kernel(kind, d, sum_beta2, rng)
    X = X.astype(np.float32 if dt == "fp32" else np.float64)
    eng.set_precision(N.SGP_PREC_AUTO)
    eng.begin(k, Z)
    rows = np.arange(n) if n * m <= 20_000_000 else sample_rows(n, rng)
    if entry == "host":
        K = eng.kmn_sweep(X)[rows]
    else:
        Xd = to_device(X)
        Kd = torch.empty((n, m), dtype=torch.float32, device="cuda")
        eng.kmn_sweep_device(Xd.data_ptr(), X.dtype == np.float32, n, Kd.data_ptr())
        eng.sync()
        K = Kd[torch.from_numpy(rows).cuda()].cpu().numpy()
    assert K.shape == (len(rows), m) and K.dtype == np.float32
    err, slope = sweep_check(K, X[rows], Z, ok, C, beta)
    print("sweep %s: max element error %.2e, bound slope in use %.1f of %d (rows checked %d)" % (
        "d%d-m%d-n%d-%s-%s-%s-%s" % case, err, slope, SWEEP_ULPS, len(rows)))


def test_kmn_sweep_bench_shape_on_device(eng):
    """bench.py's sweep leg (262144 x 8 fp32, m = 4000: 32 tiles x point slices) on the device entry, rows sampled."""
    n, d, m = 262_144, 8, 4000
    rng = np.random.default_rng(5)
    X = rng.random((n, d), dtype=np.float32)
    Z = X[rng.permutation(n)[:m]].astype(np.float64)
    k = 1 * sg.ARDRBFKernel(np.full(d, np.sqrt(18.0 / d))) + sg.const(1) * sg.EyeKernel()
    ok = lambda: 1 * oracle.ARDRBFKernel(np.full(d, np.sqrt(18.0 / d))) + oracle.const(1) * oracle.EyeKernel()
    eng.set_precision(N.SGP_PREC_AUTO)
    eng.begin(k, Z)
    Xd = to_device(X)
    Kd = torch.empty((n, m), dtype=torch.float32, device="cuda")
    eng.kmn_sweep_device(Xd.data_ptr(), True, n, Kd.data_ptr())
    eng.sync()
    rows = sample_rows(n, rng, extra=1024)
    K = Kd[torch.from_numpy(rows).cuda()].cpu().numpy().astype(np.float64)
    del Kd
    torch.cuda.empty_cache()
    err, slope = sweep_check(K, X[rows], Z, ok, 1.0, np.full(d, np.sqrt(18.0 / d)))
    print("sweep bench shape 262144 x 8, m=4000 (device): max element error %.2e, bound slope in use %.1f" % (err, slope))


# ---------------- d. a sweep inside a statistics window leaves the window alone ------------------------------------------
def test_sweep_does_not_touch_statistics_window(eng):
    """begin -> accumulate (AUTO -> int8) -> sweep points with large in-range norms -> sweep points outside the fp16
    range (OperandRangeError) -> sweep good points (must succeed) -> finish: finish succeeds and G, b are bit-identical
    to the same window without the sweeps.  The device sweep reports nothing and changes nothing either; the active
    set's own range status from begin is still reported by the host sweep."""
    rng = np.random.default_rng(509)
    n, d, m = 100_000, 8, 256
    X = rng.random((n, d), dtype=np.float32)
    y = np.sin(X.astype(np.float64).sum(1))
    Z = X[:m].astype(np.float64)
    beta = np.full(d, np.sqrt(18.0 / d))
    k, ok = ard_pair(beta)
    G_ref, b_ref, path = stats_host(eng, k, X, y, Z, N.SGP_PREC_AUTO)
    assert path == N.SGP_PREC_I8
    centre = Z.mean(0)
    signs = rng.choice([-1.0, 1.0], (4096, d))
    X_far = centre + signs * np.sqrt(3000.0 / (np.log2(np.e) * (beta ** 2).sum()))        # |x^|^2 = 3000 <= 4096
    X_out = rng.standard_normal((4096, d)) * 1e4
    eng.begin(k, Z)
    eng.accumulate(X, y)
    assert eng.last_path() == N.SGP_PREC_I8
    K_far = eng.kmn_sweep(X_far)
    assert np.all(np.isfinite(K_far))
    with pytest.raises(sg.OperandRangeError):
        eng.kmn_sweep(X_out)
    Xod = to_device(X_out)
    Kd = torch.empty((len(X_out), m), dtype=torch.float32, device="cuda")
    eng.kmn_sweep_device(Xod.data_ptr(), False, len(X_out), Kd.data_ptr())          # no report, no side effect
    good = X[:1000]
    K = eng.kmn_sweep(good)
    sweep_check(K, good, Z, ok, 1.0, beta)
    G, b = eng.finish()
    assert np.array_equal(G, G_ref) and np.array_equal(b, b_ref)
    Z_out = Z.copy()
    Z_out[0, 0] += 300.0                                                 # one active point out of range, the points not
    eng.begin(k, Z_out)
    with pytest.raises(sg.OperandRangeError):
        eng.kmn_sweep(good)


# ---------------- e. the kappa margin of the fixed-point encoding --------------------------------------------------------
def test_kappa_margin_of_fixed_point_encoding():
    """fixed_word needs kappa * C0 + 0x4040 < 2^23, i.e. kappa < 1 + 2.05e-3 (test_host_logic.py).  A kernel value is
    <= 1 mathematically, but T = 2 x^.z^ - |x^|^2 - |z^|^2 is accumulated in fp32 from terms as large as the scaled
    norms, so for coinciding points it is 0 only up to that rounding.  Here X contains Z (the first 64 points ARE the
    first 64 active points, so the first tile of CTA (0,0) holds coinciding pairs), scaled squared norms rise from benign
    to the operand gate, and the int8 Gram with tensor-core distances is forced.  sgp_debug_i8_tile reads T and the
    fixed-point words of the first tile; the sweep reads 2^T with the same operand images and the same contraction.
    Measured on an H100 with the gate at 16384 (fp16's own limit): max T = +1.5e-5 at |x^|^2 ~ 90, +2.0e-3 at ~8800,
    +2.9e-3 at 15500 -- past the encoding's margin.  The gate is now 4096 (kI8TensorR2Max).  Checked at every norm it
    admits: kappa < 1 + 2e-3, no fixed-point word overflowed, and the forced int8 statistics stay within an error that
    grows with the norms (4e-6 |x^|^2) instead of losing the coinciding pairs' elements; above the gate finish reports
    OperandRangeError."""
    e = sg.ProjectedProcessEngine(0)
    try:
        e.debug_i8_tile()                                          # arm the dump (I8 launches write the first tile)
        rng = np.random.default_rng(601)
        n, d, m, clusters = 4096, 16, 256, 8
        signs = rng.choice([-1.0, 1.0], (clusters, d))
        jitter = 0.3 * rng.standard_normal((n, d))
        lab = rng.integers(0, clusters, n)
        k, ok = ard_pair(np.ones(d), C=1.0, eye=1e-3)
        y = rng.standard_normal(n)
        for level in (2.0, 64.0, 512.0, 2048.0, 4000.0, 6000.0):
            L = np.sqrt(level / (np.log2(np.e) * d))
            X = L * signs[lab] + jitter
            Z = X[:m].copy()
            norms = np.log2(np.e) * ((X - Z.mean(0)) ** 2).sum(1)
            inside = level < GATE
            if inside:
                X *= min(1.0, np.sqrt(0.99 * GATE / norms.max()))           # keep every point inside the gate
                Z = X[:m].copy()
                norms = np.log2(np.e) * ((X - Z.mean(0)) ** 2).sum(1)
            e.set_precision(N.SGP_PREC_I8)
            e.begin(k, Z)
            e.accumulate(X, y)
            if not inside:
                assert norms.max() > GATE
                with pytest.raises(sg.OperandRangeError):
                    e.finish()
                continue
            T, w = e.debug_i8_tile()
            G, b = e.finish()
            K = e.kmn_sweep(X)
            G0, b0 = TiledOracle(ok, X, y, Z).stats(n)
            tmax, kmax = float(T.max()), float(K.max())
            exps = np.unique((w >> 23) & 0xFF)
            word_max = int((w & 0x7FFFFF).max()) - 0x4040                  # the largest u of the tile
            eg, eb = rel(G, G0), rel(b, b0)
            print("kappa margin: max |x^|^2 = %7.1f  max T (first tile) = %+.2e  max kappa (sweep) - 1 = %+.2e"
                  "  max u / C0 - 1 = %+.2e  forced I8 dG=%.2e db=%.2e" % (
                      norms.max(), tmax, kmax - 1.0, word_max / FIXED_C0 - 1.0, eg, eb))
            assert norms.max() <= GATE
            assert 2.0 ** tmax < 1.0 + 2e-3 and kmax < 1.0 + 2e-3 and word_max < FIXED_C0 * (1.0 + 2e-3)
            assert list(exps) == [150]                                      # u + 0x4040 < 2^23: no word overflowed
            assert tmax > -1e-4                                             # coinciding pairs are in the tile (T ~ 0)
            bound = max(TOL_I8, 4e-6 * norms.max())                         # the distance error, not O(1)
            assert eg < bound and eb < bound
    finally:
        e.close()


# ---------------- f. prediction across its chunk boundary ----------------------------------------------------------------
@pytest.fixture(scope="module")
def predict_model():
    rng = np.random.default_rng(701)
    d, m = 3, 129
    beta = np.array([2.5, 1.5, 3.0])
    mk = lambda S: 1.3 * S.ARDRBFKernel(beta) + 0.6 * S.RBFKernel(0.4) + S.const(0.05) * S.EyeKernel()
    Xtr = rng.random((3000, d))
    ytr = np.sin(3 * Xtr.sum(1)) + 0.05 * rng.standard_normal(3000)
    Z = rng.random((m, d))
    ok = lambda: mk(oracle)
    G0, b0 = TiledOracle(ok, Xtr, ytr, Z).stats(len(Xtr))
    kernel0 = ok().set_hyperparameters(ok().get_hyperparameters()).set_training_vectors(Z)
    mv0, mm0 = oracle.get_magic_vector(kernel0, G0, b0)
    return dict(k=mk(sg), Z=Z, kernel0=kernel0, mv0=mv0, mm0=mm0, d=d)


@pytest.mark.parametrize("with_variance", [True, False], ids=["var", "mean"])
@pytest.mark.parametrize("n", [32767, 32768, 32769, 70001])
def test_predict_across_chunk_boundary(eng, predict_model, n, with_variance):
    """sgp_predict runs in chunks of 32768 points.  With the oracle's magic vector and matrix installed (sgp_set_magic),
    only the chunk loop, the cross kernel and the predictive sums are under test: all fp64, 1e-11 of the sum of the
    magnitudes each output adds up (|k| |v| for the mean, selfKernel + |k| |M| |k| for the variance)."""
    c = predict_model
    Xt = np.random.default_rng(n).random((n, c["d"]))
    eng.set_precision(N.SGP_PREC_AUTO)
    eng.begin(c["k"], c["Z"])
    eng.set_magic(c["mv0"], c["mm0"])
    mean, var = eng.predict(Xt, with_variance=with_variance)
    m0, v0 = oracle.GaussianProjectedProcessRawPredictor(c["mv0"], c["mm0"], c["kernel0"]).predict_many(Xt)
    K0 = np.abs(c["kernel0"].cross_kernel(Xt))
    em = float((np.abs(mean - m0) / (K0 @ np.abs(c["mv0"]))).max())
    assert mean.shape == (n,)
    if with_variance:
        scale = c["kernel0"].self_kernel(None) + np.einsum("ti,ij,tj->t", K0, np.abs(c["mm0"]), K0)
        ev = float((np.abs(var - v0) / scale).max())
    else:
        assert var is None
        ev = 0.0
    print("predict n=%d var=%s: mean err %.1e, var err %.1e (of the summed magnitudes)" % (n, with_variance, em, ev))
    assert em < TOL_PREDICT_F64 and ev < TOL_PREDICT_F64
