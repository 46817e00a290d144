"""The fp64 DMMA statistics kernel (`kmn_gram_f64_kernel`, csrc/gram_f64.cu) element by element: every G and b entry
within its own rounding bound (oracle/gram_f64_model.py; tests/test_host_gram_f64_model.py shows the bound sharp), in
all four loops (run on an H100: `pytest -m gpu`).

The normwise gates of test_gpu_gram_variants.py and test_gpu_parity.py (max |G - G0| / max |G0|) cannot see errors in
elements far below the largest; on data spread over a few length scales most of G is such elements, and they enter
A = wn K_mm + G, whose inverse the tail computes.  Every case here asserts the path, exact symmetry, and each element of
G (every row, or sampled rows where n m^2 is large) and of b within the model's bound; it prints the largest fraction
of the bound used and the rounding count R of the accumulation.
"""
import numpy as np
import pytest
import torch

import spark_gp_b200 as sg
import oracle
from oracle.gram_f64_model import GramF64Model, fractions, reference_share
from spark_gp_b200 import _native as N
from test_gpu_gram_variants import PREC, ard_unit, kernel_pair, placement_data, resolve_n, variant_cases
from test_host_gram_f64_model import rounding_budget
from test_host_i8_gram_model import entry_launches
from test_host_logic import f64_variant, host_chunks

pytestmark = pytest.mark.gpu
STRICT = N.SGP_PREC_F64_STRICT


@pytest.fixture(scope="module")
def eng():
    e = sg.ProjectedProcessEngine(0)
    yield e
    e.close()


@pytest.fixture(scope="module")
def num_sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


def run_window(eng, k, Z, calls, prec, device=False):
    """One begin..finish window over the accumulate calls [(X, y)]: (G, b, path, launches)."""
    eng.set_precision(prec)
    eng.begin(k, Z)
    launches = []
    for X, y in calls:
        f32 = X.dtype == np.float32
        if device:
            Xt, yt = torch.from_numpy(np.ascontiguousarray(X)).cuda(), torch.from_numpy(np.ascontiguousarray(y)).cuda()
            torch.cuda.synchronize()
            eng.accumulate_ptr(Xt.data_ptr(), f32, yt.data_ptr(), len(X), True)
            eng.sync()
        else:
            eng.accumulate(X, y)
        launches += entry_launches("device" if device else "host", len(X), X.shape[1], f32)
    path = eng.last_path()
    G, b = eng.finish()
    return G, b, path, launches


def check(eng, num_sms, k, ok, Z, calls, prec, label, want_path=None, device=False):
    """Runs the window and judges every element against the model; returns (G, b, model statistics)."""
    G, b, path, launches = run_window(eng, k, Z, calls, prec, device)
    X = np.concatenate([np.asarray(c[0], dtype=np.float64) for c in calls])
    y = np.concatenate([c[1] for c in calls])
    R, R_b = rounding_budget(launches, len(Z), num_sms)
    strict = (want_path if want_path is not None else prec) == STRICT
    st = GramF64Model(ok, Z, strict=strict).statistics(X, y, R, R_b)
    fg, fb = fractions(G, b, st)
    share = reference_share(st)
    label = "%s %s" % (label, {STRICT: "strict", N.SGP_PREC_F64: "f64", N.SGP_PREC_AUTO: "auto"}[prec])
    print("%s: G %.3g b %.3g of the bound, R %d, %d launches, %d of %d rows, reference %.1e of the bound" % (
        label, fg, fb, R, len(launches), len(st["rows"]), len(Z), share))
    assert path == (want_path if want_path is not None else prec)
    assert np.array_equal(G, G.T)
    assert share < 0.125
    assert fg <= 1.0 and fb <= 1.0
    return G, b, st


# ---------------- a. every loop at every m, d and slice edge (the covering list of test_gpu_gram_variants.py) -----------
@pytest.mark.parametrize("variant,m,d,terms,n,dtype,flags", variant_cases())
def test_variant_within_bound(eng, num_sms, variant, m, d, terms, n, dtype, flags):
    n = resolve_n(n, num_sms)
    prec = PREC[variant]
    assert f64_variant(prec, terms, d) == variant
    rng = np.random.default_rng(1000 * m + 10 * d + terms)
    X = rng.standard_normal((n, d))
    if dtype == "fp32":
        X = X.astype(np.float32)
    y = np.zeros(n) if "y0" in flags else rng.standard_normal(n)
    Z = rng.standard_normal((m, d))
    share = min(n, m) // 2
    Z[:share] = X[:share]
    k, okf = kernel_pair(rng, terms, d, nested="nested" in flags, n_eye=1 + (m % 2))
    G, b, _ = check(eng, num_sms, k, okf(), Z, [(X, y)], prec, "%s m=%d d=%d terms=%d n=%d %s" % (
        variant, m, d, terms, n, dtype))
    if "y0" in flags:
        assert np.all(b == 0.0)


# ---------------- b. dynamic range: data over several length scales, and far clusters ----------------------------------
@pytest.mark.parametrize("prec", [N.SGP_PREC_F64, STRICT], ids=["f64", "strict"])
@pytest.mark.parametrize("spread", [3.0, 6.0])
def test_wide_spread_within_bound(eng, num_sms, spread, prec):
    """Standard-normal data scaled to 3 and 6 length scales (n = 3000, d = 5, m = 200): min G / max G reaches 1e-34
    and below."""
    rng = np.random.default_rng(int(spread))
    X = rng.standard_normal((3000, 5)) * spread
    Z = X[rng.permutation(3000)[:200]].copy()
    y = np.sin(X.sum(1)) + 0.1 * rng.standard_normal(3000)
    k, okf = kernel_pair(rng, 1, 5)
    G, _, st = check(eng, num_sms, k, okf(), Z, [(X, y)], prec, "spread %g" % spread)
    print("   min G / max G = %.1e" % float(np.min(st["G"]) / np.max(st["G"])))


@pytest.mark.parametrize("prec", [N.SGP_PREC_F64, STRICT], ids=["f64", "strict"])
def test_far_clusters_within_bound(eng, num_sms, prec):
    """Two clusters 14 length scales apart (q ~ 200 between them, exp(-q) ~ 1e-85 below fp32's 2^-126): the
    cross-cluster tiles of G are 0 or inside the flush floor in SGP_PREC_F64, and the tiny nonzeros of the model in
    strict mode."""
    rng = np.random.default_rng(11)
    n, m = 2048, 256
    X = rng.standard_normal((n, 4)) * 0.4
    X[n // 2:, 0] += 14.0
    y = rng.standard_normal(n)
    Z = np.vstack([X[:128], X[n // 2:n // 2 + 128]])             # row tile 0 in one cluster, row tile 1 in the other
    k, ok = ard_unit(4)
    G, _, st = check(eng, num_sms, k, ok(), Z, [(X, y)], prec, "far clusters")
    far = G[128:, :128]
    if prec == STRICT:
        assert np.all(far > 0)
    else:
        assert np.all(np.abs(far) <= np.max(np.abs(G)) * 1e-60)


# ---------------- c. placement: data far from the origin ------------------------------------------------------------------
@pytest.mark.parametrize("prec", [N.SGP_PREC_F64, STRICT], ids=["f64", "strict"])
@pytest.mark.parametrize("offset", [0.0, 10.0, 100.0, 1e3, -1e3, "single"], ids=["0", "10", "100", "1e3", "-1e3", "1e3-dim0"])
def test_placement_within_bound(eng, num_sms, offset, prec):
    X, y, Z, _ = placement_data(offset, n=3000)
    k, ok = ard_unit(5)
    check(eng, num_sms, k, ok(), Z, [(X, y)], prec, "placement %s" % offset)


# ---------------- d. term scales at fp32's range ends ---------------------------------------------------------------------
@pytest.mark.parametrize("prec", [N.SGP_PREC_F64, STRICT], ids=["f64", "strict"])
@pytest.mark.parametrize("C", [1e-30, 1e30, 1e-40, 1e39])
def test_term_scale_range_within_bound(eng, num_sms, C, prec):
    """The term scale is applied in fp64 after the exponential: C above FLT_MAX gives finite G, C below FLT_MIN keeps all
    its bits, and C k below 2^-126 does not underflow."""
    rng = np.random.default_rng(5)
    X = rng.standard_normal((2000, 4)) * 2.0
    Z = X[:100].copy()
    y = rng.standard_normal(2000)
    k = C * sg.ARDRBFKernel(np.ones(4)) + sg.const(1e-2) * sg.EyeKernel()
    ok = C * oracle.ARDRBFKernel(np.ones(4)) + oracle.const(1e-2) * oracle.EyeKernel()
    G, b, _ = check(eng, num_sms, k, ok, Z, [(X, y)], prec, "C = %g" % C)
    assert np.all(np.isfinite(G)) and np.all(np.isfinite(b))


# ---------------- e. accumulation across launches and calls -----------------------------------------------------------
def launch_data(n, d, seed):
    rng = np.random.default_rng(seed)
    X = rng.standard_normal((n, d)).astype(np.float32)
    return X, rng.standard_normal(n), X[rng.permutation(n)[:20]].astype(np.float64)


def test_host_entry_several_chunks(eng, num_sms):
    """100000 points of d = 64 in fp32: two chunks of the host entry, then the same points through the device entry."""
    X, y, Z = launch_data(100_000, 64, 21)
    assert len(host_chunks(100_000, 64, True)) == 2
    k, okf = kernel_pair(np.random.default_rng(21), 1, 64)
    check(eng, num_sms, k, okf(), Z, [(X, y)], N.SGP_PREC_F64, "host entry, 2 chunks")
    check(eng, num_sms, k, okf(), Z, [(X, y)], N.SGP_PREC_F64, "device entry", device=True)


def test_several_calls_one_window(eng, num_sms):
    X, y, Z = launch_data(9000, 6, 22)
    k, okf = kernel_pair(np.random.default_rng(22), 2, 6)
    calls = [(X[:5000], y[:5000]), (X[5000:5017], y[5000:5017]), (X[5017:], y[5017:])]
    for prec in (N.SGP_PREC_F64, STRICT):
        check(eng, num_sms, k, okf(), Z, calls, prec, "three calls")


def test_auto_below_int8_threshold_runs_f64(eng, num_sms):
    """32767 points: AUTO keeps the call on the fp64 kernel."""
    X, y, Z = launch_data(32767, 4, 23)
    k, ok = ard_unit(4)
    check(eng, num_sms, k, ok(), Z, [(X, y)], N.SGP_PREC_AUTO, "AUTO at 32767", want_path=N.SGP_PREC_F64)


# ---------------- f. b over labels of every size and sign ---------------------------------------------------------------
@pytest.mark.parametrize("prec", [N.SGP_PREC_F64, STRICT], ids=["f64", "strict"])
def test_b_mixed_labels_within_bound(eng, num_sms, prec):
    rng = np.random.default_rng(31)
    n = 4000
    X = rng.standard_normal((n, 3))
    y = 10.0 ** rng.uniform(-3, 3, n) * rng.choice([-1.0, 1.0], n)
    y[rng.permutation(n)[:400]] = 0.0
    Z = X[rng.permutation(n)[:150]].copy()
    k, okf = kernel_pair(rng, 3, 3)
    check(eng, num_sms, k, okf(), Z, [(X, y)], prec, "labels 1e-3 .. 1e3")
