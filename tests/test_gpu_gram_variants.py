"""The fp64 DMMA statistics kernel (`kmn_gram_f64_kernel`, csrc/gram_f64.cu) in every loop variant, and the int8
direct-distance mode across its width limit, against the fp64 oracle (run on an H100: `pytest -m gpu`).

The fp64 kernel serves every accumulate call under 32768 points, every shard over AUTO's magnitude budget, every kernel
the int8 modes refuse, and both SGP_PREC_F64 modes.  It runs one of four loops, picked at run time (mirror:
`f64_variant` in test_host_logic.py): fp32 elements on a 128 x 64 staircase of tiles -- pipelined for one non-Eye term
with dpad <= 32, generic otherwise -- or fp64 elements on the 128 x 128 triangle (SGP_PREC_F64_STRICT) with the active
set resident for one term with dpad <= 32, chunked otherwise.  The covering list gives each variant every edge of m
(64-column staircase tiles partly or wholly past m, 128-row tiles, more tiles than SMs) and of d (dpad rounding, the
32-dim staging chunks, the 72-wide int8 limit), 1..4 non-Eye terms and both element types of X; the point counts
include the slice edges 16 num_sms +- 1 and 16 (num_sms + 1), where the last slices get no points (mirror: `f64_slices`).

Placement: the kernel values depend on the distances only, so data far from the origin must give the same statistics
as data near it.  The kernel centres both operands in fp64 before the fp32 rounding (on the active-set mean rounded to a
whole multiple of its standard deviation); the placement cases move the data up to 1e3 length scales away and check G,
b and the posterior (test_host_logic.py emulates why uncentred fp32 staging fails there).

Tolerances as in test_gpu_parity.py: G, b relative to their largest element 1e-11 (strict) / 1e-6 (F64, I8_DIRECT);
posterior mean / variance 1e-5.
"""
import numpy as np
import pytest
import torch

import oracle
import spark_gp_b200 as sg
from spark_gp_b200 import _native as N
from test_gpu_parity import _oracle_stats_chunked, rel
from test_host_logic import direct_ok, dpad4, f64_slices, f64_variant

pytestmark = pytest.mark.gpu

TOL_STRICT, TOL_STATS, TOL_PRED = 1e-11, 1e-6, 1e-5
PREC = {"pipelined": N.SGP_PREC_F64, "generic": N.SGP_PREC_F64, "resident": N.SGP_PREC_F64_STRICT,
        "chunked": N.SGP_PREC_F64_STRICT}


@pytest.fixture(scope="module")
def eng():
    e = sg.ProjectedProcessEngine(0)
    yield e
    e.close()


@pytest.fixture(scope="module")
def num_sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


def oracle_stats(ok, X, y, Z):
    """The oracle's G, b over contiguous experts of 512 points (an RBF term builds its experts' own n_e x n_e distance
    matrix when its training vectors are set, which costs more than the cross kernel at 2048-point experts)."""
    return _oracle_stats_chunked(ok, X, y, Z, chunk=512)


def run_stats(eng, kernel, X, y, Z, precision):
    eng.set_precision(precision)
    eng.begin(kernel, Z)
    eng.accumulate(X, y)
    path = eng.last_path()
    G, b = eng.finish()
    return G, b, path


def kernel_pair(rng, n_terms, d, scales=(20.0, 0.05, 1.3, 0.4), width=1.0, nested=False, n_eye=1):
    """(library kernel, oracle factory): n_terms non-Eye terms alternating ARD (non-uniform beta) and RBF with the given
    term scales, plus n_eye Eye terms; nested: the non-Eye sum under a bounded Scalar.  Inverse length scales are about
    width / sqrt(d), so that the scaled squared distances of standard-normal data (width 1) are O(1) at any d."""
    specs = []
    for t in range(n_terms):
        if t % 2 == 0:
            specs.append(("ard", scales[t], rng.uniform(0.3, 1.5, d) * width / np.sqrt(d)))
        else:
            specs.append(("rbf", scales[t], np.sqrt(d) * rng.uniform(0.7, 1.4) / width))

    def make(S):
        body = None
        for kind, C, p in specs:
            term = C * (S.ARDRBFKernel(p) if kind == "ard" else S.RBFKernel(p))
            body = term if body is None else body + term
        if nested:
            body = S.Scalar(2.0).between(0).and_(30) * body
        for e in range(n_eye):
            body = body + S.const([1e-2, 0.3][e]) * S.EyeKernel()
        return body
    return make(sg), (lambda: make(oracle))


# ---------------- a. every loop variant across the m, d, n edges ----------------------------------------------------------
M_EDGES = [1, 63, 64, 65, 127, 128, 129, 191, 192, 193, 255, 257, 1000, 2100]
D_EDGES = [1, 3, 4, 5, 31, 32, 33, 36, 63, 64, 65, 72, 73, 100, 130]
# point counts by case index: the slice edges go with m <= 128 (one tile, one slice per SM)
N_SEQ = ["16S-1", "16S+1", "16(S+1)", 1, "16(S+1)", 15, 16, 17, 33, 4000, 2500, 1234, 333, 50, 3001]


def variant_cases():
    cases = []
    for variant in ("pipelined", "generic", "resident", "chunked"):
        single = variant in ("pipelined", "resident")
        ds = [d for d in D_EDGES if dpad4(d) <= 32] if single else D_EDGES
        for i in range(max(len(M_EDGES), len(ds))):
            m, d = M_EDGES[i % len(M_EDGES)], ds[i % len(ds)]
            terms = 1 if single else [2, 3, 4, 1][i % 4]
            if f64_variant(PREC[variant], terms, d) != variant:
                terms = 2                                # one term with dpad <= 32 would take the other loop
            n = N_SEQ[i % len(N_SEQ)]
            dtype = "fp32" if i % 2 == 0 else "fp64"
            flags = ("nested" if (variant == "generic" and i == 1) else "") + ("y0" if (variant == "chunked" and i == 6) else "")
            cases.append(pytest.param(variant, m, d, terms, n, dtype, flags,
                                      id="%s-m%d-d%d-t%d-n%s-%s%s" % (variant, m, d, terms, n, dtype, "-" + flags if flags else "")))
    return cases


def resolve_n(n, num_sms):
    return {"16S-1": 16 * num_sms - 1, "16S+1": 16 * num_sms + 1, "16(S+1)": 16 * (num_sms + 1)}.get(n, n)


@pytest.mark.parametrize("variant,m,d,terms,n,dtype,flags", variant_cases())
def test_variant_vs_oracle(eng, num_sms, variant, m, d, terms, n, dtype, flags):
    n = resolve_n(n, num_sms)
    prec = PREC[variant]
    assert f64_variant(prec, terms, d) == variant
    slices = f64_slices(m, n, num_sms)
    if m <= 128 and n == 16 * (num_sms + 1):
        assert slices[-1] == 0                          # trailing slices without points
    rng = np.random.default_rng(1000 * m + 10 * d + terms)
    X = rng.standard_normal((n, d))
    if dtype == "fp32":
        X = X.astype(np.float32)
    y = np.zeros(n) if "y0" in flags else rng.standard_normal(n)
    Z = rng.standard_normal((m, d))
    share = min(n, m) // 2                              # coinciding points: kernel values of exactly 1
    Z[:share] = X[:share]
    k, ok = kernel_pair(rng, terms, d, nested="nested" in flags, n_eye=1 + (m % 2))
    G0, b0 = oracle_stats(ok, X, y, Z)
    G, b, path = run_stats(eng, k, X, y, Z, prec)
    tol = TOL_STRICT if variant in ("resident", "chunked") else TOL_STATS
    eg = rel(G, G0)
    eb = float(np.abs(b).max()) if "y0" in flags else rel(b, b0)
    print("%s m=%d d=%d terms=%d n=%d %s (%d slices, %d empty): dG=%.2e db=%.2e" % (
        variant, m, d, terms, n, dtype, len(slices), slices.count(0), eg, eb))
    assert path == prec
    assert np.array_equal(G, G.T)
    assert eg < tol
    if "y0" in flags:
        assert np.all(b == 0.0)
    else:
        assert eb < tol


# ---------------- b. placement: data far from the origin ------------------------------------------------------------------
def placement_data(offset, d=5, n=6000, m=200, seed=0):
    """n points spread over 3 length scales (unit length scale), moved by `offset` in every dimension ('single': 1e3
    in dimension 0 only); the active set is m of the points; 300 held-out points in the same region."""
    rng = np.random.default_rng(seed)
    shift = np.zeros(d)
    if offset == "single":
        shift[0] = 1e3
    else:
        shift[:] = offset
    spread = 3.0 * np.sqrt(5.0 / d)
    X = rng.random((n, d)) * spread + shift
    y = np.sin((X - shift).sum(1)) + 0.1 * rng.standard_normal(n)
    Z = X[rng.permutation(n)[:m]].copy()
    Xt = rng.random((300, d)) * spread + shift
    return X, y, Z, Xt


def oracle_posterior(ok, X, y, Z, Xt):
    G0, b0 = oracle_stats(ok, X, y, Z)
    theta = ok().get_hyperparameters()
    kernel0 = ok().set_hyperparameters(theta).set_training_vectors(Z)
    mv0, mm0 = oracle.get_magic_vector(kernel0, G0, b0)
    m0, v0 = oracle.GaussianProjectedProcessRawPredictor(mv0, mm0, kernel0).predict_many(Xt)
    return G0, b0, m0, v0


def check_placement(eng, k, ok, X, y, Z, Xt, prec, label):
    G0, b0, m0, v0 = oracle_posterior(ok, X, y, Z, Xt)
    G, b, path = run_stats(eng, k, X, y, Z, prec)
    eng.magic()
    mean, var = eng.predict(Xt)
    eg, eb, em, ev = rel(G, G0), rel(b, b0), rel(mean, m0), float(np.abs(var / v0 - 1).max())
    print("placement %s: dG=%.2e db=%.2e dmean=%.2e dvar=%.2e" % (label, eg, eb, em, ev))
    strict = prec == N.SGP_PREC_F64_STRICT
    assert path == (N.SGP_PREC_F64_STRICT if strict else N.SGP_PREC_F64)
    assert np.array_equal(G, G.T)
    tol = TOL_STRICT if strict else TOL_STATS
    assert eg < tol and eb < tol
    assert em < TOL_PRED and ev < TOL_PRED


def ard_unit(d, sigma2=1e-2):
    beta = np.ones(d)
    k = 1 * sg.ARDRBFKernel(beta) + sg.const(sigma2) * sg.EyeKernel()
    ok = lambda: 1 * oracle.ARDRBFKernel(beta) + oracle.const(sigma2) * oracle.EyeKernel()
    return k, ok


@pytest.mark.parametrize("mode", ["auto", "f64"])
@pytest.mark.parametrize("offset", [0.0, 10.0, 100.0, 1e3, -1e3, "single"], ids=["0", "10", "100", "1e3", "-1e3", "1e3-dim0"])
def test_placement_vs_oracle(eng, offset, mode):
    """n = 6000, d = 5, m = 200, sigma2 = 1e-2: AUTO keeps the call on the fp64 kernel (pipelined loop)."""
    X, y, Z, Xt = placement_data(offset)
    k, ok = ard_unit(5)
    prec = N.SGP_PREC_AUTO if mode == "auto" else N.SGP_PREC_F64
    check_placement(eng, k, ok, X, y, Z, Xt, prec, "%s offset=%s" % (mode, offset))


def test_placement_strict_control(eng):
    X, y, Z, Xt = placement_data(1e3)
    k, ok = ard_unit(5)
    check_placement(eng, k, ok, X, y, Z, Xt, N.SGP_PREC_F64_STRICT, "strict offset=1e3")


@pytest.mark.parametrize("mode", ["auto", "f64"])
def test_placement_two_terms_d80(eng, mode):
    """Two terms at d = 80 (generic loop; no int8 mode takes this kernel at any size), data 1e3 length scales out."""
    assert not direct_ok(2, 80)
    X, y, Z, Xt = placement_data(1e3, d=80, seed=1)
    beta2 = np.full(80, 0.5)
    k = 0.8 * sg.ARDRBFKernel(np.ones(80)) + 0.6 * sg.ARDRBFKernel(beta2) + sg.const(1e-2) * sg.EyeKernel()
    ok = lambda: 0.8 * oracle.ARDRBFKernel(np.ones(80)) + 0.6 * oracle.ARDRBFKernel(beta2) + oracle.const(1e-2) * oracle.EyeKernel()
    prec = N.SGP_PREC_AUTO if mode == "auto" else N.SGP_PREC_F64
    check_placement(eng, k, ok, X, y, Z, Xt, prec, "%s two terms d=80 offset=1e3" % mode)


# ---------------- c. the int8 direct-distance mode across its width limit n_terms * dpad <= 72 ----------------------------
DIRECT_SCALES = (20.0, 0.2, 20.0, 0.2)          # term scales 100x apart


def direct_data(terms, d, n, m, seed):
    rng = np.random.default_rng(seed)
    X = rng.random((n, d), dtype=np.float32)
    y = np.sin(X.astype(np.float64).sum(1)) + 0.1 * rng.standard_normal(n)
    Z = X[rng.permutation(n)[:m]].astype(np.float64)
    k, ok = kernel_pair(rng, terms, d, scales=DIRECT_SCALES, width=3.0, n_eye=1 + terms % 2)
    return X, y, Z, k, ok


@pytest.mark.parametrize("terms,d", [(1, 72), (1, 69), (2, 36), (2, 33), (3, 24), (3, 21), (4, 16), (4, 13)])
def test_direct_mode_accepted_widths(eng, terms, d):
    """16461 points at m = 1000 and m = 129 (the first 129 active points: the oracle's statistics are the leading
    block of the m = 1000 ones)."""
    assert direct_ok(terms, d)
    X, y, Z, k, ok = direct_data(terms, d, 16461, 1000, seed=100 * terms + d)
    G0, b0 = oracle_stats(ok, X, y, Z)
    for m in (1000, 129):
        G, b, path = run_stats(eng, k, X, y, Z[:m], N.SGP_PREC_I8_DIRECT)
        eg, eb = rel(G, G0[:m, :m]), rel(b, b0[:m])
        print("direct terms=%d d=%d m=%d: dG=%.2e db=%.2e" % (terms, d, m, eg, eb))
        assert path == N.SGP_PREC_I8_DIRECT
        assert np.array_equal(G, G.T)
        assert eg < TOL_STATS and eb < TOL_STATS


@pytest.mark.parametrize("terms,d", [(1, 73), (2, 37), (3, 25), (4, 17)])
def test_direct_mode_refused_widths(eng, terms, d):
    """One step past the limit both int8 modes refuse the kernel; AUTO runs a 40000-point call (above its int8 size
    threshold) on the fp64 kernel instead."""
    assert not direct_ok(terms, d)
    X, y, Z, k, ok = direct_data(terms, d, 40000, 129, seed=100 * terms + d)
    for prec in (N.SGP_PREC_I8_DIRECT, N.SGP_PREC_I8):
        with pytest.raises(ValueError):
            run_stats(eng, k, X[:1000], y[:1000], Z, prec)
    G0, b0 = oracle_stats(ok, X, y, Z)
    G, b, path = run_stats(eng, k, X, y, Z, N.SGP_PREC_AUTO)
    eg, eb = rel(G, G0), rel(b, b0)
    print("refused terms=%d d=%d, AUTO 40000 points: dG=%.2e db=%.2e" % (terms, d, eg, eb))
    assert path == N.SGP_PREC_F64
    assert np.array_equal(G, G.T)
    assert eg < TOL_STATS and eb < TOL_STATS
