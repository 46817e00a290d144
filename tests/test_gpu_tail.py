"""The m x m tail (`sgp_magic`) against the fp64 oracle (run on an H100: `pytest -m gpu`).

G and b are built on the host in fp64 from the oracle's cross kernel, so the statistics' rounding is out of the picture:
what separates the device pair (v, M) from the oracle's is the tail's own error -- K_mm (`kmm_build_kernel`),
A = wn K_mm + G, the Cholesky (or dsyevd + LU) solves and M = wn inv(A) - inv(K_mm).  `oracle.tail_errors` measures it in
units of u = 2^-53, with A0 = wn K0 + G and K0 built by the oracle in fp64:

  omega  componentwise backward error of v:  max_i |A0 v - b|_i / (|A0| |v| + |b|)_i / u          <= TOL_OMEGA = 16
  fwd_v  |v - v0|_inf / |v0|_inf / (kappa_inf(A0) u), v0 the oracle's LU solution                  <= TOL_FWD = 16
  fwd_M  max |M - M0| / (u (wn kappa_inf(A0) max|inv A0| + kappa_inf(K0) max|inv K0|)),
         M0 = wn inv(A0) - inv(K0)                                                                 <= TOL_FWD = 16

A backward-stable tail keeps all three at a few units whatever the conditioning: numpy's Cholesky tail gives omega of
1 to 6 u on these shapes, the H100 1 to 7 u (DESIGN.md 4.3).  tests/test_host_tail.py checks that plausible bugs fail
these gates: K_mm rounded to fp32 (omega 1.7e3 u and more, except where a tiny sigma2 keeps wn K_mm out of A), a kernel
term or the Eye sum missing from K_mm, the wrong wn, active-set rows read with the wrong stride, M without wn or with
the wrong sign.

The sweep covers each edge rather than every product: m at the warp and 128-row tile edges up to the configs3 size
m = 2000; d at the padding edges up to 784; the bench kernel (one ARD term, `const(1)*Eye + sigma2*Eye`), RBF, ARD + RBF,
four non-Eye terms, nested trainable scalars, `WhiteNoiseKernel` and an Eye-only kernel; unit-cube, standardised and
far-from-origin (1e3) active sets; n >> m (G dominates A), n < m (G rank-deficient, A held up by wn K_mm) and a tiny
sigma2 (A badly conditioned).  Then the production shapes with device-resident statistics, closed forms, the paths at
scale, and the state rules of `include/sgp.h`: a failed sgp_magic leaves no pair installed, and a window whose finish
returned SGP_E_RANGE keeps that status.

The bit-identity checks rely on cuSOLVER's potrf / potrs / getrf / syevd being deterministic on one card for one
problem size, which held on the H100 (DESIGN.md 4.3).
"""
import numpy as np
import pytest
import torch

import bench
import oracle
import spark_gp_b200 as sg
from spark_gp_b200 import _native as N

pytestmark = pytest.mark.gpu

U = np.finfo(np.float64).eps / 2
TOL_OMEGA = 16.0
TOL_FWD = 16.0


# ---------------- cases (shared with tests/test_host_tail.py) --------------------------------------------------------------
def make_kernel(S, name, d, sigma2=None):
    """One kernel of the sweep, built from module S (spark_gp_b200 or oracle) so that both sides get the same one."""
    rng = np.random.default_rng(d)
    beta = (0.6 + 0.8 * rng.random(d)) * np.sqrt(3.0 / d)          # ARD: q ~ 1 between unit-cube points
    beta2 = 0.5 * beta[::-1].copy()
    sigma = 0.6 * np.sqrt(d)
    s2 = {"bench": 1e-4}.get(name, 1e-3) if sigma2 is None else sigma2
    if name == "bench":
        return 1 * S.ARDRBFKernel(np.full(d, np.sqrt(18.0 / d))) + S.const(1) * S.EyeKernel() + S.const(s2) * S.EyeKernel()
    if name == "rbf":
        return 1.5 * S.RBFKernel(sigma) + S.const(s2) * S.EyeKernel()
    if name == "ard_rbf":
        return 1.3 * S.ARDRBFKernel(beta) + 0.05 * S.RBFKernel(sigma) + S.const(s2) * S.EyeKernel()
    if name == "four":
        return (1.3 * S.ARDRBFKernel(beta) + 0.05 * S.RBFKernel(sigma) + 20.0 * S.ARDRBFKernel(beta2)
                + 2.0 * S.RBFKernel(2.0 * sigma) + S.const(s2) * S.EyeKernel() + S.const(0.5) * S.EyeKernel())
    if name == "nested":
        inner = 1.5 * S.ARDRBFKernel(beta) + 0.3 * S.RBFKernel(sigma)
        return 2.0 * (0.5 * inner + 0.7 * (3.0 * S.ARDRBFKernel(beta2))) + S.const(s2) * S.EyeKernel()
    if name == "white_noise":
        return 1.0 * S.ARDRBFKernel(beta) + S.WhiteNoiseKernel(0.3, 0.0, 1.0)
    if name == "eye_only":
        return S.const(0.7) * S.EyeKernel() + S.const(s2) * S.EyeKernel()
    raise ValueError(name)


def make_points(layout, n, d, rng):
    if layout == "unit":
        return rng.random((n, d))
    if layout == "std":
        return rng.standard_normal((n, d))
    if layout == "far":
        return rng.random((n, d)) + 1e3
    raise ValueError(layout)


def tail_case(m, d, kernel, layout="unit", regime="tall", seed=0):
    """Z (m x d) and fp64 statistics G = K_mn K_nm, b = K_mn y of n points from the oracle's cross kernel.
    regime: "tall" n >> m (G dominates A); "wide" n = m / 2 (G rank-deficient); "tiny" n = m / 2 and sigma2 = 1e-7, the
    points spread over 4x the distance, so that A = 1e-7 K_mm + G is badly conditioned (kappa ~ 1e11) yet K_mm is not."""
    rng = np.random.default_rng(seed * 1000 + m + 7 * d)
    sigma2 = 1e-7 if regime == "tiny" else None
    n = 3 * m + 64 if regime == "tall" else m // 2 + 1
    spread = 4.0 if regime == "tiny" else 1.0
    Z = make_points(layout, m, d, rng) * spread
    X = make_points(layout, n, d, rng) * spread
    y = np.sin(X.sum(1)) + 0.1 * rng.standard_normal(n)
    k0 = make_kernel(oracle, kernel, d, sigma2).set_training_vectors(Z)
    Kmn = k0.cross_kernel(X).T
    return dict(m=m, d=d, Z=Z, G=Kmn @ Kmn.T, b=Kmn @ y, k0=k0, kernel=kernel, sigma2=sigma2,
                name="m=%d d=%d %s %s %s" % (m, d, kernel, layout, regime))


# (m, d, kernel, layout, regime)
CASES = ([(m, 16, "bench", "unit", "tall") for m in (1, 2, 3, 4, 31, 32, 33, 127, 128, 129, 255, 257, 1000, 2000)] + [
    (129, 1, "rbf", "unit", "tall"),
    (129, 3, "ard_rbf", "std", "tall"),
    (257, 5, "four", "unit", "tall"),
    (200, 17, "nested", "unit", "tall"),
    (129, 32, "ard_rbf", "far", "tall"),
    (255, 33, "white_noise", "std", "tall"),
    (129, 100, "four", "std", "wide"),
    (257, 784, "ard_rbf", "unit", "tall"),
    (33, 16, "eye_only", "unit", "tall"),
    (1000, 16, "bench", "far", "tall"),
    (1000, 16, "bench", "unit", "wide"),
    (257, 16, "bench", "std", "wide"),
    (200, 5, "ard_rbf", "unit", "tiny"),
    (1000, 16, "ard_rbf", "unit", "tiny"),
    (2000, 32, "bench", "unit", "wide"),
])


def case_id(c):
    return "m%d-d%d-%s-%s-%s" % c


def gate(e):
    return e["omega"] <= TOL_OMEGA and e["fwd_v"] <= TOL_FWD and e["fwd_M"] <= TOL_FWD


def report(name, e):
    return ("%s: omega %.2f u, fwd_v %.2f, fwd_M %.2f (kappa_A %.1e, kappa_K %.1e)"
            % (name, e["omega"], e["fwd_v"], e["fwd_M"], e["kappa_A"], e["kappa_K"]))


# ---------------- helpers ------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def eng():
    e = sg.ProjectedProcessEngine(0)
    yield e
    e.close()


def begin(e, c, precision=N.SGP_PREC_AUTO):
    e.set_precision(precision)
    e.begin(make_kernel(sg, c["kernel"], c["d"], c["sigma2"]), c["Z"])


def predict_all(e, X):
    """(host mean, host var, device mean, device var)."""
    hm, hv = e.predict(X)
    dm, dv = e.predict_tensor(torch.from_numpy(X).cuda())
    return hm, hv, dm.cpu().numpy(), dv.cpu().numpy()


def same_bits(a, b):
    return len(a) == len(b) and all(np.array_equal(x, y) for x, y in zip(a, b))


def indefinite(m):
    """wn K_mm - 3 I: K_mm's smallest eigenvalues are close to its Eye sum (~1), its largest are large."""
    return -3.0 * np.eye(m), np.ones(m)


# ---------------- a. the tail in isolation -------------------------------------------------------------------------------
@pytest.mark.parametrize("spec", CASES, ids=[case_id(s) for s in CASES])
def test_tail_on_oracle(eng, spec):
    c = tail_case(*spec)
    begin(eng, c)
    v, M = eng.magic(c["G"], c["b"])
    assert eng.last_tail_path() == 1
    e = oracle.tail_errors(c["k0"], c["G"], c["b"], v, M)
    print(report(c["name"], e))
    assert gate(e), report(c["name"], e)


def test_device_pair_feeds_prediction(eng):
    """magic(copy_out=False) then predict gives the bits of magic() then predict."""
    c = tail_case(257, 5, "ard_rbf")
    X = np.random.default_rng(3).random((777, 5))
    begin(eng, c)
    eng.magic(c["G"], c["b"])
    p1 = predict_all(eng, X)
    begin(eng, c)
    eng.magic(c["G"], c["b"], copy_out=False)
    p2 = predict_all(eng, X)
    assert same_bits(p1, p2)


# ---------------- b. production shapes, device-resident statistics -------------------------------------------------------
@pytest.mark.parametrize("name", ["configs1", "configs3"])
def test_production_shapes(eng, name):
    w = bench.WORKLOADS[name]
    d = w["d"]
    X, y = bench.make_shard(name, 0)
    Z = bench.active_set(name)
    eng.set_precision(N.SGP_PREC_AUTO)
    eng.begin(make_kernel(sg, "bench", d, bench.SIGMA2), Z)
    Xd, yd = torch.from_numpy(X).cuda(), torch.from_numpy(y).cuda()
    eng.accumulate_ptr(Xd.data_ptr(), True, yd.data_ptr(), len(X), device=True)
    path = eng.last_path()
    G, b = eng.finish()
    del Xd, yd
    v, M = eng.magic()                                  # on the device-resident G, b
    assert eng.last_tail_path() == 1
    v2, M2 = eng.magic(G, b)                            # on the copied-out G, b
    assert np.array_equal(v, v2) and np.array_equal(M, M2)
    k0 = make_kernel(oracle, "bench", d, bench.SIGMA2).set_training_vectors(Z)
    e = oracle.tail_errors(k0, G, b, v, M)
    print(report("%s (statistics path %d)" % (name, path), e))
    if name == "configs1":
        assert path == N.SGP_PREC_I8
    assert gate(e), report(name, e)


@pytest.mark.parametrize("mode", ["F64", "F64_STRICT", "I8", "I8_DIRECT", "AUTO"])
def test_device_statistics_every_mode(eng, mode):
    prec = getattr(N, "SGP_PREC_" + mode)
    rng = np.random.default_rng(17)
    n, d, m = 120_000, 16, 300
    X = rng.random((n, d), dtype=np.float32)
    y = np.sin(X.astype(np.float64).sum(1))
    Z = X[:m].astype(np.float64)
    eng.set_precision(prec)
    eng.begin(make_kernel(sg, "bench", d), Z)
    eng.accumulate(X, y)
    if mode != "AUTO":
        assert eng.last_path() == prec
    G, b = eng.finish()
    v, M = eng.magic()
    v2, M2 = eng.magic(G, b)
    assert np.array_equal(v, v2) and np.array_equal(M, M2)
    eng.set_precision(N.SGP_PREC_AUTO)


# ---------------- c. closed forms ----------------------------------------------------------------------------------------
# Reference values in extended precision (np.longdouble) from the fp64 kernel scales and Eye sum the library is given, so
# that only the device's own roundings count: within TOL_CLOSED u of the value, relative to the summed magnitudes.
TOL_CLOSED = 8.0


def scales_and_wn(kernel):
    terms = kernel.flatten()
    wn = sum(t["scale"] for t in terms if t["type"] == N.SGP_TERM_EYE)           # fp64, as the library sums it
    C = sum(np.longdouble(t["scale"]) for t in terms if t["type"] != N.SGP_TERM_EYE)
    return np.longdouble(C), np.longdouble(wn)


def within(x, x0, scale):
    return np.all(np.abs(np.asarray(x, dtype=np.longdouble) - x0) <= TOL_CLOSED * U * scale)


@pytest.mark.parametrize("kernel,g", [("bench", 0.0), ("bench", 3.7), ("four", 250.0), ("rbf", 1e-6)])
def test_closed_form_m1(eng, kernel, g):
    """m = 1: K_mm = C + wn, A = wn (C + wn) + g, v = b / A, M = wn / A - 1 / (C + wn)."""
    d = 5
    Z = np.random.default_rng(1).random((1, d))
    k = make_kernel(sg, kernel, d)
    C, wn = scales_and_wn(k)
    A = wn * (C + wn) + np.longdouble(g)
    b = 0.37
    eng.begin(k, Z)
    v, M = eng.magic(np.array([[g]]), np.array([b]))
    assert within(v[0], np.longdouble(b) / A, abs(np.longdouble(b) / A))
    assert within(M[0, 0], wn / A - 1 / (C + wn), wn / A + 1 / (C + wn))


@pytest.mark.parametrize("m", [3, 129, 1000])
def test_closed_form_eye_only(eng, m):
    """Eye-only kernel: K_mm = wn I; with G = diag(g), A = diag(wn^2 + g), v = b / A, M = diag(wn / A - 1 / wn)."""
    rng = np.random.default_rng(m)
    Z = rng.random((m, 4))
    g = rng.random(m) * 10.0 ** rng.uniform(-3, 3, m)
    b = rng.standard_normal(m)
    k = make_kernel(sg, "eye_only", 4)
    _, wn = scales_and_wn(k)
    eng.begin(k, Z)
    v, M = eng.magic(np.diag(g), b)
    A = wn * wn + g.astype(np.longdouble)
    bl = b.astype(np.longdouble)
    assert within(v, bl / A, np.abs(bl / A))
    assert within(np.diag(M), wn / A - 1 / wn, wn / A + 1 / wn)
    assert np.all(M[~np.eye(m, dtype=bool)] == 0.0)


# ---------------- d. paths at scale --------------------------------------------------------------------------------------
@pytest.mark.parametrize("m", [1000, 2000])
def test_paths_at_scale(eng, m):
    c = tail_case(m, 16, "bench", "unit", "wide")
    begin(eng, c)
    v1, M1 = eng.magic(c["G"], c["b"])
    assert eng.last_tail_path() == 1
    v2, M2 = eng.magic(c["G"], c["b"])
    assert np.array_equal(v1, v2) and np.array_equal(M1, M2)
    with pytest.raises(sg.NotPositiveDefiniteException):
        eng.magic(*indefinite(m))
    assert eng.last_tail_path() == 0


# ---------------- e. state ------------------------------------------------------------------------------------------------
def assert_no_pair(e, X):
    with pytest.raises(sg.TrainingVectorsNotInitializedException):
        e.predict(X)
    with pytest.raises(sg.TrainingVectorsNotInitializedException):
        e.predict_tensor(torch.from_numpy(X).cuda())


def test_failed_magic_leaves_no_pair():
    """magic -> predict -> a magic that fails -> no prediction -> magic again -> the first predictions, bit for bit; the
    same after SGP_E_SINGULAR, and after set_magic followed by a failed magic."""
    e = sg.ProjectedProcessEngine(0)
    try:
        c = tail_case(257, 5, "ard_rbf")
        X = np.random.default_rng(5).random((500, 5))
        begin(e, c)
        e.magic(c["G"], c["b"])
        p1 = predict_all(e, X)
        with pytest.raises(sg.NotPositiveDefiniteException):
            e.magic(*indefinite(257))
        assert_no_pair(e, X)
        e.magic(c["G"], c["b"])
        assert same_bits(predict_all(e, X), p1)

        rng = np.random.default_rng(6)
        e.set_magic(rng.standard_normal(257), rng.standard_normal((257, 257)))
        e.predict(X)
        with pytest.raises(sg.NotPositiveDefiniteException):
            e.magic(*indefinite(257))
        assert_no_pair(e, X)

        # a kernel without Eye terms has wn = 0, so A = G: G = 0 passes the eigenvalue check (all zero, none < 0) and
        # LU meets a zero pivot -- the reference's MatrixSingularException
        Z = np.random.default_rng(7).random((40, 3)) * 4.0
        Xs = np.random.default_rng(8).random((400, 3)) * 4.0
        k0 = (1.0 * oracle.ARDRBFKernel(np.full(3, 1.5))).set_training_vectors(Z)
        Kmn = k0.cross_kernel(Xs).T
        G, b = Kmn @ Kmn.T, Kmn @ np.sin(Xs.sum(1))
        e.begin(1.0 * sg.ARDRBFKernel(np.full(3, 1.5)), Z)
        e.magic(G, b)
        X3 = np.random.default_rng(9).random((300, 3)) * 4.0
        q1 = predict_all(e, X3)
        with pytest.raises(sg.MatrixSingularException):
            e.magic(np.zeros((40, 40)), np.zeros(40))
        assert e.last_tail_path() == 0
        assert_no_pair(e, X3)
        e.magic(G, b)
        assert same_bits(predict_all(e, X3), q1)
    finally:
        e.close()


def test_workspace_reuse_across_sizes():
    """One context runs the tail at m = 2000, 3, 1000 (indefinite: slow path), 1000, 257; each result is bit-identical
    to a fresh context's on the same inputs (the grow-only tail workspaces are reused, never trusted for their contents)."""
    steps = [(tail_case(2000, 16, "bench", "unit", "wide"), False), (tail_case(3, 16, "bench"), False),
             (tail_case(1000, 16, "bench", "unit", "wide"), True), (tail_case(1000, 16, "bench", "unit", "wide"), False),
             (tail_case(257, 5, "four"), False)]

    def run(e, c, bad):
        begin(e, c)
        if bad:
            with pytest.raises(sg.NotPositiveDefiniteException):
                e.magic(*indefinite(c["m"]))
            return (e.last_tail_path(),)
        v, M = e.magic(c["G"], c["b"])
        return e.last_tail_path(), v, M

    shared = sg.ProjectedProcessEngine(0)
    try:
        for c, bad in steps:
            got = run(shared, c, bad)
            fresh = sg.ProjectedProcessEngine(0)
            try:
                want = run(fresh, c, bad)
            finally:
                fresh.close()
            assert got[0] == want[0] == (0 if bad else 1)
            assert same_bits(got[1:], want[1:]), c["name"]
    finally:
        shared.close()


def test_range_failure_is_kept():
    """Forced int8 on points outside its operand range: finish raises OperandRangeError, a second finish raises it
    again, magic() on the window's statistics is refused, and magic(G, b) still works."""
    e = sg.ProjectedProcessEngine(0)
    try:
        rng = np.random.default_rng(5)
        X = rng.standard_normal((500, 4)) * 1e4
        y = rng.standard_normal(500)
        Z = X[:64].copy()
        e.set_precision(N.SGP_PREC_I8)
        e.begin(1 * sg.ARDRBFKernel(np.full(4, 1.0)) + sg.const(1e-2) * sg.EyeKernel(), Z)
        e.accumulate(X, y)
        with pytest.raises(sg.OperandRangeError):
            e.finish()
        with pytest.raises(sg.OperandRangeError):
            e.finish()
        with pytest.raises(sg.OperandRangeError):
            e.finish(copy_out=False)
        with pytest.raises(sg.TrainingVectorsNotInitializedException):
            e.magic()
        with pytest.raises(sg.TrainingVectorsNotInitializedException):
            e.predict(X[:3])
        k0 = (1 * oracle.ARDRBFKernel(np.full(4, 1.0)) + oracle.const(1e-2) * oracle.EyeKernel()).set_training_vectors(Z)
        Kmn = k0.cross_kernel(X).T
        G, b = Kmn @ Kmn.T, Kmn @ y
        v, M = e.magic(G, b)
        assert oracle.tail_errors(k0, G, b, v, M)["omega"] <= TOL_OMEGA
        v2, M2 = e.magic()                              # G_in closed the window with the caller's statistics
        assert np.array_equal(v, v2) and np.array_equal(M, M2)
        e.predict(X[:3])
    finally:
        e.close()
