"""GPU tests of kernel evaluation (`sgp_kernel_eval`, `sgp_kernel_eval_device`) element by element: every element of K
and of every dK against the extended-precision model of oracle/kernel_eval_model.py, within its own rounding bound.
The cases reach what the feature tests of tests/test_gpu_kernel_eval.py do not: row tiles past the 65535-tile grid
wrap, every kernel shape at the 32-wide staging edges, placements far from the origin, exp(-q) subnormal and zero, RBF
sigmas at both extremes, and hyper-parameter descriptors in any order.  Each test prints the largest fraction of the
bound it used."""
import ctypes as C
import time

import numpy as np
import pytest
import torch

import oracle
import spark_gp_b200 as sg
from oracle.kernel_eval_model import KernelEvalModel, bound_fraction, kernel_shapes
from spark_gp_b200 import _native as N

pytestmark = pytest.mark.gpu

ROWS, COLS, CHUNK = 32, 64, 32          # kernel_eval.cu: kEvalRows, kEvalCols, kEvalChunk
GRID_Y = 65535                          # launch_kernel_eval: grid.y, the row tiles of one pass of the grid
WINDOW_BYTES = 256 << 20                # sgp_internal.h: kPredictKBytes, K and dK of one host window


@pytest.fixture(scope="module")
def eng():
    e = sg.ProjectedProcessEngine(0)
    yield e
    e.close()


def dev(x):
    return torch.as_tensor(x, device="cuda:0")


def check(label, model, A, B, K, dK=None):
    """Every element of K, and of every dK plane, within the model's bound for rows A against B (B None: the training
    kernel of A).  Returns the largest fraction of the bound used."""
    X, bX, dX, bdX = model.evaluate(A, B, dK is not None)
    fr = bound_fraction(K, X, bX)
    if dK is not None:
        assert np.shape(dK) == dX.shape, label
        fr = max([fr] + [bound_fraction(g, x, b) for g, x, b in zip(dK, dX, bdX)])
    assert fr <= 1.0, (label, fr)
    return fr


def assert_symmetric(K, dK):
    np.testing.assert_array_equal(K, K.T)
    np.testing.assert_array_equal(dK, dK.transpose(0, 2, 1))


# ---- row tiles past the grid wrap -----------------------------------------------------------------------------------

N_WRAP = 2 * GRID_Y * ROWS + 33         # 131072 row tiles: CTA row 0 runs tiles 0, 65535 and 131070; the last holds 1 row


def wrap_kernel(m):
    """Four hyper-parameters (two ARD betas, a trainable scalar, sigma): five matrices.  const(0.7), not a bare 0.7,
    which would add a trainable scalar and shrink the host window below the wrap."""
    return (m.const(0.7) * m.ARDRBFKernel(np.array([0.7, 1.3])) + m.Scalar(0.4) * m.RBFKernel(0.9)
            + m.const(0.1) * m.EyeKernel())


def wrap_rows(rng, extra):
    """Every row of tiles 0, 1, 65534, 65535, 65536, 131069, 131070 and 131071, the rows `extra`, and 4096 random rows."""
    tiles = [0, 1, GRID_Y - 1, GRID_Y, GRID_Y + 1, 2 * GRID_Y - 1, 2 * GRID_Y, 2 * GRID_Y + 1]
    rows = [np.arange(t * ROWS, min((t + 1) * ROWS, N_WRAP)) for t in tiles]
    rows = np.unique(np.concatenate(rows + [extra, rng.choice(N_WRAP, 4096, replace=False)]))
    assert rows[-1] == N_WRAP - 1 and N_WRAP - 1 == (2 * GRID_Y + 1) * ROWS
    return rows


def test_row_tiles_past_the_grid_wrap(eng):
    """CROSS with derivatives on 4,194,273 rows: one device launch whose CTAs each run up to three row tiles, and a host
    call whose first window of ~2.24M rows is itself past the wrap and ends inside a tile."""
    rng = np.random.default_rng(65535)
    d, m = 2, 3
    A, B = rng.random((N_WRAP, d)), rng.random((m, d))
    k, model = wrap_kernel(sg), KernelEvalModel(wrap_kernel(oracle))
    nh = len(k.getHyperparameters())
    win = WINDOW_BYTES // ((1 + nh) * m * 8)            # sgp_kernel_eval's rows per window
    assert nh == 4 and GRID_Y * ROWS < win < N_WRAP and win % ROWS != 0
    t0 = time.perf_counter()
    K, dK = eng.kernel_eval(k, A, B, True)
    Kd, dKd = eng.kernel_eval(k, dev(A), dev(B), True)
    np.testing.assert_array_equal(K, Kd.cpu().numpy())
    del Kd
    np.testing.assert_array_equal(dK, dKd.cpu().numpy())
    del dKd
    t1 = time.perf_counter()
    rows = wrap_rows(rng, np.arange(win - 40, win + 40))
    fr = check("wrap", model, A[rows], B, K[rows], dK[:, rows])
    # the same rows in small calls of their own: an element's bits do not depend on its tile, launch or window
    for lo, hi in [(GRID_Y * ROWS - 40, GRID_Y * ROWS + 40), (2 * GRID_Y * ROWS - 8, N_WRAP), (win - 40, win + 40)]:
        Ks, dKs = eng.kernel_eval(k, A[lo:hi], B, True)
        np.testing.assert_array_equal(Ks, K[lo:hi])
        np.testing.assert_array_equal(dKs, dK[:, lo:hi])
    print("\nwrap, m = 3 with derivatives: %d rows checked, largest fraction of the bound %.3g (calls %.1f s, checks "
          "%.1f s)" % (len(rows), fr, t1 - t0, time.perf_counter() - t1))


def test_row_tiles_past_the_grid_wrap_two_column_tiles(eng):
    """K only, m = 65 (one full and one 1-column tile), one device launch past the wrap."""
    rng = np.random.default_rng(65536)
    d, m = 2, COLS + 1
    A, B = rng.random((N_WRAP, d)), rng.random((m, d))
    k, model = wrap_kernel(sg), KernelEvalModel(wrap_kernel(oracle))
    rows = wrap_rows(rng, np.arange(0))
    spans = [(GRID_Y * ROWS - 40, GRID_Y * ROWS + 40), (2 * GRID_Y * ROWS - 8, N_WRAP)]
    t0 = time.perf_counter()
    Kd, _ = eng.kernel_eval(k, dev(A), dev(B), False)
    Ks = Kd[dev(rows)].cpu().numpy()
    parts = [Kd[lo:hi].cpu().numpy() for lo, hi in spans]
    del Kd
    t1 = time.perf_counter()
    fr = check("wrap m=65", model, A[rows], B, Ks)
    for (lo, hi), p in zip(spans, parts):
        np.testing.assert_array_equal(eng.kernel_eval(k, A[lo:hi], B, False)[0], p)
    print("\nwrap, m = 65, K only: %d rows checked, largest fraction of the bound %.3g (call %.1f s, checks %.1f s)"
          % (len(rows), fr, t1 - t0, time.perf_counter() - t1))


# ---- every element, every kernel shape ------------------------------------------------------------------------------

DIMS = [1, CHUNK - 1, CHUNK, CHUNK + 1, 2 * CHUNK - 1, 2 * CHUNK, 2 * CHUNK + 1, 100]
CROSS_SIZES = [(ROWS + 1, COLS + 1), (ROWS, COLS), (ROWS - 1, COLS - 1), (2 * ROWS + 1, 2 * COLS + 1)]
TRAINING_SIZES = [COLS + 1, ROWS + 1, COLS, 2 * ROWS - 1]


@pytest.mark.parametrize("d", DIMS)
def test_every_element_every_kernel(eng, d):
    """The six kernel shapes in CROSS and TRAINING, fp64 and fp32 A, host and device entries, at tile-edge sizes."""
    i = DIMS.index(d)
    rng = np.random.default_rng(300 + d)
    (n, m), nt = CROSS_SIZES[i % 4], TRAINING_SIZES[i % 4]
    A, B, At = rng.random((n, d)), rng.random((m, d)), rng.random((nt, d))
    worst = {}
    for name, f in kernel_shapes(rng, d):
        k, model = f(sg), KernelEvalModel(f(oracle))
        for mode, A_, B_ in (("cross", A, B), ("training", At, None)):
            for X in (A_, A_.astype(np.float32)):
                K, dK = eng.kernel_eval(k, X, B_, True)
                Kd, dKd = eng.kernel_eval(k, dev(X), None if B_ is None else dev(B_), True)
                np.testing.assert_array_equal(K, Kd.cpu().numpy())
                np.testing.assert_array_equal(dK, dKd.cpu().numpy())
                if B_ is None:
                    assert_symmetric(K, dK)
                label = "%s %s %s" % (name, mode, X.dtype)
                worst[label] = check(label, model, X.astype(np.float64), B_, K, dK)
    top = max(worst, key=worst.get)
    print("\nd = %d: largest fraction of the bound %.3g (%s)" % (d, worst[top], top))


# ---- placement far from the origin ----------------------------------------------------------------------------------

@pytest.mark.parametrize("offset,dims,dtype", [(1e3, "all", np.float64), (1e6, "all", np.float64),
                                               (1e3, "one", np.float64), (1e6, "one", np.float64),
                                               (1e3, "all", np.float32), (1e3, "one", np.float32)])
def test_far_placement(eng, offset, dims, dtype):
    """A and B offset by `offset` / beta (the largest beta of any term per feature) in every feature or in the one with
    the largest beta; an fp32 A is judged by its upcast."""
    d = 33
    rng = np.random.default_rng(int(offset) + d)
    X, Y = rng.random((ROWS + 1, d)), rng.random((COLS + 1, d))
    worst = {}
    for name, f in kernel_shapes(rng, d):
        k, model = f(sg), KernelEvalModel(f(oracle))
        bmax = np.max([model.beta(t, d).astype(np.float64) for t in range(len(model.terms))] + [np.zeros(d)], axis=0)
        off = offset / np.where(bmax > 0, bmax, 1.0)
        if dims == "one":
            off = np.where(np.arange(d) == np.argmax(bmax), off, 0.0)
        A = (X + off).astype(dtype)
        for mode, B in (("cross", Y + off), ("training", None)):
            K, dK = eng.kernel_eval(k, A, B, True)
            if B is None:
                assert_symmetric(K, dK)
            label = "%s %s" % (name, mode)
            worst[label] = check(label, model, A.astype(np.float64), B, K, dK)
    top = max(worst, key=worst.get)
    print("\noffset %g (%s, %s): largest fraction of the bound %.3g (%s)"
          % (offset, dims, np.dtype(dtype).name, worst[top], top))


# ---- exp(-q) subnormal and zero -------------------------------------------------------------------------------------

Q_TARGETS = [700.0, 708.0, 740.0, 745.0, 746.0, 1e4]    # exp(-q): normal, normal, subnormal x 3 (the last rounds to 0
                                                          # or 2^-1074), 0


def test_underflow(eng):
    """Pairs whose ARD q is each target (along one feature and split over two), mixed with near pairs in one call."""
    rng = np.random.default_rng(745)
    beta = np.array([0.9, 0.4, 0.0])
    f = lambda m: (m.Scalar(0.8) * m.ARDRBFKernel(beta) + m.Scalar(0.5) * m.RBFKernel(0.3)
                   + m.WhiteNoiseKernel(0.3, 0.0, 1.0))
    k, model = f(sg), KernelEvalModel(f(oracle))
    a0 = np.array([0.3, -0.2, 0.7])
    far = []
    for q in Q_TARGETS:
        far.append(a0 + [np.sqrt(q) / beta[0], 0.0, 0.1])
        far.append(a0 + [np.sqrt(q / 2) / beta[0], np.sqrt(q / 2) / beta[1], -0.4])
    near = a0 + rng.uniform(-0.3, 0.3, (6, 3))
    A, B = np.vstack([a0, near[:3]]), np.vstack(far + [near[3:]])
    q = (((A[0] - B[:len(far)]) * beta) ** 2).sum(1)
    assert np.allclose(q, np.repeat(Q_TARGETS, 2), rtol=1e-12)
    tiny = np.finfo(np.float64).tiny
    worst, low = {}, {}
    for mode, A_, B_ in (("cross", A, B), ("training", np.vstack([A, B]), None)):
        K, dK = eng.kernel_eval(k, A_, B_, True)
        Kd, dKd = eng.kernel_eval(k, dev(A_), None if B_ is None else dev(B_), True)
        np.testing.assert_array_equal(K, Kd.cpu().numpy())
        np.testing.assert_array_equal(dK, dKd.cpu().numpy())
        if B_ is None:
            assert_symmetric(K, dK)
        worst[mode] = check(mode, model, A_, B_, K, dK)
        c0 = 0 if B_ is not None else len(A)             # the far points' first column
        row = K[0, c0:c0 + len(far)]
        assert np.any(row >= tiny) and np.any((row > 0) & (row < tiny)) and np.any(row == 0), row
        # the elements whose exact K is below fp64's smallest normal: where exp's own error is the absolute floor's
        X, bX, dX, bdX = model.evaluate(A_, B_)
        sub = X < tiny
        low[mode] = max([bound_fraction(K[sub], X[sub], bX[sub])]
                        + [bound_fraction(g[sub], x[sub], b[sub]) for g, x, b in zip(dK, dX, bdX)])
    print("\nunderflow: largest fraction of the bound %.3g (cross), %.3g (training); on elements whose exact K is "
          "subnormal or zero %.3g (cross), %.3g (training)" % (worst["cross"], worst["training"], low["cross"],
                                                              low["training"]))


@pytest.mark.parametrize("sigma", [1e-6, 1e150])
def test_rbf_sigma_extremes(eng, sigma):
    """RBF at its default lower bound (pairs at distances of order sigma and at q = 745) and at 1e150 (sigma^3
    overflows fp64: the sigma plane is 0, as the exact value rounds to)."""
    rng = np.random.default_rng(int(np.log10(sigma)) + 200)
    d = 2
    f = lambda m: m.Scalar(0.7) * m.RBFKernel(sigma) + m.const(0.2) * m.ARDRBFKernel(np.array([0.5, 1.5]))
    k, model = f(sg), KernelEvalModel(f(oracle))
    base = rng.random((ROWS + 1, d))
    if sigma < 1:
        base[1:20] = base[0] + rng.normal(size=(19, d)) * sigma
        base[20:26] = base[0] + np.array([[np.sqrt(2 * q) * sigma, 0.0] for q in Q_TARGETS])
    A, B = base[:9], base[9:]
    worst = {}
    for mode, A_, B_ in (("cross", A, B), ("training", base, None)):
        K, dK = eng.kernel_eval(k, A_, B_, True)
        if B_ is None:
            assert_symmetric(K, dK)
        worst[mode] = check(mode, model, A_, B_, K, dK)
    print("\nRBF sigma %g: largest fraction of the bound %.3g (cross), %.3g (training)"
          % (sigma, worst["cross"], worst["training"]))


# ---- descriptor order -----------------------------------------------------------------------------------------------

def test_descriptor_order(eng):
    """The descriptors in three random orders: each dK plane goes to its descriptor's index, with the canonical bits, and
    K does not move (both entries, both modes)."""
    rng = np.random.default_rng(17)
    d = 5
    A, B = rng.random((ROWS + 1, d)), rng.random((COLS + 1, d))
    lib, p = eng._lib, N.ptr
    tp = lambda t: C.c_void_p(t.data_ptr())
    for name, f in kernel_shapes(rng, d):
        k = f(sg)
        desc, arr, nh, keep = eng._descriptors(k, d)
        if nh < 2:
            continue
        perms = [rng.permutation(nh) for _ in range(3)]
        for mode, B_ in ((N.SGP_KEVAL_CROSS, B), (N.SGP_KEVAL_TRAINING, None)):
            n, m = len(A), len(A) if B_ is None else len(B_)

            def run(hypers, on_device):
                if on_device:
                    K = torch.empty((n, m), dtype=torch.float64, device="cuda:0")
                    dK = torch.empty((nh, n, m), dtype=torch.float64, device="cuda:0")
                    Ad, Bd = dev(A), None if B_ is None else dev(B_)
                    rc = lib.sgp_kernel_eval_device(eng._h, C.byref(desc), hypers, nh, tp(Ad), 0, n,
                                                    None if Bd is None else tp(Bd), m, d, mode, tp(K), tp(dK))
                    assert rc == N.SGP_OK, lib.sgp_last_error(eng._h)
                    eng.sync()
                    return K.cpu().numpy(), dK.cpu().numpy()
                K, dK = np.empty((n, m)), np.empty((nh, n, m))
                rc = lib.sgp_kernel_eval(eng._h, C.byref(desc), hypers, nh, p(A), 0, n, None if B_ is None else p(B_),
                                         m, d, mode, p(K), p(dK))
                assert rc == N.SGP_OK, lib.sgp_last_error(eng._h)
                return K, dK

            for on_device in (False, True):
                K0, dK0 = run(arr, on_device)
                for perm in perms:
                    K, dK = run((N.Hyper * nh)(*[arr[j] for j in perm]), on_device)
                    np.testing.assert_array_equal(K, K0)
                    np.testing.assert_array_equal(dK, dK0[perm])
        del keep


def test_five_terms_refused_before_any_launch(eng):
    d = 3
    b = np.array([0.5, 0.0, 1.0])
    k = (sg.ARDRBFKernel(b) + sg.RBFKernel(1.0) + sg.ARDRBFKernel(2 * b) + sg.RBFKernel(2.0) + sg.ARDRBFKernel(b / 2)
         + sg.const(0.1) * sg.EyeKernel())
    desc, arr, nh, keep = eng._descriptors(k, d)
    A = np.random.default_rng(0).random((4, d))
    K, dK = np.empty((4, 4)), np.empty((nh, 4, 4))
    Kd = torch.empty((4, 4), dtype=torch.float64, device="cuda:0")
    dKd = torch.empty((nh, 4, 4), dtype=torch.float64, device="cuda:0")
    Ad = dev(A)
    tp = lambda t: C.c_void_p(t.data_ptr())
    before = eng.launch_count()
    for fn, args in [(eng._lib.sgp_kernel_eval, (N.ptr(A), 0, 4, None, 4, d, N.SGP_KEVAL_TRAINING, N.ptr(K), N.ptr(dK))),
                     (eng._lib.sgp_kernel_eval_device, (tp(Ad), 0, 4, None, 4, d, N.SGP_KEVAL_TRAINING, tp(Kd), tp(dKd)))]:
        assert fn(eng._h, C.byref(desc), arr, nh, *args) == N.SGP_E_BADARG
        assert "too many non-Eye kernel terms" in eng._lib.sgp_last_error(eng._h).decode()
    assert eng.launch_count() == before
    del keep
