"""GPU tests of kernel evaluation (`sgp_kernel_eval`, `sgp_kernel_eval_device`) through the kernel DSL's methods:
the reference's own goldens, K and every dK against the oracle over kernels, dimensions and tile / window edges, the
bit-identity contracts (host = device = split calls, fp32 = its upcast, exact symmetry, CROSS = sgp_cross_kernel),
isolation from an open statistics window and an installed magic pair, every refusal, and the BCM gradient."""
import ctypes as C

import numpy as np
import pytest
import torch

import oracle
import spark_gp_b200 as sg
from spark_gp_b200 import _native as N

pytestmark = pytest.mark.gpu

DATASET = np.array([[1.0, 2.0], [2.0, 3.0], [5.0, 7.0]])
ROWS, COLS, CHUNK = 32, 64, 32          # kernel_eval.cu: kEvalRows, kEvalCols, kEvalChunk


@pytest.fixture(scope="module")
def eng():
    e = sg.ProjectedProcessEngine(0)
    yield e
    e.close()


def ard_beta(rng, d):
    """Non-uniform betas with zeros, scaled so that q stays of order one."""
    beta = rng.uniform(0.2, 1.5, d) / np.sqrt(d)
    beta[::3] = 0.0
    return beta


def kernels(rng, d):
    """(name, library kernel, oracle kernel) pairs: ARD, RBF, Eye only, const, nested trainable scalars, white noise, and
    sums of 1 to 4 non-Eye terms plus Eye terms."""
    b1, b2 = ard_beta(rng, d), rng.uniform(0.1, 1.0, d) / np.sqrt(d)
    s = float(np.sqrt(d))
    return [
        ("ard", lambda m: 1 * m.ARDRBFKernel(b1)),
        ("rbf", lambda m: m.RBFKernel(0.8 * s)),
        ("eye", lambda m: m.const(0.5) * m.EyeKernel()),
        ("nested", lambda m: m.Scalar(0.7) * (2.0 * m.ARDRBFKernel(b1) + m.Scalar(0.3) * m.RBFKernel(0.6 * s))
         + m.const(0.25) * m.EyeKernel() + m.WhiteNoiseKernel(0.1, 0.0, 1.0)),
        ("four", lambda m: 0.5 * m.ARDRBFKernel(b1) + m.const(0.3) * m.ARDRBFKernel(b2) + 0.2 * m.RBFKernel(s)
         + m.Scalar(0.1) * m.RBFKernel(0.5 * s) + m.WhiteNoiseKernel(0.05, 0.0, 1.0) + m.const(1e-3) * m.EyeKernel()),
    ]


def pair(factory):
    return factory(sg), factory(oracle)


def oracle_eval(ok, A, B=None):
    """The oracle's (K, dK): trainingKernelAndDerivative on A, or for CROSS the A x B block of it on [A; B] (no Eye
    term reaches that block)."""
    if B is None:
        K, dK = ok.set_training_vectors(A).training_kernel_and_derivative()
        return K, np.array(dK).reshape(-1, len(A), len(A))
    n = len(A)
    K, dK = ok.set_training_vectors(np.vstack([A, B])).training_kernel_and_derivative()
    return K[:n, n:], np.array(dK).reshape(-1, len(K), len(K))[:, :n, n:]


def close(got, ref, rel=1e-13):
    """got within rel of each matrix's largest magnitude (a few ulps of the summed terms at these sizes)."""
    got, ref = np.asarray(got), np.asarray(ref)
    assert got.shape == ref.shape
    for g, r in zip(got.reshape(-1, *ref.shape[-2:]), ref.reshape(-1, *ref.shape[-2:])):
        scale = max(np.abs(r).max(), 1e-300)
        assert np.abs(g - r).max() <= rel * scale, np.abs(g - r).max() / scale


def dev(x):
    return torch.as_tensor(x, device="cuda:0")


# ---- the reference's goldens (RBFKernelTest.scala, ARDRBFKernelTest.scala) ----------------------------------------

def test_reference_goldens():
    rbf = sg.RBFKernel(np.sqrt(0.2)).setTrainingVectors(DATASET)
    correct = np.array([[1.000000e+00, 6.737947e-03, 3.053624e-45],
                        [6.737947e-03, 1.000000e+00, 7.187782e-28],
                        [3.053624e-45, 7.187782e-28, 1.000000e+00]])
    assert np.allclose(rbf.trainingKernel(), correct, rtol=1e-6, atol=0)
    rbf.setTrainingVectors(DATASET[1:])
    assert np.allclose(rbf.crossKernel(DATASET[:1]), [[6.737947e-03, 3.053624e-45]], rtol=1e-6, atol=0)
    row = rbf.crossKernel(DATASET[0])
    assert row.shape == (2,) and np.allclose(row, [6.737947e-03, 3.053624e-45], rtol=1e-6, atol=0)
    h = 1e-3
    num = lambda k0, k1: (k1.setTrainingVectors(DATASET).trainingKernel()
                          - k0.setTrainingVectors(DATASET).trainingKernel()) / (2 * h)
    dK = sg.RBFKernel(0.2).setTrainingVectors(DATASET).trainingKernelAndDerivative()[1][0]
    assert np.all(np.abs(dK - num(sg.RBFKernel(0.2 - h), sg.RBFKernel(0.2 + h))) < 1e-3)
    beta = np.array([0.2, 0.3])
    dK = sg.ARDRBFKernel(beta).setTrainingVectors(DATASET).trainingKernelAndDerivative()[1].sum(0)
    assert np.all(np.abs(dK - num(sg.ARDRBFKernel(beta - h), sg.ARDRBFKernel(beta + h))) < 1e-3)


# ---- against the oracle ---------------------------------------------------------------------------------------------

@pytest.mark.parametrize("d", [1, 3, 16, 33, 65, 100, 784])
def test_every_kernel_against_oracle(d):
    rng = np.random.default_rng(d)
    A, B = rng.random((37, d)), rng.random((70, d))
    for name, f in kernels(rng, d):
        k, ok = pair(f)
        K, dK = k.setTrainingVectors(A).trainingKernelAndDerivative()
        K0, dK0 = oracle_eval(ok, A)
        close(K, K0)
        assert dK.shape == dK0.shape, name
        if len(dK0):
            close(dK, dK0)
        k.setTrainingVectors(B)
        K0, _ = oracle_eval(ok, A, B)
        close(k.crossKernel(A), K0)


@pytest.mark.parametrize("n", [1, ROWS - 1, ROWS + 1, 2 * ROWS + 1])
@pytest.mark.parametrize("m", [1, COLS - 1, COLS + 1])
def test_tile_edges_cross_with_derivatives(eng, n, m):
    rng = np.random.default_rng(n * 1000 + m)
    d = CHUNK + 1
    A, B = rng.random((n, d)), rng.random((m, d))
    k, ok = pair(kernels(rng, d)[3][1])
    K, dK = eng.kernel_eval(k, A, B, derivatives=True)
    K0, dK0 = oracle_eval(ok, A, B)
    close(K, K0)
    close(dK, dK0)


@pytest.mark.parametrize("n", [1, ROWS - 1, ROWS + 1, COLS - 1, COLS + 1])
def test_tile_edges_training(n):
    rng = np.random.default_rng(n)
    A = rng.random((n, 5))
    k, ok = pair(kernels(rng, 5)[4][1])
    K, dK = k.setTrainingVectors(A).trainingKernelAndDerivative()
    K0, dK0 = oracle_eval(ok, A)
    close(K, K0)
    close(dK, dK0)


# ---- bit-identity contracts -----------------------------------------------------------------------------------------

@pytest.mark.parametrize("d", [3, 33, 100])
def test_host_device_fp32_symmetry_and_splits(eng, d):
    rng = np.random.default_rng(7 + d)
    A, B = rng.random((90, d)), rng.random((130, d))
    for name, f in kernels(rng, d):
        k = f(sg)
        for A_ in (A, A.astype(np.float32)):
            up = np.asarray(A_, dtype=np.float64)
            K, dK = eng.kernel_eval(k, A_, None, True)
            Kd, dKd = eng.kernel_eval(k, dev(A_), None, True)
            assert Kd.dtype == torch.float64 and Kd.is_cuda
            np.testing.assert_array_equal(K, Kd.cpu().numpy())
            np.testing.assert_array_equal(dK, dKd.cpu().numpy())
            Ku, dKu = eng.kernel_eval(k, up, None, True)
            np.testing.assert_array_equal(K, Ku)                         # fp32 = its upcast
            np.testing.assert_array_equal(dK, dKu)
            np.testing.assert_array_equal(K, K.T)                        # exact symmetry
            np.testing.assert_array_equal(dK, dK.transpose(0, 2, 1))
            Kc, dKc = eng.kernel_eval(k, A_, B, True)
            Kcd, dKcd = eng.kernel_eval(k, dev(A_), dev(B), True)
            np.testing.assert_array_equal(Kc, Kcd.cpu().numpy())
            np.testing.assert_array_equal(dKc, dKcd.cpu().numpy())
            np.testing.assert_array_equal(Kc, eng.kernel_eval(k, up, B, True)[0])
            parts = [eng.kernel_eval(k, A_[s], B, True) for s in (slice(0, 1), slice(1, 33), slice(33, None))]
            np.testing.assert_array_equal(Kc, np.vstack([p[0] for p in parts]))   # the same rows over several calls
            np.testing.assert_array_equal(dKc, np.concatenate([p[1] for p in parts], axis=1))


def test_host_windows_equal_one_device_launch(eng):
    """A host call of three windows (16, 16 and 1 rows of 4 matrices of 2^19 columns: 256 MiB per window) against one
    device launch, bit for bit, and against the oracle on a sample of columns."""
    rng = np.random.default_rng(5)
    d, n, m = 2, 33, 1 << 19
    A, B = rng.random((n, d)), rng.random((m, d))
    k, ok = pair(lambda mod: 1 * mod.ARDRBFKernel(np.array([0.7, 0.0])) + mod.const(0.1) * mod.EyeKernel())
    K, dK = eng.kernel_eval(k, A, B, True)
    Kd, dKd = eng.kernel_eval(k, dev(A), dev(B), True)
    np.testing.assert_array_equal(K, Kd.cpu().numpy())
    del Kd
    np.testing.assert_array_equal(dK, dKd.cpu().numpy())
    del dKd
    cols = np.r_[0:3, rng.choice(m, 200, replace=False), m - 3:m]
    K0, dK0 = oracle_eval(ok, A, B[cols])
    close(K[:, cols], K0)
    close(dK[:, :, cols], dK0)


def test_training_windows_equal_one_device_launch(eng):
    """TRAINING over several host windows (the diagonal moves with each window's first row) against one launch."""
    rng = np.random.default_rng(6)
    n = 3000                                    # 1 + 17 matrices of 3000 columns: 621 rows per window
    A = rng.random((n, 16))
    k = sg.ARDRBFKernel(ard_beta(rng, 16)) + sg.const(0.2) * sg.EyeKernel()
    K, dK = eng.kernel_eval(k, A, None, True)
    Kd, dKd = eng.kernel_eval(k, dev(A), None, True)
    np.testing.assert_array_equal(K, Kd.cpu().numpy())
    np.testing.assert_array_equal(dK, dKd.cpu().numpy())
    np.testing.assert_array_equal(K, K.T)
    assert np.all(np.diag(K) == 1.2)


@pytest.mark.parametrize("d", [3, 33, 100])
def test_cross_equals_sgp_cross_kernel(eng, d):
    rng = np.random.default_rng(11 + d)
    X, Z = rng.random((150, d)), rng.random((90, d))
    for name, f in kernels(rng, d):
        k = f(sg)
        eng.begin(k, Z)
        np.testing.assert_array_equal(k.setTrainingVectors(Z).crossKernel(X), eng.cross_kernel(X))


def test_tensor_training_vectors_stay_on_device():
    rng = np.random.default_rng(3)
    A = rng.random((50, 4)).astype(np.float32)
    k = 1 * sg.ARDRBFKernel(ard_beta(rng, 4)) + sg.const(0.1) * sg.EyeKernel()
    Kh, dKh = k.setTrainingVectors(A).trainingKernelAndDerivative()
    k.setTrainingVectors(dev(A))
    Kd, dKd = k.trainingKernelAndDerivative()
    assert Kd.is_cuda and Kd.dtype == torch.float64 and dKd.shape == (5, 50, 50)
    np.testing.assert_array_equal(Kh, Kd.cpu().numpy())
    np.testing.assert_array_equal(dKh, dKd.cpu().numpy())
    row = k.crossKernel(dev(A[0]))
    assert row.is_cuda and row.shape == (50,)
    assert np.allclose(row.cpu().numpy(), Kh[0] - 0.1 * (np.arange(50) == 0), rtol=1e-14, atol=0)
    diag = k.trainingKernelDiag()
    assert diag.is_cuda and torch.equal(diag, torch.diagonal(Kd))


# ---- isolation from the statistics window and the magic pair --------------------------------------------------------

def test_window_and_magic_pair_untouched(eng):
    rng = np.random.default_rng(21)
    d = 6
    X = rng.random((20000, d))
    y = np.sin(3 * X.sum(1))
    Z, Xt = X[:120], rng.random((300, d))
    k = 1 * sg.ARDRBFKernel(np.full(d, 0.8)) + sg.const(1e-2) * sg.EyeKernel()
    other = sg.Scalar(0.4) * sg.RBFKernel(0.9) + sg.const(0.3) * sg.EyeKernel()
    evals = lambda: (eng.kernel_eval(other, Xt, None, True), eng.kernel_eval(other, dev(Xt), dev(Z), True),
                     eng.kernel_eval(other, Xt[:5], Z, False))

    def run(interleave):
        eng.set_precision(N.SGP_PREC_AUTO)
        eng.begin(k, Z)
        eng.accumulate(X[:8000], y[:8000])
        if interleave:
            evals()
        eng.accumulate(X[8000:], y[8000:])
        G, b = eng.finish()
        path = eng.last_path()
        mv, mm = eng.magic()
        p0 = eng.predict(Xt)
        if interleave:
            evals()
        return G, b, path, mv, mm, p0, eng.predict(Xt)

    ref, got = run(False), run(True)
    for r, g in zip(ref, got):
        if isinstance(r, tuple):
            for a, b in zip(r, g):
                np.testing.assert_array_equal(a, b)
        else:
            np.testing.assert_array_equal(r, g)


# ---- refusals -------------------------------------------------------------------------------------------------------

def test_refusals_before_any_launch(eng):
    lib = eng._lib
    d = 3
    k = 1 * sg.ARDRBFKernel(np.array([0.5, 0.0, 1.0])) + sg.RBFKernel(1.3) + sg.const(0.1) * sg.EyeKernel()
    desc, arr, nh, keep = eng._descriptors(k, d)
    A, B = np.random.default_rng(0).random((4, d)), np.random.default_rng(1).random((5, d))
    K, dK = np.empty((5, 5)), np.empty((nh, 5, 5))
    p = N.ptr

    def call(fn=lib.sgp_kernel_eval, desc_=desc, arr_=arr, nh_=nh, A_=p(A), n=4, B_=p(B), m=5, d_=d,
             mode=N.SGP_KEVAL_CROSS, K_=p(K), dK_=p(dK)):
        before = eng.launch_count()
        rc = fn(eng._h, C.byref(desc_) if desc_ is not None else None, arr_, nh_, A_, 0, n, B_, m, d_, mode, K_, dK_)
        assert eng.launch_count() == before + (rc == N.SGP_OK)
        return rc

    assert call() == N.SGP_OK
    eng.sync()
    before = eng.launch_count()
    bad = [dict(n=0), dict(m=0), dict(d_=0), dict(A_=None), dict(K_=None), dict(mode=2), dict(B_=None),
           dict(mode=N.SGP_KEVAL_TRAINING), dict(mode=N.SGP_KEVAL_TRAINING, B_=None, m=5),
           dict(nh_=nh - 1), dict(nh_=-1), dict(arr_=None), dict(desc_=None), dict(desc_=N.KernelDesc(0, 0, None))]
    for kw in bad:
        assert call(**kw) == N.SGP_E_BADARG, kw
    # descriptors that do not match the kernel: a repeated ARD dim, a wrong value, an RBF_SIGMA on the ARD term
    for i, field, v in [(3, "dim", 0), (3, "value", 0.25), (4, "term", 0)]:
        old = getattr(arr[i], field)
        setattr(arr[i], field, v)
        assert call() == N.SGP_E_BADARG, (i, field)
        setattr(arr[i], field, old)
    assert call() == N.SGP_OK
    eng.sync()
    # device entry: host pointers are not device memory
    KD = torch.empty((5, 5), dtype=torch.float64, device="cuda:0")
    dKD = torch.empty((nh, 5, 5), dtype=torch.float64, device="cuda:0")
    Ad, Bd = dev(A), dev(B)
    tp = lambda t: C.c_void_p(t.data_ptr())
    fn = lib.sgp_kernel_eval_device
    for kw in [dict(A_=p(A)), dict(B_=p(B)), dict(K_=p(K)), dict(dK_=p(dK))]:
        args = dict(fn=fn, A_=tp(Ad), B_=tp(Bd), K_=tp(KD), dK_=tp(dKD))
        args.update(kw)
        assert call(**args) == N.SGP_E_BADARG, kw
    # a window that does not fit: one row of 1 + 5 matrices of 2^31 - 1 columns, double buffered (the outputs are never
    # touched: the refusal comes first)
    assert call(m=2 ** 31 - 1) == N.SGP_E_NOMEM
    assert eng.launch_count() == before + 1
    del keep


# ---- the BCM gradient -----------------------------------------------------------------------------------------------

def test_bcm_gradient_from_derivatives(eng):
    rng = np.random.default_rng(41)
    d, n = 4, 100
    X = rng.random((n, d))
    y = np.sin(3 * X.sum(1)) + 0.1 * rng.standard_normal(n)
    k = (sg.Scalar(0.9) * (sg.ARDRBFKernel(ard_beta(rng, d) + 0.3) + sg.Scalar(0.4) * sg.RBFKernel(0.8))
         + sg.WhiteNoiseKernel(0.05, 0.0, 1.0))
    eng.experts_upload(X, y, [0, n])
    _, grad = eng.bcm_nll(k)
    K, dK = k.setTrainingVectors(X).trainingKernelAndDerivative()
    Kinv = np.linalg.inv(K)
    alpha = Kinv @ y
    mine = -0.5 * np.einsum("hij,ij->h", dK, np.outer(alpha, alpha) - Kinv)
    assert np.abs(mine - grad).max() <= 1e-10 * np.abs(grad).max()
