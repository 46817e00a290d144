"""Prediction on the GPU (`sgp_predict`, `sgp_predict_device`) against the fp64 oracle (run on an H100: `pytest -m gpu`).

A magic pair (v, M) is installed with `sgp_set_magic`, so that only prediction is under test: the oracle's cross kernel
gives K0 = k(X, Z), and mean = K0 v, var = selfKernel + K0 M K0^T.  Everything is fp64; the tolerance is 1e-11 of the
summed magnitudes each output adds up (|K0| |v| for the mean, selfKernel + |K0| |M| |K0|^T for the variance), as for the
chunk-boundary test of test_gpu_entry_points.py.  The edges covered: m at every 64- and 128-wide tile edge of the
triangular schedule, d at the 32-dim staging chunk edges, 1 to 4 non-Eye terms, n at the CTA and staging-window edges.
"""
import ctypes as C

import numpy as np
import pytest
import torch

import oracle
import spark_gp_b200 as sg
from spark_gp_b200 import _native as N
from spark_gp_b200.regression import ExplicitActiveSetProvider

pytestmark = pytest.mark.gpu

TOL = 1e-11


@pytest.fixture(scope="module")
def eng():
    e = sg.ProjectedProcessEngine(0)
    yield e
    e.close()


def kernels(S, n_terms, d, rng_seed=3):
    """A flattened kernel with n_terms non-Eye terms (ARD with non-uniform beta and RBF, scales 0.05 .. 20) and Eye terms."""
    rng = np.random.default_rng(rng_seed)
    parts = [lambda: 1.3 * S.ARDRBFKernel(rng_beta(rng, d)),
             lambda: 0.05 * S.RBFKernel(0.7 * np.sqrt(d)),
             lambda: 20.0 * S.ARDRBFKernel(0.5 * rng_beta(rng, d)),
             lambda: 2.0 * S.RBFKernel(1.5 * np.sqrt(d))]
    k = parts[0]()
    for t in range(1, n_terms):
        k = k + parts[t]()
    k = k + S.const(0.05) * S.EyeKernel()
    if n_terms % 2 == 0:
        k = k + S.const(1e-3) * S.EyeKernel()
    return k


def rng_beta(rng, d):
    return (0.3 + rng.random(d)) / np.sqrt(d)


def make_case(m, d, n_terms, seed=0, offset=None):
    rng = np.random.default_rng(seed)
    Z = rng.random((m, d)) * 2.0
    if offset is not None:
        Z = Z + offset
    v = rng.standard_normal(m)
    S = rng.standard_normal((m, m))
    M = (S + S.T) * 50.0                                      # entries of the size of an inverse kernel matrix's
    k_sg = kernels(sg, n_terms, d)
    k0 = kernels(oracle, n_terms, d)
    k0 = k0.set_hyperparameters(k0.get_hyperparameters()).set_training_vectors(Z)
    return dict(Z=Z, v=v, M=M, k=k_sg, k0=k0, d=d, m=m, offset=offset)


def points(c, n, seed=1):
    X = np.random.default_rng(seed).random((n, c["d"])) * 2.0
    return X + c["offset"] if c["offset"] is not None else X


def errors(c, X, mean, var, M=None):
    M = c["M"] if M is None else M
    K0 = c["k0"].cross_kernel(X)
    A = np.abs(K0)
    m0 = K0 @ c["v"]
    em = float((np.abs(mean - m0) / np.maximum(A @ np.abs(c["v"]), 1e-300)).max())
    if var is None:
        return em, 0.0
    sk = c["k0"].self_kernel(None)
    v0 = sk + np.einsum("ti,ti->t", K0 @ M, K0)
    scale = sk + np.einsum("ti,ti->t", A @ np.abs(M), A)
    return em, float((np.abs(var - v0) / scale).max())


def install(eng, c, M=None):
    eng.set_precision(N.SGP_PREC_AUTO)
    eng.begin(c["k"], c["Z"])
    eng.set_magic(c["v"], c["M"] if M is None else M)


def predict_dev(eng, X, with_var=True, f32=False):
    Xd = torch.from_numpy(np.ascontiguousarray(X, dtype=np.float32 if f32 else np.float64)).cuda()
    mean, var = eng.predict_tensor(Xd, with_variance=with_var)
    return mean.cpu().numpy(), (var.cpu().numpy() if var is not None else None)


# ---------------- oracle parity, device entry ----------------------------------------------------------------------------
@pytest.mark.parametrize("m", [1, 63, 64, 65, 127, 128, 129, 1000, 2100, 4000])
def test_parity_m(eng, m):
    c = make_case(m, 5, 2, seed=m)
    install(eng, c)
    X = points(c, 300)
    mean, var = predict_dev(eng, X)
    em, ev = errors(c, X, mean, var)
    print("m=%d: mean %.1e var %.1e" % (m, em, ev))
    assert em < TOL and ev < TOL


@pytest.mark.parametrize("d", [1, 5, 16, 33, 100, 784])
@pytest.mark.parametrize("f32", [False, True], ids=["f64", "f32"])
def test_parity_d(eng, d, f32):
    c = make_case(129, d, 1 + d % 4, seed=d)
    install(eng, c)
    X = points(c, 200)
    if f32:
        X = X.astype(np.float32).astype(np.float64)          # the oracle sees exactly what the kernel reads
    mean, var = predict_dev(eng, X, f32=f32)
    em, ev = errors(c, X, mean, var)
    print("d=%d f32=%s: mean %.1e var %.1e" % (d, f32, em, ev))
    assert em < TOL and ev < TOL


@pytest.mark.parametrize("n_terms", [1, 2, 3, 4])
def test_parity_terms(eng, n_terms):
    c = make_case(200, 7, n_terms, seed=10 + n_terms)
    install(eng, c)
    X = points(c, 150)
    mean, var = predict_dev(eng, X)
    em, ev = errors(c, X, mean, var)
    assert em < TOL and ev < TOL


# n at the CTA edges, and around the host entry's staging window (d = 784: 32 MB / (784 * 8) = 5350 points per chunk)
@pytest.mark.parametrize("n,d", [(1, 5), (63, 5), (64, 5), (65, 5), (5349, 784), (5350, 784), (5351, 784)])
def test_parity_n_host_and_device(eng, n, d):
    c = make_case(65, d, 2, seed=n)
    install(eng, c)
    X = points(c, n)
    mean, var = eng.predict(X)
    em, ev = errors(c, X, mean, var)
    assert em < TOL and ev < TOL
    dm, dv = predict_dev(eng, X)
    assert np.array_equal(dm, mean) and np.array_equal(dv, var)


def test_device_window_edge(eng):
    """m = 4000 pads to 4096 columns: the device entry's kernel window is 8192 points."""
    c = make_case(4000, 8, 1, seed=4)
    install(eng, c)
    X = points(c, 8193)
    mean, var = predict_dev(eng, X)
    em, ev = errors(c, X, mean, var)
    assert em < TOL and ev < TOL
    hm, hv = eng.predict(X)
    assert np.array_equal(hm, mean) and np.array_equal(hv, var)


# ---------------- the packing reads the symmetric part only --------------------------------------------------------------
def test_asymmetric_matrix(eng):
    c = make_case(300, 6, 2, seed=77)
    rng = np.random.default_rng(5)
    E = rng.standard_normal(c["M"].shape) * 50.0
    Ma = c["M"] + (E - E.T)
    install(eng, c, M=Ma)
    X = points(c, 400)
    mean, var = predict_dev(eng, X)
    em, ev = errors(c, X, mean, var, M=Ma)
    assert em < TOL and ev < TOL


# ---------------- bit identity -------------------------------------------------------------------------------------------
def test_bit_identity(eng):
    c = make_case(257, 16, 2, seed=9)
    install(eng, c)
    X32 = points(c, 3001).astype(np.float32)
    X = X32.astype(np.float64)
    hm, hv = eng.predict(X)
    dm, dv = predict_dev(eng, X)
    fm, fv = predict_dev(eng, X32, f32=True)
    assert np.array_equal(hm, dm) and np.array_equal(hv, dv)
    assert np.array_equal(fm, hm) and np.array_equal(fv, hv)
    a_m, a_v = eng.predict(X[:1234])
    b_m, b_v = eng.predict(X[1234:])
    assert np.array_equal(np.concatenate([a_m, b_m]), hm) and np.array_equal(np.concatenate([a_v, b_v]), hv)
    om, _ = eng.predict(X, with_variance=False)
    odm, _ = predict_dev(eng, X, with_var=False)
    assert np.array_equal(om, hm) and np.array_equal(odm, hm)
    rm, rv = eng.predict(X)
    assert np.array_equal(rm, hm) and np.array_equal(rv, hv)


# ---------------- placement ----------------------------------------------------------------------------------------------
@pytest.mark.parametrize("where", ["0", "10", "100", "1e3", "-1e3", "1e3_one_dim"])
def test_placement(eng, where):
    d = 4
    beta_scale = 1.0 / np.sqrt(d)                             # the ARD betas are O(1 / sqrt d): length scales ~ sqrt d
    if where == "1e3_one_dim":
        off = np.zeros(d)
        off[0] = 1e3 / beta_scale
    else:
        off = np.full(d, float(where) / beta_scale)
    c = make_case(150, d, 2, seed=21, offset=off)
    install(eng, c)
    X = points(c, 300)
    mean, var = predict_dev(eng, X)
    em, ev = errors(c, X, mean, var)
    print("placement %s: mean %.1e var %.1e" % (where, em, ev))
    assert em < TOL and ev < TOL


# ---------------- scale ------------------------------------------------------------------------------------------------------
def test_scale_1p3m(eng):
    c = make_case(1000, 16, 1, seed=31)
    install(eng, c)
    n = 1_300_000
    Xd = torch.rand((n, 16), dtype=torch.float64, device="cuda", generator=torch.Generator("cuda").manual_seed(7)) * 2.0
    mean, var = eng.predict_tensor(Xd)
    idx = np.concatenate([[0, n - 1], np.random.default_rng(3).choice(n, 5000, replace=False)])
    X = Xd[torch.from_numpy(idx).cuda()].cpu().numpy()
    em, ev = errors(c, X, mean.cpu().numpy()[idx], var.cpu().numpy()[idx])
    assert em < TOL and ev < TOL


# ---------------- state and isolation --------------------------------------------------------------------------------------
def test_state_and_arguments():
    e = sg.ProjectedProcessEngine(0)
    try:
        lib, h = e._lib, e._h
        Xd = torch.zeros((4, 3), dtype=torch.float64, device="cuda")
        out = torch.zeros(4, dtype=torch.float64, device="cuda")
        assert lib.sgp_predict_device(h, C.c_void_p(Xd.data_ptr()), 0, 4, C.c_void_p(out.data_ptr()), None) == N.SGP_E_STATE
        c = make_case(10, 3, 1)
        e.begin(c["k"], c["Z"])
        assert lib.sgp_predict_device(h, C.c_void_p(Xd.data_ptr()), 0, 4, C.c_void_p(out.data_ptr()), None) == N.SGP_E_STATE
        e.set_magic(c["v"], c["M"])
        assert lib.sgp_predict_device(h, None, 0, 4, C.c_void_p(out.data_ptr()), None) == N.SGP_E_BADARG
        assert lib.sgp_predict_device(h, C.c_void_p(Xd.data_ptr()), 0, 4, None, None) == N.SGP_E_BADARG
        assert lib.sgp_predict_device(h, C.c_void_p(Xd.data_ptr()), 0, -1, C.c_void_p(out.data_ptr()), None) == N.SGP_E_BADARG
        assert lib.sgp_predict_device(h, None, 0, 0, None, None) == N.SGP_OK
        assert lib.sgp_predict(h, None, 0, None, None) == N.SGP_OK
        assert lib.sgp_predict(h, None, 4, None, None) == N.SGP_E_BADARG
    finally:
        e.close()


def test_predict_leaves_open_window_alone(eng):
    c = make_case(130, 5, 2, seed=41)
    rng = np.random.default_rng(2)
    X = rng.random((40000, 5)) * 2.0
    y = np.sin(X.sum(1))

    def window(with_predict):
        eng.set_precision(N.SGP_PREC_AUTO)
        eng.begin(c["k"], c["Z"])
        eng.accumulate(X[:20000], y[:20000])
        if with_predict:
            eng.set_magic(c["v"], c["M"])
            eng.predict(X[:5000])
            predict_dev(eng, X[:5000])
        eng.accumulate(X[20000:], y[20000:])
        return eng.finish()

    G0, b0 = window(False)
    G1, b1 = window(True)
    assert np.array_equal(G0, G1) and np.array_equal(b0, b1)


# ---------------- estimator surface ------------------------------------------------------------------------------------------
def test_estimator_surface_on_cuda_tensors():
    rng = np.random.default_rng(8)
    X = rng.random((600, 3))
    y = np.sin(3 * X.sum(1))
    Z = X[:40]
    gpr = (sg.GaussianProcessRegression().setKernel(lambda: 1.0 * sg.RBFKernel(0.5)).setMaxIter(0)
           .setActiveSetProvider(ExplicitActiveSetProvider(Z)))
    model = gpr.fit(X, y)
    Xt = rng.random((333, 3))
    Xd = torch.from_numpy(Xt).cuda()
    for fn in (model.predict, model.transform):
        out = fn(Xd)
        assert out.is_cuda and np.array_equal(out.cpu().numpy(), fn(Xt))
    one = model.predict(Xd[5])
    assert one.is_cuda and one.item() == model.predict(Xt[5])
    mean, var = model.rawPredictor.predict(Xd)
    m0, v0 = model.rawPredictor.predict(Xt)
    assert mean.is_cuda and var.is_cuda and np.array_equal(mean.cpu().numpy(), m0) and np.array_equal(var.cpu().numpy(), v0)
    m1, v1 = model.rawPredictor.predict(Xd[7])
    assert m1.item() == model.rawPredictor.predict(Xt[7])[0] and v1.item() == model.rawPredictor.predict(Xt[7])[1]
    f32 = model.predict(Xd.float())
    assert np.array_equal(f32.cpu().numpy(), model.predict(Xt.astype(np.float32).astype(np.float64)))

    yc = (y > np.median(y)).astype(np.float64)
    gpc = (sg.GaussianProcessClassifier().setKernel(lambda: 1.0 * sg.RBFKernel(0.5)).setMaxIter(0)
           .setActiveSetProvider(ExplicitActiveSetProvider(Z)))
    cm = gpc.fit(X, yc)
    raw = cm.predictRaw(Xd)
    assert raw.is_cuda and np.array_equal(raw.cpu().numpy(), cm.predictRaw(Xt))
    pred = cm.predict(Xd)
    assert pred.is_cuda and np.array_equal(pred.cpu().numpy(), cm.predict(Xt))
    prob = cm.predictProbability(Xd)
    assert prob.is_cuda and np.allclose(prob.cpu().numpy(), cm.predictProbability(Xt), rtol=1e-14, atol=0)
    assert np.array_equal(cm.predictRaw(Xd[3]).cpu().numpy(), cm.predictRaw(Xt[3]))
