"""The averaged probability on the GPU (`sgp_predict_probability`, `sgp_predict_probability_device`, the classifiers'
`predictAveragedProbability`; run on an H100: `pytest -m gpu`).

p = (1/sqrt(pi)) sum_i w_i sigmoid(mean + sqrt(2 max(var, 0)) x_i) with the n-node Gauss-Hermite rule.  The mean and
variance the probability entries return must be `sgp_predict`'s, bit for bit, and p must be within 3e-14 of the oracle's
rule (`oracle.integrator.averaged_probability`, numpy's hermgauss) applied to that same (mean, var): n_nodes x eps at 256
nodes, the two sides differing only in exp ulps, the rules' last bits and the summation order.  A magic pair is
installed with `sgp_set_magic`, as in test_gpu_predict.py (whose case builder this file reuses), over the same edges: m
at the 64/128 tile edges, d at the 32-dim staging edges, 1-4 non-Eye terms, n at the CTA and window edges.  Its random
M gives large variances of either sign, case by case; the rule-size cases shift M so that the variances straddle 0."""
import ctypes as C
import os

import numpy as np
import pytest
import torch

import oracle
import spark_gp_b200 as sg
from oracle.integrator import averaged_probability
from spark_gp_b200 import _native as N
from spark_gp_b200.regression import ExplicitActiveSetProvider
from test_gpu_predict import install, make_case, points

pytestmark = pytest.mark.gpu

TOL_P = 3e-14
GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
NODES = [1, 2, 100, 256]


@pytest.fixture(scope="module")
def eng():
    e = sg.ProjectedProcessEngine(0)
    yield e
    e.close()


def bits(a):
    return np.ascontiguousarray(a, dtype=np.float64).view(np.uint64)


def same(a, b):
    return np.array_equal(bits(a), bits(b))


def prob_dev(eng, X, nodes, with_mv=True, f32=False):
    Xd = torch.from_numpy(np.ascontiguousarray(X, dtype=np.float32 if f32 else np.float64)).cuda()
    p, m, v = eng.predict_probability_tensor(Xd, nodes=nodes, with_mean_var=with_mv)
    host = lambda t: t.cpu().numpy() if t is not None else None
    return host(p), host(m), host(v)


def check(eng, X, nodes, device=True):
    """Both probability entries against sgp_predict and the oracle rule; returns p."""
    hm, hv = eng.predict(X)
    p, m, v = eng.predict_probability(X, nodes, with_mean_var=True)
    assert same(m, hm) and same(v, hv)
    assert not np.isnan(p).any()
    err = np.abs(p - averaged_probability(hm, hv, nodes)).max()
    assert err < TOL_P, err
    if device:
        dp, dm, dv = prob_dev(eng, X, nodes)
        assert same(dp, p) and same(dm, hm) and same(dv, hv)
    return p


# ---------------- parity over the prediction edges ----------------------------------------------------------------------
@pytest.mark.parametrize("m", [1, 63, 64, 65, 127, 128, 129, 1000])
def test_parity_m(eng, m):
    c = make_case(m, 5, 2, seed=m)
    install(eng, c)
    X = points(c, 300)
    check(eng, X, NODES[m % 4])


@pytest.mark.parametrize("d", [1, 16, 33, 784])
@pytest.mark.parametrize("f32", [False, True], ids=["f64", "f32"])
def test_parity_d(eng, d, f32):
    c = make_case(129, d, 1 + d % 4, seed=d)
    install(eng, c)
    X = points(c, 200)
    if f32:
        X = X.astype(np.float32).astype(np.float64)
    p = check(eng, X, 100)
    fp, _, _ = prob_dev(eng, X, 100, f32=f32)
    assert same(fp, p)


@pytest.mark.parametrize("n_terms", [1, 2, 3, 4])
def test_parity_terms(eng, n_terms):
    c = make_case(200, 7, n_terms, seed=10 + n_terms)
    install(eng, c)
    check(eng, points(c, 150), 100)


@pytest.mark.parametrize("nodes", NODES)
def test_parity_nodes(eng, nodes):
    c = make_case(300, 6, 2, seed=50 + nodes)
    X = points(c, 1000)
    # M + a 1 1^T adds a (sum_j k_j)^2 to the variance: pick a so that the variances straddle 0
    K0 = c["k0"].cross_kernel(X)
    s2 = K0.sum(1) ** 2
    a = -np.median(np.einsum("ti,ti->t", K0 @ c["M"], K0) / s2)
    install(eng, c, M=c["M"] + a)
    check(eng, X, nodes)
    _, v = eng.predict(X)
    assert (v < 0).sum() > 100 and (v > 0).sum() > 100          # both sides of the clamp


# n at the CTA edges, and around the host entry's staging window (d = 784: 5350 points per chunk)
@pytest.mark.parametrize("n,d", [(1, 5), (63, 5), (64, 5), (65, 5), (5350, 784), (5351, 784)])
def test_parity_n(eng, n, d):
    c = make_case(65, d, 2, seed=n)
    install(eng, c)
    check(eng, points(c, n), 100)


def test_device_window_edge(eng):
    """m = 4000 pads to 4096 columns: the device entry's kernel window is 8192 points."""
    c = make_case(4000, 8, 1, seed=4)
    install(eng, c)
    check(eng, points(c, 8193), 100)


# ---------------- bit identity and launches -----------------------------------------------------------------------------
def test_bit_identity(eng):
    c = make_case(257, 16, 2, seed=9)
    install(eng, c)
    X32 = points(c, 3001).astype(np.float32)
    X = X32.astype(np.float64)
    p, m, v = eng.predict_probability(X, 100, with_mean_var=True)
    assert same(eng.predict_probability(X, 100)[0], p)                                # without mean / var
    dp, dm, dv = prob_dev(eng, X, 100)
    assert same(dp, p) and same(dm, m) and same(dv, v)
    assert same(prob_dev(eng, X, 100, with_mv=False)[0], p)                          # mean in the workspace
    fp, fm, fv = prob_dev(eng, X32, 100, f32=True)
    assert same(fp, p) and same(fm, m) and same(fv, v)
    a, _, _ = eng.predict_probability(X[:1234], 100)
    b, _, _ = eng.predict_probability(X[1234:], 100)
    assert same(np.concatenate([a, b]), p)
    p2, _, _ = eng.predict_probability(X, 2)                   # another rule size, then back
    assert not same(p2, p) and same(eng.predict_probability(X, 100)[0], p)
    hm, hv = eng.predict(X)
    assert same(hm, m) and same(hv, v)


def test_launch_count(eng):
    c = make_case(1000, 784, 2, seed=12)
    X = points(c, 40000)                                       # 8 host windows of 5350 points, 2 device windows
    counts = {}
    for what in ("predict", "probability"):
        install(eng, c)                                        # a fresh pair: the first variance call packs it
        l0 = eng.launch_count()
        if what == "predict":
            eng.predict(X)
        else:
            eng.predict_probability(X, 100)
        l1 = eng.launch_count()
        if what == "predict":
            eng.predict(X)
            eng.predict_tensor(torch.from_numpy(X).cuda())
        else:
            eng.predict_probability(X, 100)
            prob_dev(eng, X, 100, with_mv=False)
        counts[what] = (l1 - l0, eng.launch_count() - l1)
    assert counts["predict"] == counts["probability"], counts
    assert counts["probability"] == (3 * 8 + 1, 3 * 8 + 3 * 2), counts


def test_negative_variance_gives_sigmoid_of_mean(eng):
    c = make_case(120, 4, 1, seed=61)
    Mneg = -1e3 * np.eye(c["m"])                               # var = selfKernel - 1000 |k|^2 < 0 near the active set
    install(eng, c, M=Mneg)
    X = np.concatenate([c["Z"][:40] + 1e-3, points(c, 200)])
    for nodes in NODES:
        p, m, v = eng.predict_probability(X, nodes, with_mean_var=True)
        assert (v < 0).sum() >= 40 and not np.isnan(p).any()
        wsum = np.polynomial.hermite.hermgauss(nodes)[1].sum() / np.sqrt(np.pi)
        neg = v < 0
        assert np.abs(p[neg] - wsum / (1.0 + np.exp(-m[neg]))).max() < TOL_P
        assert np.abs(p - averaged_probability(m, v, nodes)).max() < TOL_P


def test_nan_propagates(eng):
    c = make_case(70, 3, 1, seed=62)
    install(eng, c)
    X = points(c, 10)
    X[3, 1] = np.nan
    p, m, v = eng.predict_probability(X, 100, with_mean_var=True)
    assert np.isnan(m[3]) and np.isnan(p[3]) and not np.isnan(np.delete(p, 3)).any()


# ---------------- refusals ------------------------------------------------------------------------------------------------
def test_state_and_arguments():
    e = sg.ProjectedProcessEngine(0)
    try:
        lib, h = e._lib, e._h
        X = np.zeros((4, 3))
        p = np.zeros(4)
        Xd = torch.zeros((4, 3), dtype=torch.float64, device="cuda")
        pd = torch.zeros(4, dtype=torch.float64, device="cuda")
        dev = lambda t: C.c_void_p(t.data_ptr())
        assert lib.sgp_predict_probability(h, N.ptr(X), 4, 100, N.ptr(p), None, None) == N.SGP_E_STATE
        assert lib.sgp_predict_probability_device(h, dev(Xd), 0, 4, 100, dev(pd), None, None) == N.SGP_E_STATE
        c = make_case(10, 3, 1)
        e.begin(c["k"], c["Z"])
        assert lib.sgp_predict_probability(h, N.ptr(X), 4, 100, N.ptr(p), None, None) == N.SGP_E_STATE
        e.set_magic(c["v"], c["M"])
        l0 = e.launch_count()
        for nodes in (0, -1, 257):
            assert lib.sgp_predict_probability(h, N.ptr(X), 4, nodes, N.ptr(p), None, None) == N.SGP_E_BADARG
            assert lib.sgp_predict_probability_device(h, dev(Xd), 0, 4, nodes, dev(pd), None, None) == N.SGP_E_BADARG
        assert lib.sgp_predict_probability(h, None, 4, 100, N.ptr(p), None, None) == N.SGP_E_BADARG
        assert lib.sgp_predict_probability(h, N.ptr(X), 4, 100, None, N.ptr(p), None) == N.SGP_E_BADARG
        assert lib.sgp_predict_probability(h, N.ptr(X), -1, 100, N.ptr(p), None, None) == N.SGP_E_BADARG
        assert lib.sgp_predict_probability_device(h, None, 0, 4, 100, dev(pd), None, None) == N.SGP_E_BADARG
        assert lib.sgp_predict_probability_device(h, dev(Xd), 0, 4, 100, None, None, None) == N.SGP_E_BADARG
        assert lib.sgp_predict_probability_device(h, dev(Xd), 0, -1, 100, dev(pd), None, None) == N.SGP_E_BADARG
        # host memory where device memory is expected: refused before any launch
        assert lib.sgp_predict_probability_device(h, N.ptr(X), 0, 4, 100, dev(pd), None, None) == N.SGP_E_BADARG
        assert lib.sgp_predict_probability_device(h, dev(Xd), 0, 4, 100, N.ptr(p), None, None) == N.SGP_E_BADARG
        assert lib.sgp_predict_probability_device(h, dev(Xd), 0, 4, 100, dev(pd), N.ptr(p), None) == N.SGP_E_BADARG
        assert lib.sgp_predict_probability_device(h, dev(Xd), 0, 4, 100, dev(pd), None, N.ptr(p)) == N.SGP_E_BADARG
        assert b"not device memory" in lib.sgp_last_error(h)
        assert lib.sgp_predict_probability(h, None, 0, 100, None, None, None) == N.SGP_OK
        assert lib.sgp_predict_probability_device(h, None, 0, 0, 100, None, None, None) == N.SGP_OK
        assert e.launch_count() == l0
        with pytest.raises(ValueError):
            e.predict_probability(X, 0)
    finally:
        e.close()


# ---------------- fitted models -------------------------------------------------------------------------------------------
def oracle_pair(model, kernel_o):
    """The oracle predictor's (mean, var) for the model's own magic pair, kernel and active set."""
    rp = model.rawPredictor
    k0 = kernel_o.set_hyperparameters(model.hyperparameters).set_training_vectors(np.asarray(rp.activeSet))
    return oracle.GaussianProjectedProcessRawPredictor(rp.magicVector, rp.magicMatrix, k0)


def check_model(model, kernel_o, Xte, nodes=100):
    P = model.predictAveragedProbability(Xte, nodes)
    assert P.shape == (len(Xte), 2)
    mean, var = model.rawPredictor.predict(Xte)
    assert same(P[:, 0], 1.0 - P[:, 1])
    assert np.abs(P[:, 1] - averaged_probability(mean, var, nodes)).max() < TOL_P
    m0, v0 = oracle_pair(model, kernel_o).predict_many(Xte)
    err = np.abs(P[:, 1] - averaged_probability(m0, v0, nodes)).max()
    print("p vs the oracle predictor's (mean, var): %.1e" % err)
    assert err < 1e-10
    Pd = model.predictAveragedProbability(torch.from_numpy(Xte).cuda(), nodes)
    assert Pd.is_cuda and Pd.dtype == torch.float64 and same(Pd.cpu().numpy(), P)
    one = model.predictAveragedProbability(Xte[3], nodes)
    assert one.shape == (1, 2) and same(one, P[3:4])
    # the existing outputs are what they were: predictRaw from the mean-only call, the quirky probability on it
    raw = model.predictRaw(Xte)
    f, _ = model.rawPredictor._engine.predict(Xte, with_variance=False)
    assert same(raw[:, 1], f) and same(raw[:, 0], -f)
    p0 = 1.0 / (1.0 + np.exp(raw[..., 0]))
    assert same(model.predictProbability(Xte), np.stack([p0, 1.0 - p0], axis=-1))
    assert same(model.predict(Xte), np.argmax(raw, axis=-1).astype(np.float64))
    return P


def test_mnist68_binary_model():
    c = np.load(os.path.join(GOLD, "mnist68_case.npz"))
    n = int(c["n_rows"])
    X = (c["pixels"].astype(np.float64) - c["mean"]) / c["std"]
    Xtr, Xte, ytr = X[:n], X[n:n + 100], c["y01"][:n]
    sigma = float(c["sigma"])
    gp = (sg.GaussianProcessClassifier().setDatasetSizeForExpert(100).setActiveSetSize(500)
          .setKernel(lambda: sg.RBFKernel(sigma)).setTol(1e-3)
          .setActiveSetProvider(ExplicitActiveSetProvider(Xtr[c["active_idx"]])))
    model = gp.fit(Xtr, ytr, hyperparameters=np.array([sigma]))
    P = check_model(model, oracle.RBFKernel(sigma) + oracle.const(1e-3) * oracle.EyeKernel(), Xte)
    assert np.mean((P[:, 1] > 0.5) == (c["y01"][n:n + 100] == 1)) > 0.95
    for nodes in NODES:
        check_model(model, oracle.RBFKernel(sigma) + oracle.const(1e-3) * oracle.EyeKernel(), Xte[:20], nodes)


def test_iris_one_vs_rest_model():
    c = np.load(os.path.join(GOLD, "iris_case.npz"))
    tr, te = c["train_idx"], c["test_idx"]
    Xtr, ytr, Xte = c["X"][tr], c["y"][tr], c["X"][te]
    gp = (sg.GaussianProcessClassifier().setDatasetSizeForExpert(20).setActiveSetSize(30)
          .setActiveSetProvider(ExplicitActiveSetProvider(Xtr[c["active_idx"]])))
    model = sg.OneVsRest().setClassifier(gp).fit(Xtr, ytr, hyperparameters=c["thetas"])
    P = model.predictAveragedProbability(Xte)
    assert P.shape == (len(Xte), model.numClasses)
    for k, mk in enumerate(model.models):
        Pk = check_model(mk, oracle.RBFKernel() + oracle.const(1e-3) * oracle.EyeKernel(), Xte)
        assert same(P[:, k], Pk[:, 1])
    Pd = model.predictAveragedProbability(torch.from_numpy(Xte).cuda())
    assert Pd.is_cuda and same(Pd.cpu().numpy(), P)
    assert model.predictAveragedProbability(Xte[0]).shape == (1, model.numClasses)
    assert np.mean(np.argmax(P, axis=1) == c["y"][te]) > 0.8
