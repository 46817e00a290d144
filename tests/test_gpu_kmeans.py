"""The K-means active-set provider on the GPU (`sgp_kmeans`, csrc/kmeans.cu) against the restatement of Spark 3.1 MLlib
KMeans in oracle/kmeans.py (run on an H100: `pytest -m gpu`).

Bit-for-bit checks use integer data: every fp32 squared distance and every fp64 cost sum is then exact, so both sides
take the same branch on every draw.  Real-valued data are checked on what the fp32 distances guarantee: every label is
within a small fraction of the data's spread of the true nearest centre, and the centres are the fp64 means of the
labels the GPU returned."""
import os

import numpy as np
import pytest

import oracle
from oracle import kmeans as okm
import spark_gp_b200 as sg

pytestmark = pytest.mark.gpu
GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")


@pytest.fixture(scope="module")
def eng():
    e = sg.ProjectedProcessEngine(0)
    yield e
    e.close()


def _int_blobs(d, seed=5, n_blobs=64, per=50):
    rng = np.random.default_rng(seed)
    centres = 1000.0 * rng.choice(np.arange(-40, 41), size=(n_blobs, d))
    while len({tuple(r) for r in centres}) < n_blobs:
        centres = 1000.0 * rng.choice(np.arange(-40, 41), size=(n_blobs, d))
    X = np.concatenate([c + rng.integers(-2, 3, (per, d)) for c in centres]).astype(np.float64)
    return X[rng.permutation(len(X))]


def _true_d2(X, C):
    """fp64 squared distances of every point to every centre (centred expansion form, blocks of points)."""
    o = X.mean(0)
    Xc, Cc = X - o, C - o
    cn = (Cc * Cc).sum(1)
    out = np.empty((len(X), len(C)))
    for s in range(0, len(X), 8192):
        B = Xc[s:s + 8192]
        out[s:s + 8192] = np.maximum((B * B).sum(1)[:, None] - 2.0 * B @ Cc.T + cn[None, :], 0.0)
    return out


def _check_one_pass(X, C0, C, lab, cost, lab_tol=1e-5):
    """max_iter = 1 from C0: labels near-optimal against C0, centres = fp64 means of those labels (empty: C0)."""
    X64 = np.asarray(X, dtype=np.float64)
    D = _true_d2(X64, C0)
    msd = float(((X64 - X64.mean(0)) ** 2).sum(1).mean())
    gap = D[np.arange(len(X64)), lab] - D.min(1)
    assert gap.max() <= lab_tol * msd, "a label is not the nearest centre: gap %.3e x msd" % (gap.max() / msd)
    sums = np.zeros_like(C0)
    np.add.at(sums, lab, X64)
    cnt = np.bincount(lab, minlength=len(C0)).astype(np.float64)
    want = np.where(cnt[:, None] > 0, sums * (1.0 / np.maximum(cnt, 1.0))[:, None], C0)
    scale = max(np.abs(want).max(), 1.0)
    assert np.abs(C - want).max() <= 1e-12 * scale
    cost0 = float(D[np.arange(len(X64)), lab].sum())
    assert abs(cost - cost0) <= 1e-6 * cost0 + 1e-12 * msd * len(X64)


# ---- 1. initialisation, bit for bit ---------------------------------------------------------------------------------
def test_kmeans_parallel_candidates_bit_for_bit(eng):
    rng = np.random.default_rng(11)
    sites = rng.integers(-20, 21, (300, 5)).astype(np.float64)
    X = sites[rng.integers(0, 300, 20000)]
    cand, _ = okm.kmeans_parallel_candidates(X, 1000, 17)
    assert len(cand) <= 300                                           # at most k distinct: the candidates are the result
    C, lab, it, cost = eng.kmeans(X, 1000, max_iter=0, seed=17)
    assert C.shape == cand.shape and np.array_equal(C, cand)
    assert it == 0


@pytest.mark.parametrize("d", [2, 16, 33])
def test_kmeans_integer_blobs_match_oracle(eng, d):
    X = _int_blobs(d)
    k, seed = 64, 3
    C0 = okm.init_centres(X, k, seed)
    _, _, margin = okm.assign(X, C0)
    lab0, best0, _ = okm.assign(X, C0)
    assert np.all(margin > 1e-3 * (best0 + 1.0)), "oracle assignment margin too small for a pinned comparison"
    C, _, it, _ = eng.kmeans(X, k, max_iter=0, seed=seed)
    assert C.shape == C0.shape and np.abs(C - C0).max() <= 1e-12 * np.abs(C0).max()
    Cw, labw, itw, costw = okm.kmeans(X, k, max_iter=20, seed=seed)
    _, bestw, marginw = okm.assign(X, Cw)
    assert np.all(marginw > 1e-3 * (bestw + 1.0))
    C, lab, it, cost = eng.kmeans(X, k, max_iter=20, seed=seed)
    assert C.shape == Cw.shape and np.abs(C - Cw).max() <= 1e-12 * np.abs(Cw).max()
    assert it == itw and np.array_equal(lab, labw)
    assert abs(cost - costw) <= 1e-6 * costw                          # fp32 distances to non-integer means


# ---- 2. Lloyd alone ---------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("offset", [0.0, 1e3, -1e3])
def test_lloyd_one_pass_from_given_centres(eng, offset):
    rng = np.random.default_rng(2)
    X = (rng.random((100_000, 16), dtype=np.float32) + np.float32(offset)).astype(np.float32)
    C0 = X[:1000].astype(np.float64)
    C, lab, it, cost = eng.kmeans(X, 1000, max_iter=1, init_centers=C0)
    assert it == 1 and C.shape == (1000, 16)
    _check_one_pass(X, C0, C, lab, cost)


# ---- 3. rules ---------------------------------------------------------------------------------------------------------
def test_empty_cluster_keeps_its_centre_and_stopping_rules(eng):
    rng = np.random.default_rng(4)
    X = rng.random((5000, 4))
    C0 = X[:20].copy()
    C0[7] = 1e6 + np.arange(4)
    C, lab, it, _ = eng.kmeans(X, 20, max_iter=5, init_centers=C0)
    assert np.array_equal(C[7], C0[7]) and not np.any(lab == 7)
    _, _, it, _ = eng.kmeans(X, 20, max_iter=50, tol=1e9, init_centers=C0)
    assert it == 1
    C, lab, it, cost = eng.kmeans(X, 20, max_iter=0, init_centers=C0)
    assert it == 0 and np.array_equal(C, C0)
    labo, besto, _ = okm.assign(X, C0)
    assert np.array_equal(lab, labo) and abs(cost - besto.sum()) <= 1e-6 * besto.sum()


# ---- 4. edges ---------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("d", [1, 3, 16, 17, 32, 33, 100, 784])
def test_edges_in_d(eng, d):
    if d == 784:
        c = np.load(os.path.join(GOLD, "mnist68_case.npz"))
        n = int(c["n_rows"])
        X = ((c["pixels"].astype(np.float64) - c["mean"]) / c["std"])[:n]
    else:
        X = np.random.default_rng(d).standard_normal((3000, d)) * 3.0 + 7.0
    k = 100
    C0 = X[:k].copy()
    C, lab, it, cost = eng.kmeans(X, k, max_iter=1, init_centers=C0)
    _check_one_pass(X, C0, C, lab, cost)
    Ck, labk, itk, costk = eng.kmeans(X, k, max_iter=3, seed=1)
    assert Ck.shape == (k, d) and np.all(np.isfinite(Ck)) and labk.max() < k and 1 <= itk <= 3


@pytest.mark.parametrize("k", [2, 127, 128, 129, 1000, 4000])
def test_edges_in_k(eng, k):
    X = np.random.default_rng(k).random((20000, 8))
    C0 = X[:k].copy()
    C, lab, it, cost = eng.kmeans(X, k, max_iter=1, init_centers=C0)
    _check_one_pass(X, C0, C, lab, cost)
    Ck, labk, _, _ = eng.kmeans(X, k, max_iter=2, seed=k)
    assert Ck.shape == (k, 8) and np.all(np.isfinite(Ck)) and 0 <= labk.min() and labk.max() < k


@pytest.mark.parametrize("which", ["1", "2", "k-1", "k", "k+1", "131073"])
def test_edges_in_n(eng, which):
    k = 128
    n = {"1": 1, "2": 2, "k-1": k - 1, "k": k, "k+1": k + 1, "131073": 131073}[which]
    X = np.random.default_rng(n).random((n, 4))
    C, lab, it, cost = eng.kmeans(X, k, max_iter=10, seed=2)
    assert 1 <= len(C) <= min(k, n) and np.all(np.isfinite(C)) and len(lab) == n and lab.max() < len(C)
    if n <= k:
        assert len({tuple(r) for r in C}) == len(C)
    if n >= k:
        C0 = X[:k].copy()
        C1, lab1, _, cost1 = eng.kmeans(X, k, max_iter=1, init_centers=C0)
        _check_one_pass(X, C0, C1, lab1, cost1)


def test_identical_points_and_precision_forms(eng):
    X = np.tile(np.array([[0.3, -1.25, 7.0]]), (1000, 1))
    C, lab, it, cost = eng.kmeans(X, 10, seed=1)
    assert C.shape == (1, 3) and np.allclose(C[0], X[0], rtol=1e-12, atol=0) and np.all(lab == 0) and cost <= 1e-20
    X32 = np.random.default_rng(0).random((30000, 6), dtype=np.float32)
    a = eng.kmeans(X32, 200, max_iter=5, seed=4)
    b = eng.kmeans(X32.astype(np.float64), 200, max_iter=5, seed=4)
    assert np.array_equal(a[0], b[0]) and np.array_equal(a[1], b[1]) and a[2] == b[2] and a[3] == b[3]


# ---- 5. determinism and isolation -----------------------------------------------------------------------------------
def test_deterministic_and_leaves_an_open_window_untouched(eng):
    rng = np.random.default_rng(6)
    X = rng.random((60000, 10), dtype=np.float32)
    a = eng.kmeans(X, 500, max_iter=10, seed=8)
    b = eng.kmeans(X, 500, max_iter=10, seed=8)
    assert np.array_equal(a[0], b[0]) and np.array_equal(a[1], b[1]) and a[3] == b[3] and a[2] == b[2]
    d = 10
    kernel = 1 * sg.ARDRBFKernel(np.full(d, 0.8)) + sg.const(1e-2) * sg.EyeKernel()
    Z = X[:64].astype(np.float64)
    y = np.sin(X.astype(np.float64).sum(1))

    def window(with_kmeans):
        eng.begin(kernel, Z)
        eng.accumulate(X[:40000], y[:40000])
        if with_kmeans:
            eng.kmeans(X, 300, max_iter=3, seed=1)
        eng.accumulate(X[40000:], y[40000:])
        path = eng.last_path()
        G, bb = eng.finish()
        return G, bb, path

    G0, b0, p0 = window(False)
    G1, b1, p1 = window(True)
    assert np.array_equal(G0, G1) and np.array_equal(b0, b1) and p0 == p1


# ---- 6. bad arguments -------------------------------------------------------------------------------------------------
def test_bad_arguments_raise_and_the_context_survives(eng):
    X = np.random.default_rng(0).random((100, 3))
    for kw in [dict(k=1), dict(k=0), dict(max_iter=-1), dict(tol=-1e-3), dict(tol=float("nan"))]:
        args = dict(k=4)
        args.update(kw)
        with pytest.raises(ValueError):
            eng.kmeans(X, **args)
    with pytest.raises(ValueError):
        eng.kmeans(np.zeros((0, 3)), 4)
    with pytest.raises(ValueError):
        eng.kmeans(np.zeros((10, 0)), 4)
    for bad in (np.nan, np.inf):
        Xb = X.copy()
        Xb[57, 1] = bad
        with pytest.raises(ValueError):
            eng.kmeans(Xb, 4)
        with pytest.raises(ValueError):
            eng.kmeans(Xb.astype(np.float32), 4)
    C, lab, it, cost = eng.kmeans(X, 4, max_iter=1, init_centers=X[:4])
    _check_one_pass(X, X[:4], C, lab, cost)


# ---- 7. provider ------------------------------------------------------------------------------------------------------
def test_provider_on_gpu_recovers_blobs():
    rng = np.random.default_rng(0)
    centres = rng.random((5, 3)) * 10
    X = np.concatenate([c + 0.05 * rng.standard_normal((40, 3)) for c in centres])
    prov = sg.KMeansActiveSetProvider(maxIter=20, on_gpu=True)
    A = prov(5, X, None, None, None, 13)
    assert A.shape == (5, 3) and A.dtype == np.float64 and A.flags["C_CONTIGUOUS"]
    assert np.array_equal(A, prov(5, X, None, None, None, 13))
    d = np.linalg.norm(A[:, None, :] - centres[None, :, :], axis=2)
    assert np.all(d.min(axis=0) < 0.05)


def test_provider_on_gpu_in_fit_matches_projected_process():
    c = np.load(os.path.join(GOLD, "airfoil_case.npz"))
    sigma2, theta = float(c["sigma2"]), c["theta"]
    X, y = c["X"], c["y"]
    gp = (sg.GaussianProcessRegression().setKernel(lambda: 1 * sg.ARDRBFKernel(5) + sg.const(1) * sg.EyeKernel())
          .setSigma2(sigma2).setDatasetSizeForExpert(100).setActiveSetSize(1000).setMaxIter(0).setSeed(7)
          .setActiveSetProvider(sg.KMeansActiveSetProvider(maxIter=20, on_gpu=True)))
    active = gp._activeSetProvider(1000, X, y, gp.getKernel, theta, 7, gp=gp)
    model = gp.fit(X, y, hyperparameters=theta)
    ofac = oracle.get_kernel(lambda: 1 * oracle.ARDRBFKernel(5) + oracle.const(1) * oracle.EyeKernel(), sigma2)
    experts = oracle.get_expert_labels_and_kernels(X, y, ofac, 100)
    pred, _, _ = oracle.projected_process(experts, active, ofac, theta)
    m0, _ = pred.predict_many(c["Xtest"])
    assert np.abs(model.predict(c["Xtest"]) - m0).max() / np.abs(m0).max() <= 1e-5


def test_provider_cost_against_scikit_learn(eng):
    from sklearn.cluster import KMeans
    rng = np.random.default_rng(9)
    X = rng.random((200_000, 16), dtype=np.float32)
    _, _, _, cost = eng.kmeans(X, 1000, max_iter=20, seed=0)
    km = KMeans(n_clusters=1000, init="k-means++", n_init=1, max_iter=20, tol=1e-4, random_state=0, algorithm="lloyd")
    km.fit(X.astype(np.float64))
    print("k-means cost at 200k x 16, k = 1000: GPU %.6e, scikit-learn %.6e (ratio %.4f)" % (cost, km.inertia_,
                                                                                          cost / km.inertia_))
    assert cost <= 1.10 * km.inertia_
