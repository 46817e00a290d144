"""CPU checks of the K-means restatement (oracle/kmeans.py) that the GPU K-means is pinned on: its Lloyd iterations against
an independent implementation (scikit-learn), and the invariants of its k-means|| initialisation."""
import numpy as np
import pytest

from oracle import kmeans as okm


def _blobs(rng, n_blobs, per, d, spread):
    centres = rng.random((n_blobs, d)) * 100.0
    X = np.concatenate([c + spread * rng.standard_normal((per, d)) for c in centres])
    return X, centres


def test_generator_scalar_and_vector_forms_agree():
    idx = np.array([0, 1, 2, 12345, 2 ** 31 - 1], dtype=np.int64)
    vec = okm.u(7, 1, idx)
    assert np.array_equal(vec, [okm.u(7, 1, int(i)) for i in idx])
    assert np.all((vec >= 0.0) & (vec < 1.0))
    assert okm.u(7, 1, 3) != okm.u(7, 2, 3) and okm.u(7, 1, 3) != okm.u(8, 1, 3)
    assert okm.u(-1, 0, 0) == okm.u(2 ** 64 - 1, 0, 0)               # the seed is taken modulo 2^64


@pytest.mark.parametrize("d", [2, 7])
def test_lloyd_matches_scikit_learn(d):
    """From given centres on well-separated blobs (no empty cluster) with tol = 0, the restated Lloyd iterations end where
    scikit-learn's Lloyd ends."""
    from sklearn.cluster import KMeans
    rng = np.random.default_rng(3 + d)
    X, _ = _blobs(rng, 6, 60, d, 4.0)
    C0 = X[rng.choice(len(X), 6, replace=False)]
    C, lab, it, cost = okm.lloyd(X, C0, 100, 0.0)
    km = KMeans(n_clusters=6, init=C0, n_init=1, algorithm="lloyd", tol=0.0, max_iter=100).fit(X)
    assert np.bincount(lab, minlength=6).min() > 0
    assert np.abs(C - km.cluster_centers_).max() <= 1e-12 * np.abs(C).max()
    assert np.array_equal(lab, km.labels_)
    assert abs(cost - km.inertia_) <= 1e-9 * cost
    assert 1 <= it < 100


def test_at_most_k_distinct_points_are_the_result():
    rng = np.random.default_rng(1)
    sites = rng.integers(-5, 6, (7, 3)).astype(np.float64)
    X = sites[rng.integers(0, 7, 500)]
    cand, chosen = okm.kmeans_parallel_candidates(X, 10, 5)
    C = okm.init_centres(X, 10, 5)
    assert np.array_equal(C, cand) and len(C) <= 7
    assert len({tuple(r) for r in C}) == len(C)
    first = [X[i] for i in chosen]
    keep = []
    for r in first:                                                   # first occurrence order
        if not any(np.array_equal(r, q) for q in keep):
            keep.append(r)
    assert np.array_equal(np.array(keep), C)


def test_identical_points_give_one_centre():
    X = np.tile([[1.5, -2.0, 3.25]], (50, 1))
    C, lab, it, cost = okm.kmeans(X, 4, max_iter=5, seed=9)
    assert C.shape == (1, 3) and np.array_equal(C[0], X[0])
    assert np.all(lab == 0) and cost == 0.0 and it == 1


def test_zero_weights_are_never_drawn():
    rng = np.random.default_rng(2)
    cand = rng.random((40, 3))
    w = rng.integers(1, 5, 40).astype(np.float64)
    zero = rng.choice(40, 15, replace=False)
    w[zero] = 0.0
    for seed in range(20):
        C = okm.local_kmeans_pp(cand, w, 8, seed, max_iterations=0)
        picked = [int(np.nonzero((cand == c).all(1))[0][0]) for c in C]
        assert not set(picked) & set(zero.tolist())


def test_full_run_on_blobs_recovers_the_centres():
    rng = np.random.default_rng(4)
    X, centres = _blobs(rng, 5, 40, 3, 0.05)
    C, lab, it, cost = okm.kmeans(X, 5, max_iter=20, seed=13)
    d = np.linalg.norm(C[:, None, :] - centres[None, :, :], axis=2)
    assert C.shape == (5, 3) and np.all(d.min(axis=0) < 0.05)
    C2 = okm.kmeans(X, 5, max_iter=20, seed=13)[0]
    assert np.array_equal(C, C2)
