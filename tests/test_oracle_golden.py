"""Pins the oracle on every known-answer vector the reference's own tests hold
(`/root/reference/src/test/scala/org/apache/spark/ml/commons/kernel/*.scala`) and on the derived
smoke values of SURVEY.md section 8(c)."""
import numpy as np
import pytest

import oracle
from oracle import (ARDRBFKernel, RBFKernel, EyeKernel, Scalar, const, WhiteNoiseKernel,
                    TrainingVectorsNotInitializedException)

DATASET = np.array([[1.0, 2.0], [2.0, 3.0], [5.0, 7.0]])


def test_rbf_not_initialised_training_kernel():            # RBFKernelTest.scala:9-16
    with pytest.raises(TrainingVectorsNotInitializedException):
        RBFKernel().training_kernel()


def test_rbf_not_initialised_derivative():                 # RBFKernelTest.scala:18-25
    with pytest.raises(TrainingVectorsNotInitializedException):
        RBFKernel().training_kernel_and_derivative()


def test_rbf_training_kernel_golden():                     # RBFKernelTest.scala:29-39
    rbf = RBFKernel(np.sqrt(0.2)).set_training_vectors(DATASET)
    correct = np.array([[1.000000e+00, 6.737947e-03, 3.053624e-45],
                        [6.737947e-03, 1.000000e+00, 7.187782e-28],
                        [3.053624e-45, 7.187782e-28, 1.000000e+00]])
    K = rbf.training_kernel()
    assert np.all(np.abs(K - correct) < 1e-4)              # the reference's own tolerance
    assert np.allclose(K, correct, rtol=1e-6, atol=0)      # and to the 7 printed digits


def _rbf_numeric_derivative(sigma, h):
    l = RBFKernel(sigma - h).set_training_vectors(DATASET)
    r = RBFKernel(sigma + h).set_training_vectors(DATASET)
    return (r.training_kernel() - l.training_kernel()) / (2 * h)


def test_rbf_derivative_vs_numeric():                      # RBFKernelTest.scala:51-60
    rbf = RBFKernel(0.2).set_training_vectors(DATASET)
    analytical = rbf.training_kernel_and_derivative()[1][0]
    assert np.all(np.abs(analytical - _rbf_numeric_derivative(0.2, 1e-3)) < 1e-3)


def test_rbf_cross_kernel_golden():                        # RBFKernelTest.scala:62-68
    rbf = RBFKernel(np.sqrt(0.2)).set_training_vectors(DATASET[1:])
    ck = rbf.cross_kernel(DATASET[:1])
    assert ck.shape == (1, 2)                              # test.length x train.length
    correct = np.array([[6.737947e-03, 3.053624e-45]])
    assert np.all(np.abs(ck - correct) < 1e-4)
    assert np.allclose(ck, correct, rtol=1e-6, atol=0)


def test_rbf_cross_kernel_single_vector_golden():          # RBFKernelTest.scala:70-76
    rbf = RBFKernel(np.sqrt(0.2)).set_training_vectors(DATASET[1:])
    ck = rbf.cross_kernel_vec(DATASET[0])
    assert ck.shape == (2,)
    assert np.allclose(ck, [6.737947e-03, 3.053624e-45], rtol=1e-6, atol=0)


def test_ard_derivative_vs_numeric():                      # ARDRBFKernelTest.scala:11-31
    beta = np.array([0.2, 0.3])
    ard = ARDRBFKernel(beta).set_training_vectors(DATASET)
    analytical = sum(ard.training_kernel_and_derivative()[1])
    h = 1e-3
    l = ARDRBFKernel(beta - h).set_training_vectors(DATASET)
    r = ARDRBFKernel(beta + h).set_training_vectors(DATASET)
    numeric = (r.training_kernel() - l.training_kernel()) / (2 * h)
    assert np.all(np.abs(analytical - numeric) < 1e-3)


# ---- derived smoke values (SURVEY.md 8(c); computed from the formulas, NOT from reference tests) ----

def test_ard_smoke_values():
    ard = ARDRBFKernel(np.array([0.2, 0.3])).set_training_vectors(DATASET)
    K = ard.training_kernel()
    assert np.isclose(K[0, 1], 0.878095430921, rtol=1e-11)
    assert np.isclose(K[0, 2], 0.055576212611, rtol=1e-10)
    assert np.isclose(K[1, 2], 0.165298888222, rtol=1e-11)
    d = sum(ard.training_kernel_and_derivative()[1])
    assert np.isclose(d[0, 1], -0.878095430921, rtol=1e-10)
    assert np.isclose(d[0, 2], -1.189330949886, rtol=1e-10)
    assert np.isclose(d[1, 2], -2.181945324525, rtol=1e-10)


def _smoke_setup():
    user = lambda: 1 * ARDRBFKernel(np.array([0.2, 0.3])) + const(1) * EyeKernel()
    factory = oracle.get_kernel(user, 1e-4)
    y = np.array([0.5, -1.0, 2.0])
    Z = DATASET[[0, 2]]
    return factory, y, Z


def test_projected_process_smoke_values():
    factory, y, Z = _smoke_setup()
    k = factory()
    assert np.isclose(k.white_noise_var, 1.0001)
    theta = k.get_hyperparameters()
    assert np.allclose(theta, [1.0, 0.2, 0.3])            # C prepended, Eye/const add none
    experts = [(y, factory().set_training_vectors(DATASET))]
    pred, G, b = oracle.projected_process(experts, Z, factory, theta)
    assert np.allclose(G, [[1.774140301212, 0.256300623707], [0.256300623707, 1.030412437856]], rtol=1e-11)
    assert np.allclose(b, [-0.266943005698, 1.862489218084], rtol=1e-11)
    assert np.allclose(pred.magic_vector, [-0.122545269186, 0.627149214156], rtol=1e-10)
    assert np.allclose(pred.magic_matrix, [[-0.233122498440, -0.013597424403],
                                           [-0.013597424403, -0.167542879982]], rtol=1e-10)
    mean, var = pred.predict(np.array([3.0, 4.0]))
    assert np.isclose(mean, 0.164885948858, rtol=1e-10)
    assert np.isclose(var, 1.887496212554, rtol=1e-10)
    m2, v2 = pred.predict_many(np.array([[3.0, 4.0]]))
    assert np.isclose(m2[0], mean, rtol=1e-14) and np.isclose(v2[0], var, rtol=1e-14)


def test_regression_nll_smoke_values():
    factory, y, _ = _smoke_setup()
    k = factory().set_training_vectors(DATASET)
    nll, grad = oracle.regression_likelihood_and_gradient(y, k, np.array([1.0, 0.2, 0.3]))
    assert np.isclose(nll, 2.554558544113, rtol=1e-11)
    assert np.allclose(grad, [0.091179101215, -0.365504180268, -0.951631586041], rtol=1e-9)


def test_hyperparameter_layout_and_bounds():
    k = Scalar(1.0).between(0).and_(30) * RBFKernel(0.1, 1e-6, 10) + WhiteNoiseKernel(0.5, 0, 1)
    assert np.allclose(k.get_hyperparameters(), [1.0, 0.1, 0.5])
    lo, up = k.hyperparameter_boundaries()
    assert np.allclose(lo, [0, 1e-6, 0]) and np.allclose(up, [30, 10, 1])
    k.set_hyperparameters([2.0, 0.3, 0.25])
    assert np.allclose(k.get_hyperparameters(), [2.0, 0.3, 0.25])
    assert np.isclose(k.white_noise_var, 0.25)
    with pytest.raises(ValueError):
        Scalar(-1.0) * RBFKernel()                         # require(C >= 0)  ScalarTimesKernel.scala:7


def test_eye_cross_kernel_is_zero_and_sum_semantics():
    X = np.random.default_rng(0).random((7, 3))
    Z = X[:4]
    k = (2.0 * ARDRBFKernel(3) + const(1) * EyeKernel() + const(1e-3) * EyeKernel()).set_training_vectors(X)
    ck = k.cross_kernel(Z)
    assert ck.shape == (4, 7)
    assert np.allclose(ck, 2.0 * ARDRBFKernel(3).set_training_vectors(X).cross_kernel(Z))
    assert np.isclose(ck[0, 0], 2.0)                       # Eye adds NOTHING to the cross kernel, even at x==z
    tk = k.training_kernel()
    assert np.isclose(tk[0, 0], 2.0 + 1.0 + 1e-3)          # ...but sits on the training-kernel diagonal
    assert np.isclose(k.self_kernel(X[0]), 3.001)


def test_group_for_experts():
    groups = oracle.group_for_experts(1503, 100)
    assert len(groups) == 15
    assert sorted(len(g) for g in groups) == [100] * 12 + [101] * 3
    assert np.array_equal(groups[3][:3], [3, 18, 33])
    assert len(oracle.group_for_experts(150, 100)) == 2    # Math.round(1.5) == 2
    with pytest.raises(ZeroDivisionError):
        oracle.group_for_experts(40, 100)


def test_not_positive_definite():
    k = (1 * ARDRBFKernel(2) + const(1e-12) * EyeKernel()).set_training_vectors(DATASET)
    with pytest.raises(oracle.NotPositiveDefiniteException):
        oracle.get_magic_vector(k, -10.0 * np.eye(3), np.ones(3))


def test_scaling():
    X = np.array([[1.0, 5.0], [3.0, 5.0]])
    s = oracle.scale(X)
    assert np.allclose(s, [[-1.0, 0.0], [1.0, 0.0]])       # population variance; zero variance -> 1


# ---- greedy active-set provider (ActiveSetProvider.scala:58-139) --------------------------------------------------
def test_greedy_provider_fold_semantics():
    from oracle.active_set import _fold_expert
    nan = float("nan")
    assert _fold_expert(np.array([1.0, 3.0, 2.0])) == (3.0, 1)
    assert _fold_expert(np.array([1.0, 3.0, 3.0])) == (3.0, 2)             # ties: the later point wins (oldMax > delta is false)
    md, mi = _fold_expert(np.array([1.0, nan, 5.0]))                       # math.max(NaN, x) = NaN poisons the expert
    assert np.isnan(md) and mi == 2
    assert _fold_expert(np.array([])) == (-1.7976931348623157e308, -1)


def test_greedy_provider_deltas_and_selection():
    """candidate_deltas (vectorised) against a scalar transcription of ASP:109-124, and the selection loop."""
    import math
    from oracle.active_set import candidate_deltas, greedy_active_set, get_next
    rng = np.random.default_rng(4)
    n, d = 120, 3
    X = rng.random((n, d)); y = np.sin(X.sum(1)) + 0.05 * rng.standard_normal(n)
    fac = oracle.get_kernel(lambda: 1.2 * oracle.ARDRBFKernel(np.full(d, 1.5)) + oracle.const(1) * oracle.EyeKernel(), 1e-2)
    theta = fac().get_hyperparameters()
    experts = oracle.get_expert_labels_and_kernels(X, y, fac, 40)
    for _, k in experts:
        k.set_hyperparameters(theta)
    active = X[[5, 17, 60]]
    inst = fac().set_hyperparameters(theta).set_training_vectors(active)
    kmm, s2 = inst.training_kernel(), inst.white_noise_var
    assert abs(s2 - 1.01) < 1e-15                                          # whiteNoiseVar, not the sigma2 parameter
    ye, ke = experts[1]
    c = ke.cross_kernel(active)
    g = sum(k.cross_kernel(active) @ k.cross_kernel(active).T for _, k in experts)
    b = sum(k.cross_kernel(active) @ yy for yy, k in experts)
    pdm = s2 * kmm + g
    kinv, pinv, mv = np.linalg.inv(kmm), np.linalg.inv(pdm), np.linalg.solve(pdm, b)
    dv = candidate_deltas(c, ye, ke.training_kernel_diag(), kinv, pinv, mv, s2)
    for i in (0, 7, len(ye) - 1):
        col = c[:, i]
        pi, qi, mui = col @ kinv @ col, col @ pinv @ col, col @ mv
        sigma = math.sqrt(s2); li = math.sqrt(ke.training_kernel_diag()[i] - pi)
        ksii = 1.0 / ((sigma / li) ** 2 + 1 - qi); kappai = ksii * (1 + 2 * (sigma / li) ** 2)
        delta = -math.log(sigma / li) - (math.log(ksii) + ksii * (1 - kappai) / s2 * (ye[i] - mui) ** 2 - kappai + 2) / 2
        assert abs(dv[i] - delta) <= 1e-12 * max(1.0, abs(delta))
    nxt = get_next(kmm, experts, active, s2)
    assert any(np.array_equal(nxt, x) for x in X)
    sel = greedy_active_set(6, experts, fac, theta, X[5])
    assert sel.shape == (6, d) and np.array_equal(sel[0], X[5])
    assert len({tuple(r) for r in sel}) == 6                               # distinct points on this data
    assert np.array_equal(sel, greedy_active_set(6, experts, fac, theta, X[5]))


def test_greedy_vectorised_fold_matches_scalar_fold():
    """fold_experts (all experts at once, what round_scores selects with) against _fold_expert per expert followed by
    filter(!isNaN).max() (ASP:108-135), on coarse-rounded scores (plenty of ties) with NaNs, up to every expert poisoned."""
    from oracle.active_set import _fold_expert, fold_experts
    rng = np.random.default_rng(12)
    for trial in range(300):
        n = int(rng.integers(1, 120)); E = int(rng.integers(1, n + 1))
        delta = np.round(rng.standard_normal(n), 1)
        if trial % 3 == 0:
            delta[rng.integers(n, size=int(rng.integers(1, 4)))] = np.nan
        if trial % 17 == 0:
            delta[:] = np.nan
        best, best_idx, pick = fold_experts(delta, E)
        want = None
        for e in range(E):
            md, mi = _fold_expert(delta[e::E])
            assert (np.isnan(md) and np.isnan(best[e])) or md == best[e]
            assert best_idx[e] == mi * E + e
            if not np.isnan(md) and (want is None or not (want[0] >= md)):
                want = (md, mi * E + e)
        assert pick == (-1 if want is None else want[1])


def test_greedy_round_scores_matches_get_next():
    """round_scores (all N points at once, BLAS-3) against the oracle's per-expert candidate_deltas and get_next: the
    deltas in both of its formulations, and the pick, for prefixes of 1 to 12 points; a NaN label poisons every expert."""
    from oracle.active_set import candidate_deltas, get_next, round_scores
    rng = np.random.default_rng(31)
    for trial, (n, d, E) in enumerate([(150, 3, 7), (97, 2, 97), (240, 5, 1), (301, 4, 13)]):
        X = rng.random((n, d)); y = np.sin(3 * X.sum(1)) + 0.1 * rng.standard_normal(n)
        beta = rng.uniform(1.0, 3.0, d)
        fac = oracle.get_kernel(lambda: 1.1 * oracle.ARDRBFKernel(beta) + oracle.const(0.5) * oracle.RBFKernel(0.7)
                                + oracle.const(1) * oracle.EyeKernel(), 1e-2)
        theta = fac().get_hyperparameters()
        experts = [(y[e::E], fac().set_hyperparameters(theta).set_training_vectors(X[e::E])) for e in range(E)]
        for r in (1, 2, 5, 12):
            active_idx = rng.permutation(n)[:r]
            rs = round_scores(X, y, active_idx, fac, theta, E)
            inst = fac().set_hyperparameters(theta).set_training_vectors(X[active_idx])
            kmm, s2 = inst.training_kernel(), inst.white_noise_var
            g = sum(k.cross_kernel(X[active_idx]) @ k.cross_kernel(X[active_idx]).T for _, k in experts)
            b = sum(k.cross_kernel(X[active_idx]) @ ye for ye, k in experts)
            pdm = s2 * kmm + g
            kinv, pinv, mv = np.linalg.inv(kmm), np.linalg.inv(pdm), np.linalg.solve(pdm, b)
            for e, (ye, k) in enumerate(experts):
                dv = candidate_deltas(k.cross_kernel(X[active_idx]), ye, k.training_kernel_diag(), kinv, pinv, mv, s2)
                assert np.allclose(rs.delta[e::E], dv, rtol=1e-10, atol=1e-12)
            assert np.allclose(rs.delta_chol, rs.delta, rtol=1e-9, atol=1e-11)
            assert rs.min_eig_a > 0
            assert np.array_equal(X[rs.pick], get_next(kmm, experts, X[active_idx], s2))
        y_bad = y.copy(); y_bad[trial] = np.nan
        rs = round_scores(X, y_bad, [0], fac, theta, E)
        assert rs.pick == -1 and np.all(np.isnan(rs.best))
        bad = [(y_bad[e::E], k) for e, (_, k) in enumerate(experts)]
        with pytest.raises(ValueError, match="empty.max"):
            get_next(fac().set_hyperparameters(theta).set_training_vectors(X[[0]]).training_kernel(), bad, X[[0]], s2)
