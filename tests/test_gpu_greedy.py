"""The greedy active-set provider on the GPU (`sgp_greedy_active_set`, csrc/greedy.cu) against the per-round oracle
`oracle.active_set.round_scores` (run on an H100: `pytest -m gpu`).  Everything goes through
`ProjectedProcessEngine.greedy_active_set`.

Selection is discontinuous: two correct fp64 implementations may pick different points on a near-tie, so whole index
sequences are not compared.  Round r is checked conditionally on the GPU's own prefix g_0 ... g_{r-1}:
  j*, delta*  the oracle's pick and its score for that prefix (delta = the reference's algebra, `RoundScores.delta`)
  tau_r       max(16 max_i |delta_i - delta_chol_i| over finite entries, 1e-10 (1 + |delta*|)): the disagreement of two
              correct fp64 formulations (explicit inverses + LU against Cholesky solves), with headroom
  delta_2     the best oracle score among points != j* in experts that are not poisoned
  near-optimal  delta[g_r] >= delta* - tau_r
  decisive      if delta* - delta_2 > 2 tau_r then g_r == j*
Every case requires at least 80 % of its checked rounds to be decisive, so that none passes vacuously.  Rounds checked:
all of them up to m = 65, else 1, 2, 3, 2^k - 1, 2^k + 1 and the last.

The fold and argmax semantics (ties, poisoning, the first expert winning) are pinned exactly at the first scoring round
(m_target = 2), where no GEMM is involved and two identical input rows get bit-identical deltas on the device."""
import time

import numpy as np
import pytest

import oracle
from oracle.active_set import round_scores
import spark_gp_b200 as sg

pytestmark = pytest.mark.gpu

TOL_PRED = 1e-5
REFRESH_REL = 1e-7            # greedy.cu refreshes both inverses when a Schur complement falls below this x its diagonal


@pytest.fixture(scope="module")
def eng():
    e = sg.ProjectedProcessEngine(0)
    yield e
    e.close()


def checked_rounds(m):
    if m <= 65:
        return list(range(1, m))
    r = {1, 2, 3, m - 1}
    k = 2
    while k - 1 < m:
        r.update(x for x in (k - 1, k + 1) if 1 <= x < m)
        k *= 2
    return sorted(r)


def tau_of(rs, dstar):
    if not np.isfinite(rs.delta_chol).any():
        return np.inf                  # A does not factor: the round's scores are not determined in fp64
    fin = np.isfinite(rs.delta) & np.isfinite(rs.delta_chol)
    spread = float(np.abs(rs.delta[fin] - rs.delta_chol[fin]).max(initial=0.0))
    return max(16.0 * spread, 1e-10 * (1.0 + abs(dstar)))


def check_round(rs, g, E):
    """The per-round check of the module docstring: returns (shortfall / tau, decisive)."""
    j = rs.pick
    assert j >= 0, "the oracle finds every expert poisoned"
    dstar = rs.delta[j]
    tau = tau_of(rs, dstar)
    dg = rs.delta[g]
    assert dg >= dstar - tau, "GPU pick %d scores %.17g, the oracle's %d scores %.17g (tau %.3g)" % (g, dg, j, dstar, tau)
    alive = ~np.isnan(rs.best)[np.arange(len(rs.delta)) % E]
    others = np.where(alive, rs.delta, -np.inf)
    others[j] = -np.inf
    d2 = np.nanmax(others)
    decisive = bool(dstar - d2 > 2.0 * tau)
    if decisive:
        assert g == j, "decisive round: GPU picked %d, the oracle %d (margin %.3g, tau %.3g)" % (g, j, dstar - d2, tau)
    return (dstar - dg) / tau, decisive


def check_selection(X, y, sel, ofac, theta, E, rounds=None, finite=True, label=""):
    """Every checked round of a GPU selection against round_scores on the GPU's own prefix; returns the summary line."""
    inst = ofac().set_hyperparameters(theta).set_training_vectors(X[sel])
    K = inst.cross_kernel(X)                                   # N x m, column r = k(X, x_{g_r})
    rounds = checked_rounds(len(sel)) if rounds is None else rounds
    worst, n_dec, tau_max = -np.inf, 0, 0.0
    for r in rounds:
        rs = round_scores(X, y, sel[:r], ofac, theta, E, cross=K[:, :r])
        if finite:
            assert not np.isnan(rs.delta).any(), "round %d: the oracle itself finds NaN deltas" % r
        short, dec = check_round(rs, int(sel[r]), E)
        worst, n_dec = max(worst, short), n_dec + dec
        tau_max = max(tau_max, tau_of(rs, rs.delta[rs.pick]))
    line = "%s: %d rounds checked, %d decisive, largest shortfall %.3g tau, largest tau %.3g" % (
        label, len(rounds), n_dec, worst, tau_max)
    print(line)
    assert n_dec >= 0.8 * len(rounds), line
    return line


def _uniform(n, d, seed, f=1.0):
    rng = np.random.default_rng(seed)
    X = rng.random((n, d))
    return X, np.sin(f * X.sum(1)) + 0.1 * rng.standard_normal(n)


def _pair(user_sg, user_or, sigma2):
    """The estimator's kernel (GPC:18 appends sigma2.const * Eye) in the package's DSL and the oracle's."""
    ofac = oracle.get_kernel(user_or, sigma2)
    return user_sg() + sg.const(sigma2) * sg.EyeKernel(), ofac, ofac().get_hyperparameters()


def _default(d, beta, sigma2):
    return _pair(lambda: 1 * sg.ARDRBFKernel(np.full(d, beta)) + sg.const(1) * sg.EyeKernel(),
                 lambda: 1 * oracle.ARDRBFKernel(np.full(d, beta)) + oracle.const(1) * oracle.EyeKernel(), sigma2)


def _four_terms(d):
    rng = np.random.default_rng(3)
    b1, b2 = rng.uniform(0.2, 0.4, d), rng.uniform(0.4, 0.7, d)
    return _pair(lambda: 0.7 * sg.ARDRBFKernel(b1) + 0.5 * sg.ARDRBFKernel(b2) + 0.4 * sg.RBFKernel(1.1)
                 + 0.3 * sg.RBFKernel(2.3) + sg.WhiteNoiseKernel(0.2, 0, 1),
                 lambda: 0.7 * oracle.ARDRBFKernel(b1) + 0.5 * oracle.ARDRBFKernel(b2) + 0.4 * oracle.RBFKernel(1.1)
                 + 0.3 * oracle.RBFKernel(2.3) + oracle.WhiteNoiseKernel(0.2, 0, 1), 1e-2)


# ---- A. per-round parity at production sizes ---------------------------------------------------------------------------
CASES = {
    "default-kernel": dict(n=50_000, d=8, m=512, E=500, first=11, kernel=lambda: _default(8, 1.5, 1e-2)),
    "baseline-size": dict(n=20_000, d=5, m=1000, E=200, first=3, kernel=lambda: _default(5, np.sqrt(18 / 5), 1e-2)),
    "rbf-d1": dict(n=20_011, d=1, m=128, E=2001, first=7,
                   kernel=lambda: _pair(lambda: 1.3 * sg.RBFKernel(0.05), lambda: 1.3 * oracle.RBFKernel(0.05), 0.1)),
    "four-terms": dict(n=30_000, d=17, m=256, E=300, first=29, kernel=lambda: _four_terms(17)),
    "wide": dict(n=8_000, d=100, m=96, E=80, first=0,
                 kernel=lambda: _pair(lambda: 1 * sg.ARDRBFKernel(np.full(100, 0.15)) + sg.const(1) * sg.EyeKernel(),
                                      lambda: 1 * oracle.ARDRBFKernel(np.full(100, 0.15)) + oracle.const(1) * oracle.EyeKernel(),
                                      1e-2)),
    "scale": dict(n=200_000, d=8, m=256, E=2000, first=7, kernel=lambda: _default(8, 3.0, 1e-1)),
}


@pytest.mark.parametrize("case", list(CASES))
def test_rounds_match_oracle_at_production_sizes(eng, case):
    c = CASES[case]
    X, y = _uniform(c["n"], c["d"], seed=len(case), f=2.0)
    kernel, ofac, theta = c["kernel"]()
    t0 = time.perf_counter()
    sel = eng.greedy_active_set(kernel, X, y, c["E"], c["first"], c["m"])
    t1 = time.perf_counter()
    assert sel.shape == (c["m"],) and sel[0] == c["first"] and sel.min() >= 0 and sel.max() < c["n"]
    line = check_selection(X, y, sel, ofac, theta, c["E"], label="%s %d x %d, m = %d, E = %d" % (case, c["n"], c["d"], c["m"], c["E"]))
    print("%s: GPU %.3f s, %d distinct, oracle %.1f s" % (line, t1 - t0, len(np.unique(sel)), time.perf_counter() - t1))


# ---- B. a repeated selection: the Cholesky refresh ------------------------------------------------------------------------
def _schur(X, ofac, theta, prefix, j):
    """(s~, kii, s, s2 kii + gamma) of greedy.cu's bordered step that adds point j to the active set X[prefix]."""
    inst = ofac().set_hyperparameters(theta).set_training_vectors(X[list(prefix) + [j]])
    K = inst.cross_kernel(X)                                   # N x (r + 1)
    kmm = inst.training_kernel()
    s2, kii = inst.white_noise_var, float(inst.training_kernel_diag()[0])
    A = s2 * kmm + K.T @ K
    r = len(prefix)
    c, w = kmm[:r, r], A[:r, r]
    s1 = kii - c @ np.linalg.solve(kmm[:r, :r], c)
    s = A[r, r] - w @ np.linalg.solve(A[:r, :r], w)
    return s1, kii, s, A[r, r], A


# (seed, sigma2, n, d, E, m): 1e-6 on the larger set is the case where skipping the refresh turns the NotPositiveDefinite
# the reference raises into garbage scores (every expert NaN)
REFRESH = [(0, 1e-8, 4000, 3, 40, 40), (0, 1e-5, 4000, 3, 40, 40), (1, 1e-6, 20000, 2, 200, 64)]


@pytest.mark.parametrize("seed,sigma2,n,d,E,m", REFRESH)
def test_repeated_point_takes_the_refresh_path(eng, seed, sigma2, n, d, E, m):
    """Two ARD terms, no Eye term but sigma2, clustered data: the reference does not exclude selected points, and here it
    selects one twice.  At that round the oracle confirms that a Schur complement crosses greedy.cu's refresh threshold;
    the rounds after it must stay near-optimal.  With sigma2 <= 1e-6 the bordered A becomes singular to working precision:
    a NotPositiveDefiniteException is accepted only where the oracle's smallest eigenvalue of A is within tau_r ||A|| of
    0 (tau_r of the round whose pick the failed step adds)."""
    rng = np.random.default_rng(seed)
    centres = rng.random((8, d))
    X = centres[rng.integers(8, size=n)] + 0.02 * rng.standard_normal((n, d))
    y = np.sin(3 * X.sum(1)) + 0.1 * rng.standard_normal(n)
    b1, b2 = np.full(d, 1.5), np.full(d, 6.0)
    kernel, ofac, theta = _pair(lambda: 0.8 * sg.ARDRBFKernel(b1) + 0.5 * sg.ARDRBFKernel(b2),
                                lambda: 0.8 * oracle.ARDRBFKernel(b1) + 0.5 * oracle.ARDRBFKernel(b2), sigma2)
    try:
        sel = eng.greedy_active_set(kernel, X, y, E, 5, m)
        failed_at = None
    except sg.NotPositiveDefiniteException:
        failed_at = next(k for k in range(2, m + 1) if not _completes(eng, kernel, X, y, E, k))
        sel = eng.greedy_active_set(kernel, X, y, E, 5, failed_at - 1)
    rep = next((r for r in range(1, len(sel)) if sel[r] in sel[:r]), None)
    assert rep is not None, "no point was selected twice: the case does not reach the refresh path"
    rs = round_scores(X, y, sel[:rep], ofac, theta, E)
    check_round(rs, int(sel[rep]), E)
    s1, kii, s, diag, A = _schur(X, ofac, theta, sel[:rep], int(sel[rep]))
    print("sigma2 %g: point %d selected again at round %d: s~/kii = %.3g, s/(s2 kii + gamma) = %.3g" % (
        sigma2, sel[rep], rep, s1 / kii, s / diag))
    assert s1 < REFRESH_REL * kii or s < REFRESH_REL * diag, "the repeat does not cross the refresh threshold"
    if failed_at is not None:
        last = failed_at - 2                                   # the round whose pick the failed bordered step adds
        assert last >= rep, "NotPositiveDefinite before any point was selected twice"
        if last > rep:
            rs = round_scores(X, y, sel[:last], ofac, theta, E)
            check_round(rs, int(sel[last]), E)
            A = _schur(X, ofac, theta, sel[:last], int(sel[last]))[4]
        ev = np.linalg.eigvalsh(A)
        tau = tau_of(rs, rs.delta[rs.pick])
        print("sigma2 %g: NotPositiveDefinite adding round %d's pick: lambda_min(A) = %.3g, tau ||A|| = %.3g" % (
            sigma2, last, ev[0], tau * ev[-1]))
        assert abs(ev[0]) <= tau * ev[-1]
        return
    assert len(sel) == m
    check_selection(X, y, sel, ofac, theta, E, rounds=list(range(rep + 1, m)), finite=False,
                    label="refresh sigma2 %g, after the repeat at round %d" % (sigma2, rep))


def _completes(eng, kernel, X, y, E, k):
    try:
        eng.greedy_active_set(kernel, X, y, E, 5, k)
        return True
    except sg.NotPositiveDefiniteException:
        return False


# ---- C. fold and argmax semantics, exactly ---------------------------------------------------------------------------------
def _twin_case(E, n0, i0):
    """X = [X0; X0], y = [y0; y0] with a planted best point i0 (a large label): its two copies i0 and i0 + n0 tie
    bit for bit at the first scoring round."""
    rng = np.random.default_rng(E + n0)
    X0 = rng.random((n0, 2))
    y0 = np.sin(3 * X0.sum(1)) + 0.1 * rng.standard_normal(n0)
    y0[i0] = 6.0
    return np.vstack([X0, X0]), np.concatenate([y0, y0])


# (E, n0, i0): same expert (n0 % E == 0, the later copy wins) or two experts (the smaller wins) on the same argmax thread
# (e = e' mod 256) or on two threads; experts >= 256 are only reached by a thread's second and later visits
TWINS = [(1, 300, 17), (2, 300, 17), (2, 301, 18), (255, 510, 300), (255, 700, 40), (256, 512, 300), (256, 700, 255),
         (257, 514, 300), (257, 1284, 257), (257, 1285, 256), (257, 700, 3), (1000, 3000, 2600), (1000, 3256, 1300),
         (1000, 3700, 1100), (5000, 10000, 9000), (5000, 10512, 4300), (5000, 7000, 6000)]


@pytest.mark.parametrize("E,n0,i0", TWINS)
def test_ties_and_experts_resolve_as_the_reference(eng, E, n0, i0):
    X, y = _twin_case(E, n0, i0)
    kernel, ofac, theta = _default(2, 2.0, 1e-2)
    first = (i0 + 1) % n0
    rs = round_scores(X, y, [first], ofac, theta, E)
    twins = [i0, i0 + n0]
    assert rs.delta[i0] == rs.delta[i0 + n0]
    rest = np.delete(rs.delta, twins)
    assert rs.delta[i0] - rest.max() > 1e-3 * abs(rs.delta[i0]), "the planted point is not the clear best"
    e1, e2 = i0 % E, (i0 + n0) % E
    assert rs.pick == (i0 + n0 if e1 == e2 else (i0 if e1 < e2 else i0 + n0))
    sel = eng.greedy_active_set(kernel, X, y, E, first, 2)
    assert list(sel) == [first, rs.pick]


# ---- D. edges and error paths ------------------------------------------------------------------------------------------------
def test_one_point_selects_nothing_on_the_device(eng):
    X, y = _uniform(500, 3, 1)
    kernel, _, _ = _default(3, 1.5, 1e-2)
    before = eng.launch_count()
    assert list(eng.greedy_active_set(kernel, X, y, 5, 123, 1)) == [123]
    assert eng.launch_count() == before


@pytest.mark.parametrize("n,first,m,E", [(500, 499, 2, 5), (1, 0, 3, 1), (37, 36, 12, 37), (999, 998, 20, 10)])
def test_edges_match_oracle(eng, n, first, m, E):
    X, y = _uniform(n, 3, n + m)
    kernel, ofac, theta = _default(3, 1.5, 1e-2)
    sel = eng.greedy_active_set(kernel, X, y, E, first, m)
    assert sel[0] == first and len(sel) == m
    for r in range(1, m):
        rs = round_scores(X, y, sel[:r], ofac, theta, E)
        if n == 1:
            assert rs.pick == 0 and sel[r] == 0
        else:
            check_round(rs, int(sel[r]), E)


def test_nan_label_is_empty_max_and_the_context_survives(eng):
    X, y = _uniform(3000, 4, 2)
    kernel, ofac, theta = _default(4, 1.5, 1e-2)
    bad = y.copy()
    bad[1234] = np.nan
    assert round_scores(X, bad, [5], ofac, theta, 30).pick == -1
    with pytest.raises(ValueError, match="empty.max"):
        eng.greedy_active_set(kernel, X, bad, 30, 5, 4)
    sel = eng.greedy_active_set(kernel, X, y, 30, 5, 24)
    check_selection(X, y, sel, ofac, theta, 30, label="after empty.max")


def test_too_large_is_nomem_before_allocating_and_the_context_survives(eng):
    n = 12_000_000                       # the N x m cross kernel alone is 96 GB at m = 1000
    X = np.zeros((n, 1))
    y = np.zeros(n)
    kernel, _, _ = _default(1, 1.0, 1e-2)
    with pytest.raises(sg.SgpError, match="does not fit"):
        eng.greedy_active_set(kernel, X, y, 1000, 0, 1000)
    del X, y
    X, y = _uniform(2000, 2, 4)
    kernel, ofac, theta = _default(2, 2.0, 1e-2)
    sel = eng.greedy_active_set(kernel, X, y, 20, 9, 16)
    check_selection(X, y, sel, ofac, theta, 20, label="after NOMEM")


def test_deterministic_and_leaves_an_open_window_untouched(eng):
    X, y = _uniform(20000, 5, 6)
    kernel, _, _ = _default(5, 1.5, 1e-2)
    a = eng.greedy_active_set(kernel, X, y, 200, 17, 64)
    b = eng.greedy_active_set(kernel, X, y, 200, 17, 64)
    assert np.array_equal(a, b)
    Z = X[:48]

    def window(with_greedy):
        eng.begin(kernel, Z)
        eng.accumulate(X[:12000], y[:12000])
        if with_greedy:
            eng.greedy_active_set(kernel, X, y, 200, 3, 20)
        eng.accumulate(X[12000:], y[12000:])
        G, bb = eng.finish()
        return G, bb

    G0, b0 = window(False)
    G1, b1 = window(True)
    assert np.array_equal(G0, G1) and np.array_equal(b0, b1)


# ---- E. through the estimator -------------------------------------------------------------------------------------------------
def test_fit_with_the_default_provider_matches_projected_process():
    n, d, m = 30_000, 6, 64
    X, y = _uniform(n, d, 8, f=2.0)
    beta = np.full(d, 1.2)
    gp = (sg.GaussianProcessRegression().setKernel(lambda: 1 * sg.ARDRBFKernel(beta) + sg.const(1) * sg.EyeKernel())
          .setSigma2(1e-2).setDatasetSizeForExpert(100).setActiveSetSize(m).setMaxIter(0).setSeed(5)
          .setActiveSetProvider(sg.GreedilyOptimizingActiveSetProvider()))
    theta = gp.getKernel().getHyperparameters()
    assert int(np.floor(n / 100 + 0.5)) > 256
    active = gp._activeSetProvider(m, X, y, gp.getKernel, theta, 5, gp=gp)
    model = gp.fit(X, y, hyperparameters=theta)
    ofac = oracle.get_kernel(lambda: 1 * oracle.ARDRBFKernel(beta) + oracle.const(1) * oracle.EyeKernel(), 1e-2)
    experts = oracle.get_expert_labels_and_kernels(X, y, ofac, 100)
    pred, _, _ = oracle.projected_process(experts, active, ofac, theta)
    Xt = np.random.default_rng(9).random((300, d))
    m0, _ = pred.predict_many(Xt)
    assert np.abs(model.predict(Xt) - m0).max() / np.abs(m0).max() <= TOL_PRED
