"""The BCM objective's general (LU) path -- gen_build_kernel, cuBLAS batched LU / inverse, gen_objective_kernel -- against
the fp64 oracle at every expert size it serves (run on an H100: `pytest -m gpu`).

Every case compares `eng.bcm_nll` (or `eng.bcm_nll_folds`) with test_host_bcm_general.blockwise_objective, the blockwise
restatement of oracle.regression.regression_likelihood_and_gradient, under test_gpu_objectives' per-component gate:
TOL_NLL = 1e-9 on the value, |g_i - g0_i| <= RTOL_G |g0_i| + gradient_atol_i on each gradient component.  Every case
asserts that the LU path ran and that a second evaluation returns the same bits, and prints its worst error / gate.
Which launch a case reaches (rows staged, y and alpha in shared memory or in the workspace, refusal) follows from
test_host_bcm_general.lu_plan / lu_outcome.
"""
import functools
import time

import numpy as np
import pytest

import oracle
import spark_gp_b200 as sg
from spark_gp_b200 import _native as N
from spark_gp_b200.hyperopt import lbfgsb, lbfgsb_bounds, pack_experts
from test_gpu_objectives import RTOL_G, TOL_NLL, check_components, kernel_pair, layout, sizes
from test_host_bcm_general import blockwise_objective, lu_outcome, lu_plan

pytestmark = pytest.mark.gpu

WORST = {}


@pytest.fixture(scope="module")
def eng():
    e = sg.ProjectedProcessEngine(0)
    yield e
    e.close()
    if WORST:
        case, ratio = max(WORST.items(), key=lambda kv: kv[1])
        print("\nLU path: largest error / gate %.2e (%s)" % (ratio, case))


def oracle_experts(Xp, yp, off, ofac, theta, factor="lu"):
    """(nll, gradient, per-component atol) of the blockwise oracle, summed over the packed experts."""
    nll0, g0, atol = 0.0, np.zeros(len(theta)), np.zeros(len(theta))
    for e in range(len(off) - 1):
        l, g, a = blockwise_objective(yp[off[e]:off[e + 1]], Xp[off[e]:off[e + 1]], ofac, theta, factor=factor)
        nll0 += l; g0 += g; atol += a
    return nll0, g0, atol


def check_lu(eng, k, want, label, evaluate=None):
    """Evaluates k twice on the uploaded experts; LU path, same bits, value and every gradient component in the gate."""
    nll0, g0, atol = want
    evaluate = evaluate or (lambda: eng.bcm_nll(k))
    t0 = time.perf_counter()
    nll, g = evaluate()
    seconds = time.perf_counter() - t0
    assert eng.last_bcm_path() == 1, label
    nll2, g2 = evaluate()
    assert nll2 == nll and np.array_equal(g2, g), label
    assert len(g) == len(g0)
    dnll = abs(nll - nll0) / abs(nll0)
    assert dnll <= TOL_NLL, "%s: nll %.17g vs %.17g" % (label, nll, nll0)
    worst = max(check_components(g, g0, atol, RTOL_G, label), dnll / TOL_NLL)
    WORST[label] = worst
    print("lu %-48s dnll=%.1e  err/gate=%.2e  (%.2f s)" % (label, dnll, worst, seconds))
    return worst


def run_case(eng, kind, n_max, d, ragged=False, lay="standardised", E=3, seed=0):
    rng = np.random.default_rng(seed + 1000 * n_max + 10 * d + len(kind))
    N_, n_e = sizes(n_max, ragged, E)
    X, beta = layout(lay, N_, d, rng)
    y = np.sin(X.sum(1)) + 0.3 * rng.standard_normal(N_)
    k, ofac = kernel_pair(kind, d, beta, rng)
    Xp, yp, off = pack_experts(X, y, n_e)
    assert np.diff(off).max() == n_max and lu_outcome(len(off) - 1, n_max, d, 1 << 62) == "ok"
    eng.experts_upload(Xp, yp, off)
    plan = lu_plan(len(off) - 1, n_max, d)
    label = "%s %s n_max=%d d=%d%s %s" % (kind, lay, n_max, d, " ragged" if ragged else "",
                                        "staged" if plan["staged"] else "global")
    return check_lu(eng, k, oracle_experts(Xp, yp, off, ofac, k.getHyperparameters()), label)


# ---------------- sizes, uniform and one expert one point short --------------------------------------------------------
@pytest.mark.parametrize("ragged", [False, True])
@pytest.mark.parametrize("n_max", [169, 170, 200, 256, 400, 1000, 2000])
def test_lu_sizes(eng, n_max, ragged):
    run_case(eng, "ard", n_max, 3, ragged=ragged, E=3 if n_max <= 400 else 2)


# ---------------- ARD sweeps: d > 16 needs a second sweep of the gradient ----------------------------------------------
@pytest.mark.parametrize("d", [1, 16, 17, 33, 64])
def test_lu_ard_dimensions(eng, d):
    run_case(eng, "ard_noise" if d == 64 else "ard", 300, d, ragged=(d == 17), E=2)


def test_lu_hyper_parameter_limit(eng):
    """Scale + 71 ARD betas (the hyper-parameter limit): five ARD sweeps."""
    run_case(eng, "ard", 400, 71, E=2)


# ---------------- the row-staging edge: rows in shared memory on one side, read from global memory on the other ---------
@pytest.mark.parametrize("n_max,d", [(381, 64), (382, 64), (1345, 16), (1346, 16)])
def test_lu_staging_edge(eng, n_max, d):
    assert lu_plan(2, n_max, d)["staged"] == (n_max in (381, 1345))
    run_case(eng, "ard", n_max, d, E=2)


# ---------------- kernel families above 169 points ----------------------------------------------------------------------
@pytest.mark.parametrize("kind", ["ard", "ard_noise", "rbf", "ard2", "four", "nested"])
def test_lu_kernel_families(eng, kind):
    run_case(eng, kind, 300, 6, ragged=True, E=2)


@pytest.mark.parametrize("n_max", [400, 1000])
def test_lu_clustered_layout(eng, n_max):
    run_case(eng, "ard", n_max, 4, lay="clustered", E=2)


# ---------------- extreme raggedness: the identity padding of small experts ----------------------------------------------
@pytest.mark.parametrize("counts", [(1, 169, 700), (700, 2, 169, 33)])
def test_lu_extreme_ragged(eng, counts):
    rng = np.random.default_rng(sum(counts))
    d = 3
    X, beta = layout("standardised", sum(counts), d, rng)
    y = np.sin(X.sum(1)) + 0.3 * rng.standard_normal(len(X))
    off = np.concatenate([[0], np.cumsum(counts)]).astype(np.int64)
    k, ofac = kernel_pair("ard2", d, beta, rng)
    eng.experts_upload(X, y, off)
    check_lu(eng, k, oracle_experts(X, y, off, ofac, k.getHyperparameters()), "ard2 experts of %s points" % (counts,))


# ---------------- the shared-memory edge: y and alpha in shared memory (14 511) or in the workspace (14 512) -------------
EDGE_D = 2


@functools.lru_cache(maxsize=None)
def edge_case(n):
    """One expert of n points (the rows with odd index of 2n seeded points), its kernel and the oracle's result (log|det|
    and K^-1 from Cholesky: test_host_bcm_general.test_cholesky_form_matches_lu_oracle)."""
    rng = np.random.default_rng(77)
    X2, beta = layout("standardised", 2 * n, EDGE_D, rng)
    y2 = np.sin(X2.sum(1)) + 0.3 * rng.standard_normal(2 * n)
    k, ofac = kernel_pair("ard", EDGE_D, beta, rng)
    X, y = X2[1::2], y2[1::2]
    return X2, y2, X, y, k, oracle_experts(X, y, np.array([0, n]), ofac, k.getHyperparameters(), factor="cholesky")


@pytest.mark.parametrize("n", [14511, 14512])
def test_lu_shared_memory_edge(eng, n):
    """About three minutes per evaluation on an H100 (one expert: cuBLAS' batched LU and inverse on one 14 512 x 14 512
    matrix and one CTA for the objective), two evaluations per case."""
    assert lu_plan(1, n, EDGE_D)["ya_in_ws"] == (n == 14512)
    _, _, X, y, k, want = edge_case(n)
    eng.experts_upload(X, y, np.array([0, n], dtype=np.int64))
    check_lu(eng, k, want, "ard one expert of %d points d=%d" % (n, EDGE_D))


# ---------------- fold slots on the LU path: each slot against its training set's experts ---------------------------------
def test_lu_folds_slots(eng):
    """Three folds of 2 400 points in experts of ~500 (534 / 533 / 533 points per set), slots over sets 0 and 2."""
    rng = np.random.default_rng(31)
    n, d, n_e = 2400, 3, 500
    X, beta = layout("standardised", n, d, rng)
    y = np.sin(X.sum(1)) + 0.3 * rng.standard_normal(n)
    k, ofac = kernel_pair("ard2", d, beta, rng)
    fold_of = np.arange(n) % 3
    assert list(eng.experts_upload_folds(X, y, fold_of, 3, n_e)) == [3, 3, 3]
    for slot, s in enumerate((0, 2)):
        Xp, yp, off = pack_experts(X[fold_of != s], y[fold_of != s], n_e)
        assert list(np.diff(off)) == [534, 533, 533]
        check_lu(eng, k, oracle_experts(Xp, yp, off, ofac, k.getHyperparameters()), "folds: ard2 set %d" % s,
                 evaluate=lambda slot=slot: tuple(a[slot] for a in eng.bcm_nll_folds([0, 2], [k, k])))


# ---------------- refusal and memory: nothing launched, and the context still evaluates ----------------------------------
def normal_case(eng):
    run_case(eng, "ard", 400, 3, E=2, seed=5)


def refusal_inputs(E, n_e, d=1, seed=3):
    rng = np.random.default_rng(seed)
    X = rng.standard_normal((E * n_e, d))
    y = rng.standard_normal(E * n_e)
    return X, y, 1.3 * sg.ARDRBFKernel(np.full(d, 0.7)) + sg.const(1e-2) * sg.EyeKernel()


def test_lu_workspace_above_the_card_is_nomem(eng):
    """2 600 experts of 2 000 points: 166 GB of LU workspace, more than the card has."""
    X, y, k = refusal_inputs(2600, 2000)
    eng.experts_upload(*pack_experts(X, y, 2000))
    assert lu_outcome(2600, 2000, 1, 80 * 2 ** 30) == "nomem"
    launches = eng.launch_count()
    with pytest.raises(sg.SgpError, match="error %d" % N.SGP_E_NOMEM):
        eng.bcm_nll(k)
    assert eng.launch_count() == launches
    normal_case(eng)


def test_lu_expert_above_the_size_limit_is_refused(eng):
    """One expert of 75 000 points (above 46 340): SGP_E_BADARG before any allocation or launch."""
    X, y, k = refusal_inputs(1, 75000)
    eng.experts_upload(X, y, np.array([0, 75000], dtype=np.int64))
    assert lu_outcome(1, 75000, 1, 1 << 62) == "badarg"
    launches = eng.launch_count()
    with pytest.raises(ValueError, match="46340"):
        eng.bcm_nll(k)
    assert eng.launch_count() == launches
    normal_case(eng)


def test_lu_folds_workspace_above_the_card_is_nomem(eng):
    X, y, k = refusal_inputs(2 * 2600, 2000)
    assert list(eng.experts_upload_folds(X, y, np.arange(len(X)) % 2, 2, 2000)) == [2600, 2600]
    launches = eng.launch_count()
    with pytest.raises(sg.SgpError, match="error %d" % N.SGP_E_NOMEM):
        eng.bcm_nll_folds([0, 1], [k, k])
    assert eng.launch_count() == launches
    normal_case(eng)


def test_lu_folds_expert_above_the_size_limit_is_refused(eng):
    X, y, k = refusal_inputs(2, 75000)
    assert list(eng.experts_upload_folds(X, y, np.arange(len(X)) % 2, 2, 75000)) == [1, 1]
    launches = eng.launch_count()
    with pytest.raises(ValueError, match="46340"):
        eng.bcm_nll_folds([1], [k])
    assert eng.launch_count() == launches
    normal_case(eng)


# ---------------- the estimator: L-BFGS-B on the LU objective against the same fit on the oracle -------------------------
def test_regression_fit_with_400_point_experts():
    rng = np.random.default_rng(21)
    n, d, sigma2, iters = 1200, 3, 1e-2, 4
    X = rng.standard_normal((n, d))
    y = np.sin(X.sum(1)) + 0.2 * rng.standard_normal(n)
    beta0 = np.full(d, 0.6)
    gp = (sg.GaussianProcessRegression().setKernel(lambda: 1.0 * sg.ARDRBFKernel(beta0)).setSigma2(sigma2)
          .setDatasetSizeForExpert(400).setActiveSetSize(50).setMaxIter(iters).setTol(1e-9))
    model = gp.fit(X, y)
    ofac = oracle.get_kernel(lambda: 1.0 * oracle.ARDRBFKernel(beta0), sigma2)
    experts = [(y[idx], X[idx]) for idx in oracle.group_for_experts(n, 400)]
    assert len(experts) == 3

    def objective(theta):
        nll, g = 0.0, np.zeros(len(theta))
        for ye, Xe in experts:
            l, ge, _ = blockwise_objective(ye, Xe, ofac, theta)
            nll += l; g += ge
        return nll, g

    k0 = gp.getKernel()
    res, _ = lbfgsb(objective, k0.getHyperparameters(), lbfgsb_bounds(k0), iters, 1e-9)
    theta, theta0 = np.asarray(model.hyperparameters), res.x
    print("fit: GPU %s (%d iterations)  oracle %s (%d iterations)" % (theta, gp.last_objective["iterations"], theta0,
                                                                      res.nit))
    assert gp.last_objective["iterations"] == res.nit
    assert np.abs(theta - theta0).max() <= 1e-7 * np.abs(theta0).max()
    assert abs(gp.last_objective["value"] - res.fun) <= TOL_NLL * abs(res.fun)
