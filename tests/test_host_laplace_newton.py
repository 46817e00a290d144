"""The Laplace Newton loop where it branches: a catalogue of cases and its checks on the oracle; no GPU needed.

GPCls:91-111 (classification/GaussianProcessClassifier.scala) compares each candidate with the objective of two accepted
steps back, halves `step` on a rejection and never undoes it, also stops when step <= tol, and after the loop takes pi,
W, L, a and grad log p from the last iteration's input f but d3logP from the final f.  On noisy labels at unit scale
and tol = 1e-6 none of that shows: the loop converges quadratically without a halving.  CASES below are warm-started
θ sequences, found by a seeded search on the oracle and written here as literals, that leave that path:

  (a) halving   a rejected candidate, then an accepted damped step (step < 1, so (1 - step) f counts)
  (b) step      exit by step exhaustion: step <= tol while |old - new| > tol
  (c) loose     tol in {0.1, 0.5, 0.999}: 1 to 3 iterations, the last iteration's input f differs from the final f
  (d) saturated some |f| > 37: the sigmoid rounds to 1 and W to 0
  (e) nan       some |f| > 709: exp(-f) overflows, pi = 0 and d3logP = 0 inf, so the whole gradient is NaN while the
                value stays finite; a later evaluation warm-starts from those modes and recovers
  (f) -inf      a candidate of -inf (log of an underflowed sigmoid)

Each case is one expert of n points (on chip for n <= 117, the global-memory kernel above), so the trace of every
evaluation is the trace of that expert.  The checks:
1. every case reaches its regimes, on both size classes;
2. every decision is decisive: each cand vs old_obj and each |old - new| vs tol clears its threshold by more than
   1e-9 max(1, |.|), so a kernel that rounds differently takes the same branch;
3. the gate of every case (tests/test_gpu_laplace_newton.py uses the same): the existing per-quantity gates, widened to
   16x the oracle's own spread under a 1-ulp symmetric perturbation of K where B is ill-conditioned, and that spread is
   at most 1e-6 relative;
4. numpy restatements of the loop that each make one plausible kernel mistake move the value, the gradient or the
   modes of some case by more than 100x its gate -- so the GPU tests can see every one of them;
5. the oracle raises at tol >= 1: no iteration runs and L stays zero.
"""
import warnings

import numpy as np
import pytest
import scipy.linalg as sla

from oracle.classification import classification_likelihood_and_gradient
from test_gpu_objectives import ATOL_LAP, RTOL_LAP, TOL_NLL, kernel_pair

ON_CHIP_MAX = 117
DECISIVE = 1e-9
SPREAD_FACTOR, SPREAD_CAP = 16.0, 1e-6
MUTANT_FACTOR = 100.0
LOOSE_TOLS = (0.1, 0.5, 0.999)

# (name, data seed, n, d, label noise, kernel family, [θ per evaluation], [tol per evaluation], regimes).  Found by a
# seeded search over n, d, noise in {0, 0.3, 1}, scale 10^U(-2, 5.5), ARD betas 10^U(-2, 1) and tol in {1e-6, 1e-3,
# 1e-1, 0.5, 0.999}, keeping decisive cases whose spread stays under the cap; θ = (scale, betas) of kernel_pair's "ard".
CASES = [
    ("nan_45", 5003, 45, 2, 0.0, "ard",
     [[32200.0, 0.0529, 0.113], [60400.0, 0.612, 0.408], [1.64, 0.507, 0.181]], [1e-06, 0.001, 0.1],
     ("halving", "step", "saturated", "nan", "-inf")),
    ("loose_115", 372, 115, 1, 0.0, "ard",
     [[1640.0, 0.274], [21000.0, 0.212], [3540.0, 0.304], [60900.0, 2.52]], [0.999, 0.5, 0.001, 0.001],
     ("halving", "step", "loose", "saturated", "-inf")),
    ("nan_165", 5003, 165, 2, 0.0, "ard",
     [[32200.0, 0.0529, 0.113], [60400.0, 0.612, 0.408], [1.64, 0.507, 0.181]], [1e-06, 0.001, 0.1],
     ("halving", "step", "saturated", "nan", "-inf")),
    ("loose_nan_120", 5026, 120, 2, 0.3, "ard",
     [[245000.0, 0.436, 0.0171], [151000.0, 0.589, 2.31], [0.777, 0.0101, 0.0379]], [1e-06, 0.1, 0.1],
     ("halving", "step", "loose", "saturated", "nan", "-inf")),
]


# ---- inputs ------------------------------------------------------------------------------------------------------------
def case_data(case):
    """(X, y 0/1, GPU kernel, oracle kernel of the expert) of a case: X ~ N(0, 1), y = [x_0 + noise N(0, 1) > 0]."""
    name, seed, n, d, noise, kind = case[:6]
    rng = np.random.default_rng(seed)
    X = rng.standard_normal((n, d))
    y = (X[:, 0] + noise * rng.standard_normal(n) > 0).astype(np.float64)
    k, ofac = kernel_pair(kind, d, np.ones(d), rng)
    return X, y, k, ofac().set_training_vectors(X)


class FixedKernel:
    """An oracle kernel with K replaced (the derivatives kept): the oracle's sensitivity to a perturbation of K."""

    def __init__(self, K, dK):
        self.K, self.dK = K, dK

    def set_hyperparameters(self, x):
        return self

    def training_kernel_and_derivative(self):
        return self.K, self.dK


def quiet(fn, *a, **kw):
    with warnings.catch_warnings(), np.errstate(all="ignore"):
        warnings.simplefilter("ignore")
        return fn(*a, **kw)


def oracle_sequence(case):
    """Runs the oracle over the case's evaluations from zero modes.  Returns one dict per evaluation: theta, tol, f_in,
    value, grad, f (after), trace, K, dK."""
    X, y, _, ke = case_data(case)
    f = np.zeros(len(y))
    out = []
    for theta, tol in zip(case[6], case[7]):
        theta = np.asarray(theta, dtype=np.float64)
        ke.set_hyperparameters(theta)
        K, dK = ke.training_kernel_and_derivative()
        f_in, tr = f.copy(), []
        v, g = quiet(classification_likelihood_and_gradient, y, f, ke, theta, tol, trace=tr)
        out.append(dict(theta=theta, tol=tol, f_in=f_in, value=v, grad=g, f=f.copy(), trace=tr, K=K, dK=dK))
    return out


# ---- regimes and decisions ---------------------------------------------------------------------------------------------
def regimes(evals):
    """The regimes (a)-(f) the oracle's traces show."""
    got = set()
    for i, ev in enumerate(evals):
        its, exit_ = ev["trace"][:-1], ev["trace"][-1]["exit"]
        halved = False
        for r in its:
            halved |= not r["accepted"]
            if halved and r["accepted"] and r["step"] < 1.0:
                got.add("halving")
            if r["max_abs_f"] > 37.0:
                got.add("saturated")
            if r["cand"] == -np.inf:
                got.add("-inf")
        if exit_ == "step":                               # the trace's exit: |old - new| > tol still holds
            got.add("step")
        if ev["tol"] in LOOSE_TOLS and 1 <= len(its) <= 3:
            got.add("loose")
        if np.abs(ev["f"]).max() > 709.0 and np.all(np.isnan(ev["grad"])) and np.isfinite(ev["value"]) and any(
                np.all(np.isfinite(later["grad"])) for later in evals[i + 1:]):
            got.add("nan")
    return got


def decision_margins(evals):
    """The closest of the rounded comparisons the loop makes, as |lhs - rhs| / max(1, |lhs|, |rhs|): cand > old_obj,
    and |old - new| > tol after each iteration.  A comparison with an infinite side is exact, and so is step > tol
    (step is a power of two, halved exactly): those need no margin."""
    m = [np.inf]
    for ev in evals:
        for r in ev["trace"][:-1]:
            old, new = (r["new_obj"], r["cand"]) if r["accepted"] else (r["old_obj"], r["new_obj"])
            for lhs, rhs, scale in ((r["cand"], r["old_obj"], max(1.0, abs(r["cand"]), abs(r["old_obj"]))),
                                    (abs(old - new), ev["tol"], max(1.0, abs(old), abs(new)))):
                if np.isfinite(lhs) and np.isfinite(rhs):
                    m.append(abs(lhs - rhs) / scale)
    return min(m)


# ---- gates -------------------------------------------------------------------------------------------------------------
def symmetric_signs(n, seed):
    r = np.where(np.random.default_rng(seed).random((n, n)) < 0.5, -1.0, 1.0)
    return np.triu(r) + np.triu(r, 1).T


def gates(case, evals):
    """Per evaluation: (value gate, gradient gate per component, modes gate, the widest spread / cap).  The existing
    gates (TOL_NLL, RTOL_LAP / ATOL_LAP, modes 1e-9 max(1, |f|)) widened to SPREAD_FACTOR x the oracle's spread when K
    is perturbed entry-wise by (1 + 2^-52 r), r = +-1 symmetric, two seeds, from the same warm start."""
    _, y, _, _ = case_data(case)
    out = []
    for ev in evals:
        sv, sg_, sf = 0.0, np.zeros(len(ev["grad"])), 0.0
        for seed in (1, 2):
            Kp = ev["K"] * (1.0 + 2.0 ** -52 * symmetric_signs(len(y), seed))
            f = ev["f_in"].copy()
            v, g = quiet(classification_likelihood_and_gradient, y, f, FixedKernel(Kp, ev["dK"]), ev["theta"], ev["tol"])
            sv = max(sv, abs(v - ev["value"]))
            fin = np.isfinite(ev["grad"])
            sg_[fin] = np.maximum(sg_[fin], np.abs(g[fin] - ev["grad"][fin]))
            sf = max(sf, float(np.abs(f - ev["f"]).max()))
        g0 = np.where(np.isfinite(ev["grad"]), ev["grad"], 0.0)
        atol = ATOL_LAP * np.array([float(np.abs(d).sum()) for d in ev["dK"]])
        fmax = max(1.0, float(np.abs(ev["f"]).max()))
        gv = max(TOL_NLL * abs(ev["value"]), SPREAD_FACTOR * sv)
        gg = np.maximum(RTOL_LAP * np.abs(g0) + atol, SPREAD_FACTOR * sg_)
        gf = max(1e-9 * fmax, SPREAD_FACTOR * sf)
        need = max(SPREAD_FACTOR * sv / max(1.0, abs(ev["value"])),
                   float((SPREAD_FACTOR * sg_ / np.maximum(1.0, np.abs(g0))).max()), SPREAD_FACTOR * sf / fmax)
        out.append((gv, gg, gf, need / SPREAD_CAP))
    return out


def err_over_gate(value, grad, f, ev, gate):
    """The largest error / gate of one evaluation; infinite when the NaN pattern of the gradient differs."""
    gv, gg, gf, _ = gate
    nan0 = np.isnan(ev["grad"])
    if not np.array_equal(np.isnan(grad), nan0) or not np.isfinite(value):
        return np.inf
    fin = ~nan0
    r = [abs(value - ev["value"]) / gv, float(np.abs(f - ev["f"]).max()) / gf]
    if fin.any():
        r.append(float((np.abs(grad[fin] - ev["grad"][fin]) / gg[fin]).max()))
    return max(r)


# ---- the loop with one mistake -----------------------------------------------------------------------------------------
MISTAKES = ("post_final_f", "d3_pre_update", "cmp_new_obj", "step_reset", "L_last_accepted", "no_writeback_on_step")


def _sigmoid(x):
    return 1.0 / (1.0 + np.exp(-x))


def newton(y, f, K, dK, tol, mistake=None):
    """GPCls:74-129 in vector form, with one optional mistake:
    post_final_f          the post-loop pi, W, L, a and grad log p recomputed from the final f
    d3_pre_update         d3logP from the last iteration's input f
    cmp_new_obj           the candidate compared with new_obj
    step_reset            step reset to 1 after an accepted step
    L_last_accepted       L kept from the last accepted iteration
    no_writeback_on_step  the modes not written back after a step-exhausted exit
    Mutates f; returns (-log Z, -grad log Z)."""
    n = len(y)
    old_obj, new_obj, step = -np.inf, -np.finfo(np.float64).max, 1.0
    L = L_acc = np.zeros((n, n))
    pi, sw, a, glp = np.zeros(n), np.zeros(n), np.zeros(n), np.zeros(n)
    f_start, f_last_in = f.copy(), f.copy()

    def iterate(fv, step):
        pi = _sigmoid(fv)
        w = pi * (1.0 - pi)
        sw = np.sqrt(w)
        L = sla.cholesky(np.outer(sw, sw) * K + np.eye(n), lower=True)
        glp = y - pi
        b = w * fv + glp
        t = sla.solve_triangular(L.T, sla.solve_triangular(L, sw * (K @ b), lower=True), lower=False)
        a = b - sw * t
        return pi, sw, L, glp, a, (1.0 - step) * fv + step * (K @ a)

    while abs(old_obj - new_obj) > tol and step > tol:
        f_last_in = f.copy()
        pi, sw, L, glp, a, nf = iterate(f, step)
        cand = -float(a @ nf) / 2.0 + float(np.sum(np.log(_sigmoid((y * 2.0 - 1.0) * nf))))
        if cand > (new_obj if mistake == "cmp_new_obj" else old_obj):
            f[:] = nf
            old_obj, new_obj = new_obj, cand
            L_acc = L
            if mistake == "step_reset":
                step = 1.0
        else:
            step /= 2.0
    step_exit = abs(old_obj - new_obj) > tol
    if mistake == "post_final_f":
        pi, sw, L, glp, a, _ = iterate(f, step)
    if mistake == "L_last_accepted":
        L = L_acc
    logZ = new_obj - float(np.sum(np.log(np.diag(L))))
    R = sw[:, None] * sla.solve_triangular(L.T, sla.solve_triangular(L, np.diag(sw), lower=True), lower=False)
    C = sla.solve_triangular(L, sw[:, None] * K, lower=True)
    fd = f_last_in if mistake == "d3_pre_update" else f
    d3 = -(2.0 * pi - 1.0) * pi * pi * np.exp(-fd)
    s2 = -0.5 * (np.diag(K) - np.sum(C * C, axis=0)) * d3
    grad = []
    for d in dK:
        bb = d @ glp
        grad.append(0.5 * float(a @ d @ a) - 0.5 * float(np.sum(R * d)) + float(s2 @ (bb - K @ (R @ bb))))
    if mistake == "no_writeback_on_step" and step_exit:
        f[:] = f_start
    return -logZ, -np.array(grad)


def mutant_effect(case, evals, gate, mistake):
    """The largest err / gate over the case's evaluations when the whole sequence runs with the mistake."""
    _, y, _, _ = case_data(case)
    f = np.zeros(len(y))
    worst = 0.0
    for ev, gt in zip(evals, gate):
        try:
            v, g = quiet(newton, y, f, ev["K"], ev["dK"], ev["tol"], mistake)
        except (np.linalg.LinAlgError, ValueError):
            return np.inf
        worst = max(worst, err_over_gate(v, g, f, ev, gt))
    return worst


# ---- the tests ---------------------------------------------------------------------------------------------------------
def case_id(case):
    return case[0]


@pytest.fixture(scope="module")
def catalogue():
    out = {}
    for case in CASES:
        evals = oracle_sequence(case)
        out[case[0]] = (evals, gates(case, evals))
    return out


def test_catalogue_covers_every_regime_on_both_size_classes():
    want = {"halving", "step", "loose", "saturated", "nan"}
    for on_chip in (True, False):
        got = set().union(*[set(c[8]) for c in CASES if (c[2] <= ON_CHIP_MAX) == on_chip])
        assert want <= got, ("on chip" if on_chip else "global", want - got)
    assert all(len(c[6]) == len(c[7]) for c in CASES)


@pytest.mark.parametrize("case", CASES, ids=case_id)
def test_case_reaches_its_regimes_decisively(case, catalogue):
    evals, gate = catalogue[case[0]]
    got = regimes(evals)
    margin = decision_margins(evals)
    widest = max(g[3] for g in gate)
    print("%-14s n=%3d: regimes %-40s min decision margin %.2e, widest spread / cap %.2e" % (
        case[0], case[2], ",".join(sorted(got)), margin, widest))
    assert set(case[8]) <= got, (case[0], set(case[8]) - got)
    assert margin > DECISIVE, (case[0], margin)
    assert widest <= 1.0, (case[0], widest)


@pytest.mark.parametrize("case", CASES, ids=case_id)
def test_restated_loop_matches_the_oracle(case, catalogue):
    """The numpy restatement without a mistake is the oracle (so a mutant's distance is the mistake's alone)."""
    evals, gate = catalogue[case[0]]
    assert mutant_effect(case, evals, gate, None) <= 1e-3


@pytest.mark.parametrize("mistake", MISTAKES)
def test_every_mistake_moves_some_case_far_past_its_gate(mistake, catalogue):
    effects = {c[0]: mutant_effect(c, *catalogue[c[0]], mistake) for c in CASES}
    best = max(effects, key=effects.get)
    print("%-22s moves %s" % (mistake, ", ".join("%s %.1e" % (k, v) for k, v in sorted(effects.items(),
                                                                                     key=lambda kv: -kv[1])[:4])))
    assert effects[best] > MUTANT_FACTOR, (mistake, effects)


@pytest.mark.parametrize("tol", [1.0, 1.5, np.inf])
def test_oracle_raises_when_no_iteration_runs(tol):
    case = ("t", 0, 30, 2, 0.3, "ard", [[1.3, 1.0, 1.0]], [tol], ())
    _, y, _, ke = case_data(case)
    theta = np.array([1.3, 1.0, 1.0])
    tr, f = [], np.zeros(len(y))
    with pytest.raises(np.linalg.LinAlgError):
        quiet(classification_likelihood_and_gradient, y, f, ke, theta, tol, trace=tr)
    assert tr == [{"exit": "none"}] and not f.any()
    tr = []
    quiet(classification_likelihood_and_gradient, y, f, ke, theta, 0.999, trace=tr)
    assert len(tr) >= 2 and tr[-1]["exit"] != "none"                 # just below 1 the loop runs


def test_trace_changes_no_bit():
    case = ("t", 3, 40, 2, 0.0, "ard", [], [], ())
    _, y, _, ke = case_data(case)
    for theta, tol in (([30.0, 2.0, 1.0], 1e-6), ([3e3, 0.3, 0.5], 1e-3), ([1.3, 1.0, 1.0], 0.5)):
        theta = np.array(theta)
        f1, f2 = np.zeros(len(y)), np.zeros(len(y))
        v1, g1 = quiet(classification_likelihood_and_gradient, y, f1, ke, theta, tol)
        v2, g2 = quiet(classification_likelihood_and_gradient, y, f2, ke, theta, tol, trace=[])
        assert np.array_equal(np.float64(v1).view(np.int64), np.float64(v2).view(np.int64))
        assert np.array_equal(g1.view(np.int64), g2.view(np.int64)) and np.array_equal(f1.view(np.int64),
                                                                                        f2.view(np.int64))
