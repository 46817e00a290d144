"""Hyper-parameter optimisation, host side (commons/GaussianProcessCommons.scala:66-92 `optimizeHypers`).

Expert grouping as the reference (GPC:26-31: E = Math.round(N / n_e), point i -> expert i % E); the BCM objective
(sum over experts of the negative log marginal likelihood, GPR:55-68, + gradient) runs on the GPU (`sgp_bcm_nll`);
the bound-constrained quasi-Newton loop is SciPy's L-BFGS-B in place of Breeze's `LBFGSB(lower, upper, maxIter,
tolerance = tol)` -- the reference pins no test on the iterate trajectory, so results are compared on the objective
value and on predictive metrics, not on theta.  `optimise_slots` runs that loop for every estimator and model selector
here, over one slot or several in lock-step."""
from __future__ import annotations

import threading

import numpy as np
from scipy.optimize import minimize

from .engine import ProjectedProcessEngine


def lbfgsb_bounds(kernel):
    """Kernel.hyperparameterBoundaries as SciPy bounds (an infinite upper bound is None)."""
    lo, up = kernel.hyperparameterBoundaries()
    return [(float(l), None if np.isinf(u) else float(u)) for l, u in zip(lo, up)]


def lbfgsb(objective, x0, bounds, max_iter: int, tol: float):
    """The optimisation step of GaussianProcessClassifier (GPC:66-92 with GPCls's objective): SciPy's L-BFGS-B in place of
    Breeze's LBFGSB(lower, upper, maxIter, tolerance = tol), on `objective(theta) -> (value, gradient)` memoised like
    DiffFunctionMemoized (a point L-BFGS-B visits again is not evaluated again, so the latent modes it warm-starts from
    only move on new points).  Returns (SciPy result, number of evaluations)."""
    memo = {}

    def f(theta):
        key = tuple(theta)
        if key not in memo:
            memo[key] = objective(np.asarray(theta))
        return memo[key]

    res = minimize(f, x0, jac=True, method="L-BFGS-B", bounds=bounds, options=dict(maxiter=max_iter, ftol=tol, gtol=tol))
    return res, len(memo)


class _Aborted(Exception):
    """Raised inside a class's optimisation when another class's evaluation failed."""


def lbfgsb_lockstep(evaluate, x0s, bounds, max_iter: int, tol: float):
    """C independent `lbfgsb` optimisations advanced together.  SciPy's minimize has no reverse-communication interface,
    so each runs in a thread of its own; a round waits until every class still iterating has asked for a new point, then
    `evaluate([(c, theta_c), ...]) -> [(value, gradient), ...]` answers them all at once.  Each class sees exactly the
    values an independent `lbfgsb` would, so its trajectory is the independent one.  An exception in `evaluate` or in a
    class's optimisation stops every class and is raised here.  Returns ([(result, evaluations)] per class, rounds)."""
    n = len(x0s)
    cv = threading.Condition()
    pending, answers, active = {}, {}, set(range(n))
    out, errors = [None] * n, []

    def ask(c, theta):
        with cv:
            pending[c] = theta
            cv.notify_all()
            while c not in answers and not errors:
                cv.wait()
            if c not in answers:
                raise _Aborted()
            return answers.pop(c)

    def run(c):
        try:
            out[c] = lbfgsb(lambda theta: ask(c, theta), x0s[c], bounds, max_iter, tol)
        except _Aborted:
            pass
        except BaseException as e:          # noqa: BLE001 -- handed to the caller below
            with cv:
                errors.append(e)
        finally:
            with cv:
                active.discard(c)
                cv.notify_all()

    threads = [threading.Thread(target=run, args=(c,), daemon=True) for c in range(n)]
    for t in threads:
        t.start()
    rounds = 0
    try:
        while True:
            with cv:
                while active and not errors and not active <= set(pending):
                    cv.wait()
                if errors or not active:
                    break
                batch = sorted(pending.items())
                pending.clear()
            try:
                values = evaluate(batch)
            except BaseException as e:      # noqa: BLE001
                with cv:
                    errors.append(e)
                    cv.notify_all()
                break
            rounds += 1
            with cv:
                for (c, _), v in zip(batch, values):
                    answers[c] = v
                cv.notify_all()
    finally:
        with cv:
            if not errors and active:
                errors.append(RuntimeError("lock-step optimisation stopped early"))
            cv.notify_all()
        for t in threads:
            t.join()
    if errors:
        raise errors[0]
    return out, rounds


def optimise_slots(evaluate, x0s, bounds, max_iter: int, tol: float):
    """The hyper-parameter optimisation of every estimator here: one `lbfgsb` per slot, from x0s[i], with
    `evaluate([(i, theta_i), ...]) -> [(value, gradient), ...]` as the objective of the listed slots.  One slot runs
    `lbfgsb` on the calling thread; several run in lock-step (`lbfgsb_lockstep`), each on the trajectory of its
    independent run.  maxIter <= 0 evaluates nothing (SciPy's L-BFGS-B would still evaluate x0).  Returns (each slot's
    theta, each slot's record dict(value, evaluations, iterations) or None when nothing was optimised, rounds: the
    number of `evaluate` calls)."""
    if max_iter <= 0:
        return [np.asarray(x0, dtype=np.float64) for x0 in x0s], None, 0
    if len(x0s) == 1:
        res, evaluations = lbfgsb(lambda theta: evaluate([(0, theta)])[0], x0s[0], bounds, max_iter, tol)
        results, rounds = [(res, evaluations)], evaluations
    else:
        results, rounds = lbfgsb_lockstep(evaluate, x0s, bounds, max_iter, tol)
    return ([np.asarray(res.x, dtype=np.float64) for res, _ in results],
            [dict(value=float(res.fun), evaluations=ev, iterations=int(res.nit)) for res, ev in results], rounds)


def group_for_experts(n_points: int, dataset_size_for_expert: int):
    """GPC:26-31."""
    n_experts = int(np.floor(n_points / dataset_size_for_expert + 0.5))
    if n_experts <= 0:
        raise ZeroDivisionError("numberOfExperts == 0 (N < datasetSizeForExpert / 2)")
    return [np.arange(e, n_points, n_experts) for e in range(n_experts)]


def pack_experts(X, y, dataset_size_for_expert: int):
    """Expert-major copy of (X, y) for sgp_experts_upload: expert e = points e, e+E, e+2E, ... (GPC:26-31).
    The grouping is a strided layout, so the bulk of the copy is one reshape/transpose (k = N // E full rounds);
    the first N % E experts get one more point each."""
    X = np.asarray(X, dtype=np.float64)
    y = np.asarray(y, dtype=np.float64)
    n, d = X.shape
    n_experts = int(np.floor(n / dataset_size_for_expert + 0.5))           # Math.round(N / n_e), GPC:27
    if n_experts <= 0:
        raise ZeroDivisionError("numberOfExperts == 0 (N < datasetSizeForExpert / 2)")
    k, r = divmod(n, n_experts)                       # every expert has k points, the first r experts k + 1
    sizes = np.full(n_experts, k, dtype=np.int64)
    sizes[:r] += 1
    offsets = np.concatenate([[0], np.cumsum(sizes)])
    Xp = np.empty((n, d)); yp = np.empty(n)
    if r == 0:
        Xp.reshape(n_experts, k, d)[...] = X.reshape(k, n_experts, d).transpose(1, 0, 2)
        yp.reshape(n_experts, k)[...] = y.reshape(k, n_experts).T
    else:
        # experts < r: k+1 points (rows e, e+E, ..., e+kE); experts >= r: k points
        head_X = X[:k * n_experts].reshape(k, n_experts, d)
        head_y = y[:k * n_experts].reshape(k, n_experts)
        a = Xp[:offsets[r]].reshape(r, k + 1, d)
        a[:, :k] = head_X[:, :r].transpose(1, 0, 2)
        a[:, k] = X[k * n_experts:]
        b = yp[:offsets[r]].reshape(r, k + 1)
        b[:, :k] = head_y[:, :r].T
        b[:, k] = y[k * n_experts:]
        Xp[offsets[r]:].reshape(n_experts - r, k, d)[...] = head_X[:, r:].transpose(1, 0, 2)
        yp[offsets[r]:].reshape(n_experts - r, k)[...] = head_y[:, r:].T
    return Xp, yp, offsets


def optimize_hypers(gp, X, y, engine: ProjectedProcessEngine | None = None):
    """Returns the optimal hyper-parameter vector (layout of Kernel.getHyperparameters)."""
    own = engine is None
    engine = engine or ProjectedProcessEngine.acquire(gp._device)
    try:
        # expert grouping (GPC:26-31) as a strided gather on the device while the points stream in (the host-side
        # pack_experts above is the same permutation, kept for callers that hold expert-major data and for the tests)
        n_experts = engine.experts_upload_grouped(X, y, gp._datasetSizeForExpert)
        launches0 = engine.launch_count()
        k0 = gp.getKernel()
        evaluate = lambda batch: [engine.bcm_nll(gp.getKernel().setHyperparameters(t)) for _, t in batch]
        (theta,), records, _ = optimise_slots(evaluate, [k0.getHyperparameters()], lbfgsb_bounds(k0), gp._maxIter,
                                              gp._tol)
        if records is not None:
            gp.last_objective = dict(records[0], n_experts=n_experts, launches=engine.launch_count() - launches0)
        return theta
    finally:
        if own:
            engine.release()
