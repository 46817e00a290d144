"""Hyper-parameter optimisation, host side (commons/GaussianProcessCommons.scala:66-92 `optimizeHypers`).

Expert grouping as the reference (GPC:26-31: E = Math.round(N / n_e), point i -> expert i % E); the BCM objective
(sum over experts of the negative log marginal likelihood, GPR:55-68, + gradient) runs on the GPU (`sgp_bcm_nll`);
the bound-constrained quasi-Newton loop is SciPy's L-BFGS-B in place of Breeze's `LBFGSB(lower, upper, maxIter,
tolerance = tol)` -- the reference pins no test on the iterate trajectory, so results are compared on the objective
value and on predictive metrics, not on theta.  `optimise_slots` runs that loop for every estimator and model selector
here, over one slot or several in lock-step.

The steps every estimator and model selector shares are written here once: the input rule (`fit_data`), the slot fit
(`fit_slots` over a `slot_objective`), the read-back of a slot's latent modes (`slot_modes`) and the model step
(`produce`, giving a `Fitted` slot, and `own_context`)."""
from __future__ import annotations

import threading
from collections import namedtuple

import numpy as np
from scipy.optimize import minimize

from . import _native as N
from .engine import ProjectedProcessEngine, device_fit_data, is_cuda_tensor


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


def fit_slots(eng, gp, objective, x0s, thetas=None, laplace: bool = False):
    """The hyper-parameters of every slot of `objective` (a `slot_objective`) on the experts uploaded into eng: unless
    `thetas` are given, `optimise_slots` from x0s with gp's bounds, maxIter and tol.  laplace: the Laplace fit
    (GPCls:53-60), which has nothing to optimise without hyper-parameters and runs the Laplace loop once more at every
    slot's theta (GPCls:60), so that the modes are the modes at theta.  Returns (thetas, dict(slots: each slot's
    `optimise_slots` record, or None when nothing was optimised, rounds, launches: the optimisation's, and with laplace
    launches_total: with the call at theta))."""
    launches0 = eng.launch_count()
    records, rounds = None, 0
    if thetas is None:
        thetas = [np.asarray(x0, dtype=np.float64) for x0 in x0s]
        if len(thetas[0]) > 0 or not laplace:
            thetas, records, rounds = optimise_slots(objective, x0s, lbfgsb_bounds(gp.getKernel()), gp._maxIter, gp._tol)
    fit = dict(slots=records, rounds=rounds, launches=eng.launch_count() - launches0)
    if laplace:
        objective(list(enumerate(thetas)))
        fit["launches_total"] = eng.launch_count() - launches0
    return thetas, fit


def slot_objective(gps, entry):
    """The objective of `fit_slots` over slots whose kernels are those of gps[i] (one estimator per slot): entry(slots,
    kernels) -> (values, gradients) evaluates the listed slots at their kernels, in one batched call of the engine."""
    def objective(batch):
        vals, grads = entry([i for i, _ in batch],
                            [gps[i].getKernel().setHyperparameters(np.asarray(t, dtype=np.float64)) for i, t in batch])
        return [(float(v), g) for v, g in zip(vals, grads)]
    return objective


def each(fn):
    """A `slot_objective` entry from a one-kernel entry fn(kernel) -> (value, gradient), called once per listed slot."""
    return lambda slots, kernels: zip(*[fn(k) for k in kernels])


def fit_data(X, y, device: int, what: str, keep_float32: bool = False):
    """The (X, y) of a fit: host arrays, or CUDA tensors for a CUDA tensor X (`device_fit_data`, its messages naming
    `what`).  y is float64; X float64, or float32 as given when keep_float32 (the regression reads float32 points as they
    are; the classifiers read float64)."""
    if is_cuda_tensor(X):
        import torch
        X, y = device_fit_data(X, y, device, what)
        return (X if keep_float32 and X.dtype == torch.float32 else X.to(torch.float64)), y
    X = np.asarray(X)
    return (X if keep_float32 and X.dtype == np.float32 else np.asarray(X, dtype=np.float64)), \
        np.asarray(y, dtype=np.float64)


def expert_count(n_points: int, dataset_size_for_expert: int) -> int:
    """numberOfExperts = Math.round(N / datasetSizeForExpert) (GPC:27); ZeroDivisionError when it is 0."""
    n_experts = int(np.floor(n_points / dataset_size_for_expert + 0.5))
    if n_experts <= 0:
        raise ZeroDivisionError("numberOfExperts == 0 (N < datasetSizeForExpert / 2)")
    return n_experts


def group_for_experts(n_points: int, dataset_size_for_expert: int):
    """GPC:26-31."""
    n_experts = expert_count(n_points, dataset_size_for_expert)
    return [np.arange(e, n_points, n_experts) for e in range(n_experts)]


def slot_modes(eng, on_device: bool, n: int, n_experts: int, store: int, index: int, fold=None):
    """The latent modes of one slot of an upload of n rows grouped into n_experts experts (row i -> expert
    i % n_experts, as every upload groups them), in row order: of `store` (N.SGP_MODES_*, index: the class or mode
    slot), or with fold=k of mode slot index on fold set k of a fold upload.  on_device: a CUDA float64 tensor ungrouped
    on the device; else a host array, read packed expert-major and scattered into row order."""
    if on_device:
        return eng.experts_modes_rows(store, index, n) if fold is None else eng.experts_f_fold_slot_rows(fold, index, n)
    f = np.empty(n)
    f[np.concatenate([np.arange(e, n, n_experts) for e in range(n_experts)])] = \
        eng.experts_modes(store, index, n) if fold is None else eng.experts_f_fold_slot(fold, index, n)
    return f


def pack_experts(X, y, dataset_size_for_expert: int):
    """Expert-major copy of (X, y) for sgp_experts_upload: expert e = points e, e+E, e+2E, ... (GPC:26-31).
    The grouping is a strided layout, so the bulk of the copy is one reshape/transpose (k = N // E full rounds);
    the first N % E experts get one more point each."""
    X = np.asarray(X, dtype=np.float64)
    y = np.asarray(y, dtype=np.float64)
    n, d = X.shape
    n_experts = expert_count(n, dataset_size_for_expert)
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


def optimize_hypers(gp, eng, n_experts: int):
    """The optimal hyper-parameter vector (layout of Kernel.getHyperparameters) of gp's BCM objective over the n_experts
    experts uploaded into eng; records the optimisation in gp.last_objective."""
    (theta,), fit = fit_slots(eng, gp, slot_objective([gp], each(eng.bcm_nll)), [gp.getKernel().getHyperparameters()])
    if fit["slots"] is not None:
        gp.last_objective = dict(fit["slots"][0], n_experts=n_experts, launches=fit["launches"])
    return theta


# A fitted slot: the context holding its active set and magic pair (the model's), the kernel at theta, theta, the active
# set, the magic pair, the statistics (G, b), and the latent modes its labels were (the classifiers; None for the
# regression).  The group fit has returned these eight, in this order, since before they had names.
Fitted = namedtuple("Fitted", "engine kernel theta active_set magic_vector magic_matrix stats latent")


def draw_active_set(gp, X, y, theta):
    """gp's active-set provider on (X, y) at theta (GPC:40-47)."""
    return gp._activeSetProvider(gp._activeSetSize, X, y, gp.getKernel, theta, gp._seed, gp=gp)


def produce(gp, eng, X, y, theta, active_set=None) -> Fitted:
    """produceModel -> projectedProcess (GPC:40-59, 102-110) on eng: the active set (drawn by gp's provider unless
    given), the statistics of (X, y) in gp's shards (PGPH:20-36, with the fp64-kernel fallback) and the tail (PGPH:49-60).
    The slot is eng's, with no latent modes.
    Every model starts from the default precision, as on a freshly acquired context: a fall-back to F64 in one slot's
    statistics must not decide the next slot's path."""
    eng.set_precision(N.SGP_PREC_AUTO)
    if active_set is None:
        active_set = draw_active_set(gp, X, y, theta)
    kernel = gp.getKernel().setHyperparameters(theta)
    stats = eng.statistics(kernel, active_set, X, y, getattr(gp, "_shard_points", 1 << 22))
    mv, mm = eng.magic()
    return Fitted(eng, kernel, theta, active_set, mv, mm, stats, None)


def own_context(fitted: Fitted, device: int, engine_factory=ProjectedProcessEngine) -> Fitted:
    """The fitted slot on a small context of its own, which holds its active set and magic pair: it never runs
    statistics, so it holds no statistics workspace."""
    eng = engine_factory(device)
    eng.begin(fitted.kernel, fitted.active_set)
    eng.set_magic(fitted.magic_vector, fitted.magic_matrix)
    return fitted._replace(engine=eng)
