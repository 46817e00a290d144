"""Runs the same seeded inputs through this tree's libsgp.so and another build of it (e.g. the parent commit's) in one
process, and checks that every output is bit-identical.

  python tools/compare_builds.py --lib OTHER/libsgp.so [--time] [--out DIR]

Covered, each on both builds:
  - G and b on SGP_PREC_F64, _F64_STRICT, _I8 and _I8_DIRECT, with 1 to 4 kernel terms plus an Eye term (both fp64 loops:
    the pipelined one of one term with d <= 32 and the generic one);
  - the magic vector and matrix on the Cholesky tail path and on the eigenvalue + LU path;
  - sgp_predict (mean and variance) and sgp_predict_device (fp32 and fp64 rows); sgp_cross_kernel; sgp_kmn_sweep;
  - sgp_bcm_nll value and gradient on the register, shared-memory and LU variants; sgp_laplace_nll value, gradient and
    the latent modes f; sgp_laplace_nll_any_size on the global-memory kernel and sgp_laplace_nll_classes_any_size on
    both kernels (values, gradients and every class's modes over two warm-started calls); sgp_greedy_active_set indices;
  - sgp_laplace_nll_slots_any_size on both kernels and sgp_laplace_nll_fold_slots_any_size over sets whose largest
    experts are 116, 117 and 118 points (both kernels in one call); sgp_bcm_nll_folds and sgp_bcm_nll_slots with a slot
    that falls back to LU; every mode getter, host and device;
  - refusals: the return code (the exception it maps to), the sgp_last_error text and the launches made.
Every per-expert objective case also compares the launches it made.  Outputs are compared as bit patterns.  The script
prints one line per case and exits with 1 if any case differs.
--time times the fp64 statistics kernel (both loops), prediction and the per-expert objectives (10^4 experts of 100
points, d = 16: bcm_nll, laplace_nll_any_size, laplace_nll_classes_any_size at C = 3, one fold-slot call at K = 10) on
both builds, alternated in the same process: median of 5 synchronised calls after a warm-up, with the card's name and
power limit.  --out writes the report there."""
from __future__ import annotations

import argparse
import ctypes as C
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import spark_gp_b200 as sg                          # noqa: E402
from spark_gp_b200 import _native as N              # noqa: E402
from spark_gp_b200.engine import ProjectedProcessEngine   # noqa: E402
from spark_gp_b200.hyperopt import pack_experts     # noqa: E402


class _Absent:
    """An entry this tree declares and the other build does not export (a later addition to the C-ABI)."""

    def __init__(self, name):
        self.name = name

    def __call__(self, *args):
        raise RuntimeError("%s is not in the other build" % self.name)


class _OlderLib(C.CDLL):
    def __getattr__(self, name):
        try:
            return super().__getattr__(name)
        except AttributeError:
            if name.startswith("__"):
                raise
            stub = _Absent(name)
            setattr(self, name, stub)
            return stub


def load_lib(path):
    """Another libsgp.so with the ctypes bindings of _native (the C-ABI is the same, less the entries added since)."""
    saved = N.LIB_PATH, N._lib, N.C.CDLL
    N.LIB_PATH, N._lib, N.C.CDLL = os.path.abspath(path), None, _OlderLib
    try:
        return N.load()
    finally:
        N.LIB_PATH, N._lib, N.C.CDLL = saved


def engine_on(lib):
    e = ProjectedProcessEngine.__new__(ProjectedProcessEngine)
    e._lib, e._h, e.m, e.d, e._device, e._has_comm = lib, C.c_void_p(), 0, 0, 0, False
    if lib.sgp_ctx_create(C.byref(e._h), 0) != N.SGP_OK:
        raise RuntimeError("sgp_ctx_create failed: %s" % lib.sgp_last_error(None).decode())
    return e


def kernel(n_terms, d, rng):
    """n_terms non-Eye terms (ARD, then RBF, alternating) with distinct scales, plus a noise Eye term."""
    k = None
    for t in range(n_terms):
        term = sg.ARDRBFKernel((0.5 + rng.random(d)) / np.sqrt(d)) if t % 2 == 0 else sg.RBFKernel(0.7 + 0.4 * t)
        k = (0.6 + 0.3 * t) * term if k is None else k + (0.6 + 0.3 * t) * term
    return k + sg.const(1e-3) * sg.EyeKernel()


def stats_case(e, n_terms, d, m, n, prec, seed):
    import torch
    rng = np.random.default_rng(seed)
    k = kernel(n_terms, d, rng)
    X, Z, Xt = rng.random((n, d)).astype(np.float32), rng.random((m, d)), rng.random((3000, d))
    y = np.sin(X.astype(np.float64).sum(1)) + 0.1 * rng.standard_normal(n)
    e.set_precision(prec)
    e.begin(k, Z)
    e.accumulate(X, y)
    out = dict(path=np.array([e.last_path()]))
    out["G"], out["b"] = e.finish()
    try:
        out["magic_v"], out["magic_M"] = e.magic()
        out["tail_path"] = np.array([e.last_tail_path()])
    except sg.NotPositiveDefiniteException as exc:     # int8 statistics of a small n can leave A indefinite
        out["error"] = np.frombuffer(type(exc).__name__.encode(), dtype=np.uint8)
        S = rng.standard_normal((m, m))
        e.set_magic(rng.standard_normal(m), S + S.T)
    out["mean"], out["var"] = e.predict(Xt)
    for dt in (torch.float32, torch.float64):
        mean, var = e.predict_tensor(torch.from_numpy(Xt).to("cuda", dt))
        out["device_mean_" + str(dt)], out["device_var_" + str(dt)] = mean.cpu().numpy(), var.cpu().numpy()
    out["cross_kernel"] = e.cross_kernel(Xt[:500])
    if prec == N.SGP_PREC_I8:                          # the sweep needs the tensor-core mode's shape
        out["kmn_sweep"] = e.kmn_sweep(X[:5000])
    return out


def lu_tail_case(e, seed):
    """G = -wn K_mm + v v' makes A = v v' semi-definite: Cholesky breaks down and the tail takes dsyevd + LU."""
    import oracle
    rng = np.random.default_rng(seed)
    beta = (0.5 + rng.random(3)) / np.sqrt(3)
    Z, v = rng.random((40, 3)), rng.random(40)
    e.begin(1 * sg.ARDRBFKernel(beta) + sg.const(0.1) * sg.EyeKernel(), Z)
    kmm = (1 * oracle.ARDRBFKernel(beta) + oracle.const(0.1) * oracle.EyeKernel()).set_training_vectors(Z).training_kernel()
    try:
        mv, mm = e.magic(G=-0.1 * kmm + np.outer(v, v), b=np.ones(40))
        out = dict(magic_v=mv, magic_M=mm)
    except (sg.NotPositiveDefiniteException, sg.MatrixSingularException) as exc:
        out = dict(error=np.frombuffer(type(exc).__name__.encode(), dtype=np.uint8))
    out["tail_path"] = np.array([e.last_tail_path()])
    return out


def bcm_case(e, n_terms, n_e, seed):
    rng = np.random.default_rng(seed)
    X = rng.standard_normal((20 * n_e, 4))
    y = np.sin(X.sum(1)) + 0.3 * rng.standard_normal(len(X))
    e.experts_upload(*pack_experts(X, y, n_e))
    v, g = e.bcm_nll(kernel(n_terms, 4, rng))
    return dict(value=np.array([v]), grad=g, lu=np.array([e.last_bcm_path()]))


def laplace_case(e, n_terms, seed):
    rng = np.random.default_rng(seed)
    X = rng.standard_normal((2000, 3))
    y = (np.sin(2 * X[:, 0]) + 0.3 * rng.standard_normal(len(X)) > 0).astype(np.float64)
    e.experts_upload(*pack_experts(X, y, 100))
    v, g = e.laplace_nll(kernel(n_terms, 3, rng), 1e-6)
    return dict(value=np.array([v]), grad=g, f=e.experts_f(len(X)))


def laplace_global_case(e, n_terms, seed):
    """Experts of 150 points: sgp_laplace_nll_any_size on the global-memory kernel, two warm-started evaluations."""
    rng = np.random.default_rng(seed)
    X = rng.standard_normal((600, 3))
    y = (np.sin(2 * X[:, 0]) + 0.3 * rng.standard_normal(len(X)) > 0).astype(np.float64)
    e.experts_upload(*pack_experts(X, y, 150))
    k = kernel(n_terms, 3, rng)
    out = {}
    for step in range(2):
        v, g = e.laplace_nll_any_size(k.setHyperparameters(k.getHyperparameters() * (1.0 + 0.1 * step)), 1e-6)
        out.update({"value%d" % step: np.array([v]), "grad%d" % step: g, "f%d" % step: e.experts_f(len(X))})
    out["path"] = np.array([e.last_laplace_path()])
    return out


def laplace_classes_case(e, n_terms, n_e, seed):
    """sgp_laplace_nll_classes_any_size over 3 classes: every class, then a permuted subset warm-started."""
    rng = np.random.default_rng(seed)
    X = rng.standard_normal((4 * n_e, 3))
    s = np.sin(2 * X[:, 0]) + X[:, 2] + 0.3 * rng.standard_normal(len(X))
    y = np.digitize(s, np.quantile(s, [1 / 3, 2 / 3])).astype(np.float64)
    e.experts_upload(*pack_experts(X, y, n_e))
    k = kernel(n_terms, 3, rng)
    t0 = k.getHyperparameters()
    out = {}
    for step, classes in enumerate(([0, 1, 2], [2, 0])):
        ks = [kernel(n_terms, 3, np.random.default_rng(seed)).setHyperparameters(t0 * (1.0 + 0.07 * c + 0.1 * step))
              for c in classes]
        v, g = e.laplace_nll_classes_any_size(3, classes, ks, 1e-6)
        out.update({"value%d" % step: v, "grad%d" % step: g})
        for c in range(3):
            out["f%d_class%d" % (step, c)] = e.experts_f_class(c, len(X))
    out["path"] = np.array([e.last_laplace_path()])
    return out


def launches(e, out, key, call):
    """call(), recording the launches it made under out[key + "_launches"]; returns what call returns."""
    l0 = e.launch_count()
    r = call()
    out[key + "_launches"] = np.array([e.launch_count() - l0])
    return r


def binary_data(n, d, rng):
    X = rng.standard_normal((n, d))
    return X, (np.sin(2 * X[:, 0]) + 0.3 * rng.standard_normal(n) > 0).astype(np.float64)


def laplace_slots_case(e, n_e, seed):
    """sgp_laplace_nll_slots_any_size: 4 mode slots, classes repeated, two warm-started calls, then every slot's modes."""
    rng = np.random.default_rng(seed)
    X, y = binary_data(4 * n_e, 3, rng)
    e.experts_upload_grouped(X, y, n_e)
    t0 = kernel(2, 3, rng).getHyperparameters()
    out = {}
    for step, (modes, classes) in enumerate((([0, 1, 2, 3], [1, 0, 1, 1]), ([3, 1], [0, 1]))):
        ks = [kernel(2, 3, np.random.default_rng(seed)).setHyperparameters(t0 * (1.0 + 0.05 * m + 0.1 * step))
              for m in modes]
        v, g = launches(e, out, "call%d" % step, lambda: e.laplace_nll_slots_any_size(4, modes, classes, ks, 1e-6))
        out.update({"value%d" % step: v, "grad%d" % step: g})
    for m in range(4):
        out["f_slot%d" % m] = e.experts_f_slot(m, len(X))
    out["path"] = np.array([e.last_laplace_path()])
    return out


def fold_data(rng, counts, d=3):
    """Points with fold_of giving each fold counts[k] points, in a seeded order."""
    fold_of = rng.permutation(np.repeat(np.arange(len(counts)), counts)).astype(np.int32)
    X = rng.standard_normal((len(fold_of), d))
    return X, fold_of


def laplace_fold_slots_case(e, seed):
    """sgp_laplace_nll_fold_slots_any_size over 3 sets with datasetSizeForExpert 117: folds of 232, 231 and 237 of 700
    points leave sets of 468, 469 and 463 points in 4 experts each, whose largest are 117 (on chip), 118 (global memory)
    and 116 points.  The list starts with set 1, so the on-chip | global split reorders it; two warm-started calls."""
    rng = np.random.default_rng(seed)
    X, fold_of = fold_data(rng, [232, 231, 237])
    y = (np.sin(2 * X[:, 0]) + 0.3 * rng.standard_normal(len(X)) > 0).astype(np.float64)
    out = {"experts": e.experts_upload_folds(X, y, fold_of, 3, 117)}
    t0 = kernel(1, 3, rng).getHyperparameters()
    sets, classes = [1, 0, 2, 1], [0, 1, 0, 1]
    for step in range(2):
        ks = [kernel(1, 3, np.random.default_rng(seed)).setHyperparameters(t0 * (1.0 + 0.05 * i + 0.1 * step))
              for i in range(4)]
        v, g = launches(e, out, "call%d" % step,
                        lambda: e.laplace_nll_fold_slots_any_size(5, [3, 0, 4, 1], sets, classes, ks, 1e-6))
        out.update({"value%d" % step: v, "grad%d" % step: g})
    out["path"] = np.array([e.last_laplace_path()])
    n_k = len(X) - np.bincount(fold_of)
    for s, m in zip(sets, (3, 0, 4, 1)):
        out["f_set%d_slot%d" % (s, m)] = e.experts_f_fold_slot(s, m, int(n_k[s]))
        out["f_rows_set%d_slot%d" % (s, m)] = e.experts_f_fold_slot_rows(s, m, int(n_k[s])).cpu().numpy()
    return out


def bcm_folds_case(e, seed):
    """sgp_bcm_nll_folds over 3 sets; fold 2 is the last 100 of 500 points, so set 2's experts (E = 10) hold its points in
    index order, and a copy of point 0 moved 1e-9 at index 10 shares expert 0: at a 1e-30 Eye term its Cholesky breaks
    down and that slot runs LU."""
    rng = np.random.default_rng(seed)
    fold_of = np.concatenate([rng.integers(0, 2, 400), np.full(100, 2)]).astype(np.int32)
    X = rng.standard_normal((500, 2))
    X[10] = X[0] + 1e-9
    y = np.sin(X.sum(1)) + 0.3 * rng.standard_normal(len(X))
    out = {"experts": e.experts_upload_folds(X, y, fold_of, 3, 40)}
    mk = lambda c: 1.0 * sg.RBFKernel(1.0) + sg.const(c) * sg.EyeKernel()
    v, g = launches(e, out, "call", lambda: e.bcm_nll_folds([2, 0, 2, 1], [mk(1e-2), mk(3e-2), mk(1e-30), mk(2e-2)]))
    out.update(value=v, grad=g, lu=np.array([e.last_bcm_path()]))
    return out


def bcm_slots_case(e, seed):
    """sgp_bcm_nll_slots on a grouped upload with a point 1e-9 from point 0 in expert 0: the 1e-30 slot runs LU."""
    rng = np.random.default_rng(seed)
    X = rng.standard_normal((300, 2))
    y = np.sin(X.sum(1)) + 0.3 * rng.standard_normal(len(X))
    E = e.experts_upload_grouped(X, y, 40)
    X[E], y[E] = X[0] + 1e-9, y[0]
    e.experts_upload_grouped(X, y, 40)
    mk = lambda c: 1.0 * sg.RBFKernel(1.0) + sg.const(c) * sg.EyeKernel()
    out = {}
    v, g = launches(e, out, "call", lambda: e.bcm_nll_slots([mk(1e-2), mk(1e-30), mk(2e-2)]))
    out.update(value=v, grad=g, lu=np.array([e.last_bcm_path()]))
    v, g = launches(e, out, "one", lambda: e.bcm_nll(mk(1e-30)))
    out.update(value_one=np.array([v]), grad_one=g, lu_one=np.array([e.last_bcm_path()]))
    return out


def getters_case(e, seed):
    """Every mode store filled on one grouped upload, then read by every getter, host and device."""
    rng = np.random.default_rng(seed)
    X, y = binary_data(500, 3, rng)
    e.experts_upload_grouped(X, y, 100)
    k = kernel(1, 3, rng)
    out = {}
    launches(e, out, "binary", lambda: e.laplace_nll_any_size(k, 1e-6))
    launches(e, out, "classes", lambda: e.laplace_nll_classes_any_size(2, [1, 0], [k] * 2, 1e-6))
    launches(e, out, "slots", lambda: e.laplace_nll_slots_any_size(3, [2, 0], [1, 1], [k] * 2, 1e-6))
    n = len(X)
    for store, count in ((N.SGP_MODES_BINARY, 1), (N.SGP_MODES_CLASS, 2), (N.SGP_MODES_SLOT, 3)):
        for i in range(count):
            out["host_%d_%d" % (store, i)] = e.experts_modes(store, i, n)
            out["rows_%d_%d" % (store, i)] = launches(e, out, "rows_%d_%d" % (store, i),
                                                      lambda: e.experts_modes_rows(store, i, n)).cpu().numpy()
    return out


def refusal(e, call):
    """(exception type, message, launches made) of a call that is expected to be refused."""
    l0 = e.launch_count()
    try:
        call()
        what = "no error"
    except Exception as exc:                           # noqa: BLE001
        what = "%s: %s" % (type(exc).__name__, exc)
    return {"error": np.frombuffer(what.encode(), dtype=np.uint8), "launches": np.array([e.launch_count() - l0])}


def refusals_case(e, which):
    import torch
    rng = np.random.default_rng(70)
    k = kernel(1, 1, rng)
    if which == "laplace_nll past the on-chip limit":
        X, y = binary_data(600, 1, rng)
        e.experts_upload(*pack_experts(X, y, 150))
        return refusal(e, lambda: e.laplace_nll(k, 1e-6))
    if which == "laplace_nll_classes past the on-chip limit":
        X, y = binary_data(600, 1, rng)
        e.experts_upload(*pack_experts(X, y, 150))
        return refusal(e, lambda: e.laplace_nll_classes(2, [0, 1], [k, k], 1e-6))
    if which == "laplace_nll_any_size on one 75 000-point expert":
        X, y = binary_data(75000, 1, rng)
        e.experts_upload(X, y, [0, 75000])
        return refusal(e, lambda: e.laplace_nll_any_size(k, 1e-6))
    if which == "laplace_nll tol >= 1":
        X, y = binary_data(600, 1, rng)
        e.experts_upload(*pack_experts(X, y, 100))
        return refusal(e, lambda: e.laplace_nll(k, 1.0))
    if which == "fold slots: a set above 46336 points before tol >= 1":
        X, fold_of = fold_data(rng, [50000, 50000], d=1)
        e.experts_upload_folds(X, np.zeros(len(X)), fold_of, 2, 100000)
        return refusal(e, lambda: e.laplace_nll_fold_slots_any_size(1, [0], [0], [0], [k], 1.0))
    if which == "bcm_nll above the LU size limit":
        X = rng.standard_normal((46341, 1))
        e.experts_upload(X, np.sin(X[:, 0]), [0, 46341])
        return refusal(e, lambda: e.bcm_nll(k))
    if which == "bcm_nll_slots with a singular slot":
        e.experts_upload_grouped(np.zeros((200, 2)), rng.standard_normal(200), 50)
        mk = lambda c: 1.0 * sg.RBFKernel(1.0) + sg.const(c) * sg.EyeKernel()
        return refusal(e, lambda: e.bcm_nll_slots([mk(1e-2), mk(0.0), mk(1e-2)]))
    X, y = binary_data(400, 1, rng)
    e.experts_upload(*pack_experts(X, y, 100))
    if which == "get_f_class before any objective call":
        return refusal(e, lambda: e.experts_f_class(0, 400))
    if which == "get_f_slot before any objective call":
        return refusal(e, lambda: e.experts_f_slot(0, 400))
    if which == "get_f_rows_device of an ungrouped upload":
        return refusal(e, lambda: e.experts_modes_rows(N.SGP_MODES_BINARY, 0, 400))
    if which == "get_f_rows_device of an unknown store":
        return refusal(e, lambda: e.experts_modes_rows(7, 0, 400))
    if which == "get_f_fold_slot without a fold upload":
        return refusal(e, lambda: e.experts_f_fold_slot(0, 0, 400))
    X, fold_of = fold_data(rng, [200, 200], d=1)
    e.experts_upload_folds(X, np.zeros(len(X)), fold_of, 2, 100)
    if which == "get_f_fold_slot before any objective call":
        return refusal(e, lambda: e.experts_f_fold_slot(0, 0, 200))
    e.laplace_nll_fold_slots_any_size(2, [0], [1], [0], [k], 1e-6)
    if which == "get_f_fold_rows_device: set outside the folds":
        return refusal(e, lambda: e.experts_f_fold_slot_rows(2, 0, 200))
    if which == "get_f_fold_slot: mode slot outside the store":
        return refusal(e, lambda: e.experts_f_fold_slot(0, 2, 200))
    raise KeyError(which)


REFUSALS = ("laplace_nll past the on-chip limit", "laplace_nll_classes past the on-chip limit",
            "laplace_nll_any_size on one 75 000-point expert", "laplace_nll tol >= 1",
            "fold slots: a set above 46336 points before tol >= 1", "bcm_nll above the LU size limit",
            "bcm_nll_slots with a singular slot", "get_f_class before any objective call",
            "get_f_slot before any objective call", "get_f_rows_device of an ungrouped upload",
            "get_f_rows_device of an unknown store", "get_f_fold_slot without a fold upload",
            "get_f_fold_slot before any objective call", "get_f_fold_rows_device: set outside the folds",
            "get_f_fold_slot: mode slot outside the store")


def greedy_case(e, n_terms, seed):
    rng = np.random.default_rng(seed)
    X = rng.random((4000, 5))
    y = np.sin(X.sum(1)) + 0.1 * rng.standard_normal(len(X))
    return dict(indices=e.greedy_active_set(kernel(n_terms, 5, rng), X, y, 40, 7, 60))


def cases():
    out = []
    for t in range(1, 5):
        for prec, name in ((N.SGP_PREC_F64, "F64"), (N.SGP_PREC_F64_STRICT, "F64_STRICT"), (N.SGP_PREC_I8_DIRECT, "I8_DIRECT")):
            out.append(("stats %s %d terms d=5" % (name, t), lambda e, t=t, p=prec: stats_case(e, t, 5, 300, 20000, p, t)))
    out.append(("stats F64 1 term d=40 (generic loop)", lambda e: stats_case(e, 1, 40, 200, 20000, N.SGP_PREC_F64, 5)))
    out.append(("stats I8 1 term d=16", lambda e: stats_case(e, 1, 16, 500, 70000, N.SGP_PREC_I8, 6)))
    out.append(("tail eigenvalue + LU path", lambda e: lu_tail_case(e, 7)))
    for t, n_e, label in ((1, 100, "register"), (2, 100, "shared memory"), (1, 200, "LU"), (3, 200, "LU")):
        out.append(("bcm_nll %s, %d terms" % (label, t), lambda e, t=t, n_e=n_e: bcm_case(e, t, n_e, 10 + t)))
    for t in (1, 2, 4):
        out.append(("laplace_nll %d terms" % t, lambda e, t=t: laplace_case(e, t, 20 + t)))
        out.append(("greedy_active_set %d terms" % t, lambda e, t=t: greedy_case(e, t, 30 + t)))
    for t in (1, 2):
        out.append(("laplace_nll_any_size global, %d terms" % t, lambda e, t=t: laplace_global_case(e, t, 40 + t)))
        for n_e, label in ((100, "on chip"), (150, "global")):
            out.append(("laplace_nll_classes_any_size %s, %d terms" % (label, t),
                        lambda e, t=t, n_e=n_e: laplace_classes_case(e, t, n_e, 50 + t)))
    for n_e, label in ((100, "on chip"), (150, "global")):
        out.append(("laplace_nll_slots_any_size %s" % label, lambda e, n_e=n_e: laplace_slots_case(e, n_e, 60)))
    out.append(("laplace_nll_fold_slots_any_size 116/117/118", lambda e: laplace_fold_slots_case(e, 61)))
    out.append(("bcm_nll_folds, one slot on LU", lambda e: bcm_folds_case(e, 62)))
    out.append(("bcm_nll_slots, one slot on LU", lambda e: bcm_slots_case(e, 63)))
    out.append(("mode getters, host and device", lambda e: getters_case(e, 64)))
    for which in REFUSALS:
        out.append(("refusal: " + which, lambda e, w=which: refusals_case(e, w)))
    return out


def outcome(run, e):
    """run(e), or the exception it raised, as its one output."""
    try:
        return run(e)
    except Exception as exc:                           # noqa: BLE001
        return {"raised": np.frombuffer(("%s: %s" % (type(exc).__name__, exc)).encode(), dtype=np.uint8)}


def same_bits(a, b):
    a, b = np.ascontiguousarray(a), np.ascontiguousarray(b)
    return a.shape == b.shape and a.dtype == b.dtype and a.tobytes() == b.tobytes()


def card():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                              capture_output=True, text=True).stdout.strip().splitlines()[0]
    except Exception as exc:                           # noqa: BLE001
        return "nvidia-smi unavailable (%s)" % exc


def time_builds(engines, log):
    """Median of 5 synchronised calls per build, the builds alternated call by call."""
    rng = np.random.default_rng(0)
    shapes = [("fp64 stats, pipelined loop: 1 term, 1M x 16, m = 1000", 1, 16, 1000),
              ("fp64 stats, generic loop: 2 terms, 1M x 16, m = 1000", 2, 16, 1000)]
    for label, t, d, m in shapes:
        k, Z = kernel(t, d, rng), rng.random((m, d))
        X = rng.random((1_000_000, d)).astype(np.float32)
        y = np.sin(X.sum(1, dtype=np.float64))
        def step(e):
            e.set_precision(N.SGP_PREC_F64)
            e.begin(k, Z)
            e.accumulate(X, y)
            e.finish()
        alternate(label, engines, step, log)
    k, Z = kernel(1, 16, rng), rng.random((1000, 16))
    v, S = rng.standard_normal(1000), rng.standard_normal((1000, 1000))
    Xt = rng.random((1_000_000, 16))
    for e in engines.values():
        e.begin(k, Z)
        e.set_magic(v, S + S.T)
    alternate("predict mean, 1M x 16, m = 1000", engines, lambda e: e.predict(Xt, with_variance=False), log)
    alternate("predict mean + var, 1M x 16, m = 1000", engines, lambda e: e.predict(Xt), log)
    time_objectives(engines, log)


def time_objectives(engines, log):
    """The per-expert objectives at tools/time_objectives.py's configuration: 10^4 experts of 100 points, d = 16."""
    n, d, n_e = 1_000_000, 16, 100
    rng = np.random.default_rng(3)
    X = rng.random((n, d))
    y = np.sin(X.sum(1)) + 0.1 * rng.standard_normal(n)
    k = 1 * sg.ARDRBFKernel(np.full(d, np.sqrt(18.0 / d))) + sg.const(1) * sg.EyeKernel() + sg.const(1e-4) * sg.EyeKernel()
    pack = pack_experts(X, y, n_e)
    for e in engines.values():
        e.experts_upload(*pack)
    alternate("bcm_nll, 10^4 experts x 100, d = 16", engines, lambda e: e.bcm_nll(k), log)
    yc = np.digitize(y, np.quantile(y, [1 / 3, 2 / 3])).astype(np.float64)
    pack = pack_experts(X, (yc == 1).astype(np.float64), n_e)
    for e in engines.values():
        e.experts_upload(*pack)
    alternate("laplace_nll_any_size, 10^4 experts x 100, d = 16", engines, lambda e: e.laplace_nll_any_size(k, 1e-6), log)
    pack = pack_experts(X, yc, n_e)
    for e in engines.values():
        e.experts_upload(*pack)
    alternate("laplace_nll_classes_any_size C = 3, 10^4 x 100", engines,
              lambda e: e.laplace_nll_classes_any_size(3, [0, 1, 2], [k] * 3, 1e-6), log)
    fold_of = (np.arange(n) % 10).astype(np.int32)
    for e in engines.values():
        e.experts_upload_folds(X, (yc == 1).astype(np.float64), fold_of, 10, n_e)
    alternate("laplace_nll_fold_slots_any_size K = 10, 9 * 10^3 x 100", engines,
              lambda e: e.laplace_nll_fold_slots_any_size(10, list(range(10)), list(range(10)), [1] * 10, [k] * 10, 1e-6),
              log)


def alternate(label, engines, step, log):
    ts = {name: [] for name in engines}
    for name, e in engines.items():
        step(e)
    for _ in range(5):
        for name, e in engines.items():
            t0 = time.perf_counter()
            step(e)
            e.sync()
            ts[name].append(time.perf_counter() - t0)
    log("  %-56s %s" % (label, "  ".join("%s %8.2f ms (%.2f-%.2f)" % (n, 1e3 * np.median(v), 1e3 * min(v), 1e3 * max(v))
                                          for n, v in ts.items())))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--lib", required=True, help="the other libsgp.so")
    ap.add_argument("--time", action="store_true")
    ap.add_argument("--out", help="directory for the report")
    a = ap.parse_args()
    lines = []
    def log(s):
        print(s)
        sys.stdout.flush()
        lines.append(s)
    log("card: %s" % card())
    engines = {"this": ProjectedProcessEngine(0), "other": engine_on(load_lib(a.lib))}
    differ = 0
    for label, run in cases():
        outs = {name: outcome(run, e) for name, e in engines.items()}
        keys = sorted(set(outs["this"]) | set(outs["other"]))
        bad = [k for k in keys if k not in outs["this"] or k not in outs["other"] or not same_bits(outs["this"][k], outs["other"][k])]
        differ += bool(bad)
        log("%-44s %s" % (label, "identical (%s)" % ", ".join(keys) if not bad else "DIFFERS in " + ", ".join(bad)))
    log("%d of %d cases differ" % (differ, len(cases())))
    if a.time:
        time_builds(engines, log)
    for e in engines.values():
        e.close()
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        with open(os.path.join(a.out, "compare_builds.txt"), "w") as f:
            f.write("\n".join(lines) + "\n")
    sys.exit(1 if differ else 0)


if __name__ == "__main__":
    main()
