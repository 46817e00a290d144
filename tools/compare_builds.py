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
    both kernels (values, gradients and every class's modes over two warm-started calls); sgp_greedy_active_set indices.
Outputs are compared as bit patterns.  The script prints one line per case and exits with 1 if any case differs.
--time times the fp64 statistics kernel (both loops) and prediction on both builds, alternated in the same process:
median of 5 synchronised calls after a warm-up, with the card's name and power limit.  --out writes the report there."""
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
    return out


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
        outs = {name: run(e) for name, e in engines.items()}
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
