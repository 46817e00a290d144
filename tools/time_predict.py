"""Times prediction (`sgp_predict`, `sgp_predict_device`) at the shapes users score at, and compares two builds.

  python tools/time_predict.py [--lib OTHER/libsgp.so] [--dump-outputs DIR] [--profile] [--reps 3]

Per shape (n test points x d features against an active set of m): the host entry mean-only and mean + variance, for this
tree's library and, with --lib, for another build (alternated in the same process, so both see the same card and the
same load), then the device entry with fp32 and fp64 X (this tree's library only: older builds have no device entry).
Times are a host clock around calls that end in a device synchronisation, after one warm-up call per shape and mode; the
median of --reps.  The magic pair is random (v ~ N(0,1), M symmetric): prediction costs do not depend on its values.

Counts from shapes: the triangular quadratic form is n m^2 fp64 tensor-core flops, the kernel elements n m (2d) fp64
CUDA-core flops plus n m exponentials, and K of a variance call goes to HBM once and is read back (2 n m_pad 8 bytes).
Each is printed as a share of the H100 SXM data-sheet bound (fp64 tensor 67 TFLOP/s, fp64 CUDA core 34 TFLOP/s, HBM
3.35 TB/s) over the measured call time (an end-to-end figure: the host leg includes the PCIe copies).
--dump-outputs writes both builds' mean and variance (host entry) and prints the largest difference between them, relative
to the summed magnitudes |k| |v| and selfKernel + |k| |M| |k| on a subset of rows.
--profile runs the device entry once per shape under torch.profiler and prints the kernel times (a separate run: tracing
slows the host).

  python tools/time_predict.py --probability [--reps 5]

times the averaged probability (`sgp_predict_probability`, 100 nodes) against the mean + variance call on the same
model, the two alternating in one process, through the device and the host entry, at 1M x 16 / m = 1000 and at the
11769 x 784 / m = 500 shape.  The magic pair is scaled so that the variances are O(1) and of both signs, as a fitted
model's are near zero.  It prints the card, the fused reduce kernel's time against the plain one from torch.profiler
(a separate traced call), and the largest |p - the library's rule applied in fp64 numpy to the call's own (mean, var)|."""
from __future__ import annotations

import argparse
import ctypes as C
import os
import re
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import spark_gp_b200 as sg                          # noqa: E402
from spark_gp_b200 import _native as N              # noqa: E402
from spark_gp_b200.engine import ProjectedProcessEngine   # noqa: E402

SHAPES = [(1_000_000, 16, 1000), (1_000_000, 32, 2000), (262_144, 8, 4000), (11_769, 784, 500)]
PEAK_DMMA, PEAK_FP64, PEAK_HBM = 67e12, 34e12, 3.35e12


def load_other(path):
    """A libsgp.so of another build, bound for the calls this tool makes (an older build may lack newer symbols)."""
    lib = C.CDLL(path)
    vp, i32, i64 = C.c_void_p, C.c_int32, C.c_int64
    lib.sgp_ctx_create.argtypes = [C.POINTER(vp), C.c_int]
    lib.sgp_ctx_destroy.argtypes = [vp]
    lib.sgp_last_error.argtypes = [vp]
    lib.sgp_last_error.restype = C.c_char_p
    lib.sgp_set_precision.argtypes = [vp, C.c_int]
    lib.sgp_stats_begin.argtypes = [vp, C.POINTER(N.KernelDesc), vp, i32, i32]
    lib.sgp_set_magic.argtypes = [vp, vp, vp]
    lib.sgp_predict.argtypes = [vp, vp, i64, vp, vp]
    for name in ("sgp_ctx_create", "sgp_ctx_destroy", "sgp_set_precision", "sgp_stats_begin", "sgp_set_magic", "sgp_predict"):
        getattr(lib, name).restype = C.c_int
    return lib


def engine_on(lib):
    e = ProjectedProcessEngine.__new__(ProjectedProcessEngine)
    e._lib, e._h, e.m, e.d, e._device, e._has_comm = lib, C.c_void_p(), 0, 0, 0, False
    if lib.sgp_ctx_create(C.byref(e._h), 0) != N.SGP_OK:
        raise RuntimeError("sgp_ctx_create failed: %s" % lib.sgp_last_error(None).decode())
    return e


def card():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                              capture_output=True, text=True).stdout.strip().splitlines()[0]
    except Exception as exc:                           # noqa: BLE001
        return "nvidia-smi unavailable (%s)" % exc


def timed(fn, reps):
    fn()
    ts = []
    for _ in range(reps):
        t0 = time.perf_counter()
        fn()
        ts.append(time.perf_counter() - t0)
    return float(np.median(ts))


def case(n, d, m, seed=0):
    rng = np.random.default_rng(seed)
    beta = (0.5 + rng.random(d)) / np.sqrt(d)
    kernel = 1.0 * sg.ARDRBFKernel(beta) + sg.const(1e-3) * sg.EyeKernel()
    Z = rng.random((m, d))
    S = rng.standard_normal((m, m))
    return dict(kernel=kernel, beta=beta, Z=Z, v=rng.standard_normal(m), M=(S + S.T) * 10.0,
                X=rng.random((n, d)), n=n, d=d, m=m)


def summed_magnitudes(c, rows):
    X, Z = c["X"][rows] * c["beta"], c["Z"] * c["beta"]
    q = (X * X).sum(1)[:, None] + (Z * Z).sum(1)[None, :] - 2.0 * X @ Z.T    # magnitudes only: the expansion is enough
    A = np.exp(-np.maximum(q, 0.0))
    return A @ np.abs(c["v"]), 1.0 + 1e-3 + np.einsum("ti,ti->t", A @ np.abs(c["M"]), A)


def report(label, n, d, m, t, var):
    m_pad = (m + 127) // 128 * 128
    dmma = n * m * m if var else 0.0
    elem = 2.0 * n * m * d
    kbytes = 2.0 * n * m_pad * 8 if var else 0.0
    print("  %-26s %9.2f ms   dmma %5.1f%%  fp64 %5.1f%%  hbm(K) %5.1f%%   (%.2e dmma flop, %.2e elem flop, %.2e exp, "
          "%.2e B)" % (label, t * 1e3, 100 * dmma / PEAK_DMMA / t, 100 * elem / PEAK_FP64 / t, 100 * kbytes / PEAK_HBM / t,
                       dmma, elem, n * m, kbytes))


def host_rule_probability(mean, var, nodes):
    """The library's rule applied in fp64 numpy: (1/sqrt(pi)) sum_i w_i sigmoid(mean + sqrt(2 max(var, 0)) x_i)."""
    x, w = ProjectedProcessEngine.gauss_hermite_rule(nodes)
    out = np.empty(len(mean))
    for s in range(0, len(mean), 65536):
        mu, v = mean[s:s + 65536], var[s:s + 65536]
        z = mu[:, None] + np.sqrt(2.0 * np.where(v < 0.0, 0.0, v))[:, None] * x
        with np.errstate(over="ignore"):
            out[s:s + 65536] = (1.0 / (1.0 + np.exp(-z))) @ w / np.sqrt(np.pi)
    return out


def probability(eng, reps, nodes=100):
    import torch
    from torch.profiler import ProfilerActivity, profile
    for si in (0, 3):
        n, d, m = SHAPES[si]
        c = case(n, d, m, seed=si)
        eng.begin(c["kernel"], c["Z"])
        eng.set_magic(c["v"], c["M"] * 1e-4)
        Xd = torch.from_numpy(c["X"]).to(device="cuda")
        torch.cuda.synchronize()
        print("n=%d d=%d m=%d, %d nodes" % (n, d, m, nodes))
        calls = {
            "device mean+var": lambda: eng.predict_tensor(Xd, with_variance=True),
            "device probability": lambda: eng.predict_probability_tensor(Xd, nodes=nodes),
            "host mean+var": lambda: eng.predict(c["X"], with_variance=True),
            "host probability": lambda: eng.predict_probability(c["X"], nodes=nodes),
        }
        for f in calls.values():
            f()
        ts = {k: [] for k in calls}
        for _ in range(reps):                               # alternate, so that both see the same load
            for k, f in calls.items():
                t0 = time.perf_counter()
                f()
                ts[k].append(time.perf_counter() - t0)
        for entry in ("device", "host"):
            mv, pr = np.median(ts[entry + " mean+var"]), np.median(ts[entry + " probability"])
            print("  %-7s mean+var %9.3f ms   probability %9.3f ms   difference %+8.3f ms (%+.1f %%)   spread: %s / %s" % (
                entry, mv * 1e3, pr * 1e3, (pr - mv) * 1e3, 100 * (pr - mv) / mv,
                " ".join("%.2f" % (t * 1e3) for t in ts[entry + " mean+var"]),
                " ".join("%.2f" % (t * 1e3) for t in ts[entry + " probability"])))
        for label, f in (("mean+var", calls["device mean+var"]), ("probability", calls["device probability"])):
            with profile(activities=[ProfilerActivity.CUDA]) as prof:
                f()
            for ev in prof.key_averages():
                name = re.search(r"(predict_\w+|pack_magic_kernel)(<\w+>)?", ev.key)
                if name:
                    print("    %-12s kernel %-36s %9.3f ms x %d" % (label, name.group(0), ev.device_time_total / 1e3,
                                                                  ev.count))
        p, mean, var = eng.predict_probability(c["X"], nodes=nodes, with_mean_var=True)
        hm, hv = eng.predict(c["X"])
        ref = host_rule_probability(mean, var, nodes)
        print("  mean / var equal to sgp_predict's: %s / %s;  variances < 0: %.1f %%;  max |p - host rule| = %.2e" % (
            np.array_equal(mean, hm), np.array_equal(var, hv), 100 * np.mean(var < 0), np.abs(p - ref).max()))
        del Xd
        sys.stdout.flush()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--lib", help="another libsgp.so (e.g. the parent commit's build) to time against")
    ap.add_argument("--dump-outputs", help="directory for both builds' outputs")
    ap.add_argument("--profile", action="store_true")
    ap.add_argument("--probability", action="store_true", help="time the averaged probability (see above)")
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--shapes", default="0,1,2,3", help="indices into SHAPES")
    a = ap.parse_args()
    import torch
    print("card: %s" % card())
    if a.probability:
        eng = ProjectedProcessEngine(0)
        probability(eng, a.reps)
        eng.close()
        return
    new = ProjectedProcessEngine(0)
    old = engine_on(load_other(a.lib)) if a.lib else None
    for si in [int(s) for s in a.shapes.split(",")]:
        n, d, m = SHAPES[si]
        c = case(n, d, m, seed=si)
        print("n=%d d=%d m=%d" % (n, d, m))
        outs = {}
        for with_var in (False, True):
            for name, e in [("new", new)] + ([("old", old)] if old else []):
                e.begin(c["kernel"], c["Z"])
                e.set_magic(c["v"], c["M"])
                t = timed(lambda: outs.__setitem__((name, with_var), e.predict(c["X"], with_variance=with_var)), a.reps)
                report("%s host %s" % (name, "mean+var" if with_var else "mean"), n, d, m, t, with_var)
        new.begin(c["kernel"], c["Z"])
        new.set_magic(c["v"], c["M"])
        for dt in (torch.float32, torch.float64):
            Xd = torch.from_numpy(c["X"]).to(device="cuda", dtype=dt)
            torch.cuda.synchronize()
            for with_var in (False, True):
                t = timed(lambda: new.predict_tensor(Xd, with_variance=with_var), a.reps)
                report("new device %s %s" % (str(dt).split(".")[1], "mean+var" if with_var else "mean"), n, d, m, t,
                       with_var)
            if a.profile:
                from torch.profiler import ProfilerActivity, profile
                with profile(activities=[ProfilerActivity.CUDA]) as prof:
                    new.predict_tensor(Xd, with_variance=True)
                for ev in prof.key_averages():
                    if "predict" in ev.key or "pack_magic" in ev.key:
                        print("    kernel %-60s %9.3f ms x %d" % (ev.key[:60], ev.device_time_total / 1e3, ev.count))
            del Xd
        if old:
            rows = np.unique(np.concatenate([[0, n - 1], np.random.default_rng(1).choice(n, min(n, 2000), replace=False)]))
            sm, sv = summed_magnitudes(c, rows)
            nm, nv = outs[("new", True)]
            om, ov = outs[("old", True)]
            em = float((np.abs(nm[rows] - om[rows]) / np.maximum(sm, 1e-300)).max())
            ev = float((np.abs(nv[rows] - ov[rows]) / sv).max())
            print("  new vs old (host, mean+var, %d rows): mean %.2e, var %.2e of the summed magnitudes; "
                  "all rows: max |dmean| / max|mean| %.2e, max |dvar| / max|var| %.2e" % (
                      len(rows), em, ev, np.abs(nm - om).max() / np.abs(om).max(), np.abs(nv - ov).max() / np.abs(ov).max()))
            if a.dump_outputs:
                os.makedirs(a.dump_outputs, exist_ok=True)
                np.savez(os.path.join(a.dump_outputs, "predict_%d_%d_%d.npz" % (n, d, m)), new_mean=nm, new_var=nv,
                         old_mean=om, old_var=ov)
        sys.stdout.flush()
    new.close()
    if old:
        old.close()


if __name__ == "__main__":
    main()
