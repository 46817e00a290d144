"""Times kernel evaluation through the device entry (`sgp_kernel_eval_device`) with CUDA events on the library's stream.

  python tools/time_kernel_eval.py [--reps 7] [--out DIR]

Workloads (inputs and outputs are CUDA tensors, so no PCIe copy is timed):
  cross_1M    crossKernel of 1M x 16 points against m = 1000: 8 GB of fp64 out;
  deriv_4000  trainingKernelAndDerivative of 4000 x 16 points: K and 16 derivatives, 17 matrices of 4000 x 4000;
  mnist68     crossKernel at the mnist68 shape, 11 769 x 784 against m = 500;
all with the kernel ARDRBFKernel(beta) + const(0.01) * EyeKernel.
Each time is the median of --reps calls after one warm-up call, between two events recorded on the context's stream.
Beside it: the HBM-store bound, (1 + h) n m 8 bytes over the data-sheet 3.35 TB/s (H100 SXM, 700 W), and the fp64
CUDA-core bound, the 2 fp64 operations per element and dimension (fma of the difference, fma of its square) over
34 TFLOP/s; the larger of the two is the floor the kernel is compared with.  The card's name and power limit are printed
with the numbers.  --out writes the results as JSON."""
from __future__ import annotations

import argparse
import ctypes as C
import json
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import torch                                        # noqa: E402

import spark_gp_b200 as sg                          # noqa: E402
from spark_gp_b200 import _native as N              # noqa: E402

PEAK_HBM, PEAK_FP64 = 3.35e12, 34e12


def card():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                              capture_output=True, text=True, check=True).stdout.strip()
    except (OSError, subprocess.CalledProcessError):
        return "unknown"


def time_call(eng, kernel, A, B, derivatives, reps):
    """Median ms of one sgp_kernel_eval_device call, events on the library's stream."""
    n, d = A.shape
    m = n if B is None else B.shape[0]
    desc, arr, nh, keep = eng._descriptors(kernel, d)
    K = torch.empty((n, m), dtype=torch.float64, device=A.device)
    dK = torch.empty((nh, n, m), dtype=torch.float64, device=A.device) if derivatives else None
    mode = N.SGP_KEVAL_TRAINING if B is None else N.SGP_KEVAL_CROSS
    ptr = lambda t: C.c_void_p(t.data_ptr())

    def call():
        eng._check(eng._lib.sgp_kernel_eval_device(eng._h, C.byref(desc), arr, nh, ptr(A), int(A.dtype == torch.float32),
                                                   n, None if B is None else ptr(B), m, d, mode, ptr(K),
                                                   ptr(dK) if derivatives else None))
    call()
    eng.sync()
    times = []
    for _ in range(reps):
        eng.event_record(0)
        call()
        eng.event_record(1)
        eng.sync()
        times.append(eng.event_elapsed_ms(0, 1))
    del keep
    return float(np.median(times)), (1 + (nh if derivatives else 0)), times


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=7)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    torch.manual_seed(0)
    dev = torch.device("cuda:0")
    workloads = [("cross_1M", 1_000_000, 16, 1000, False), ("deriv_4000", 4000, 16, None, True),
                 ("mnist68", 11_769, 784, 500, False)]
    eng = sg.ProjectedProcessEngine(0)
    info = card()
    print("card: %s" % info)
    results = []
    for name, n, d, m, deriv in workloads:
        beta = torch.full((d,), np.sqrt(4.0 / d), dtype=torch.float64).numpy()
        kernel = sg.ARDRBFKernel(beta) + sg.const(1e-2) * sg.EyeKernel()
        A = torch.rand((n, d), dtype=torch.float64, device=dev)
        B = None if m is None else torch.rand((m, d), dtype=torch.float64, device=dev)
        cols = n if m is None else m
        ms, mats, times = time_call(eng, kernel, A, B, deriv, args.reps)
        store = mats * n * cols * 8 / PEAK_HBM * 1e3
        flops = 2.0 * n * cols * d / PEAK_FP64 * 1e3
        bound = max(store, flops)
        r = dict(workload=name, n=n, d=d, m=cols, matrices=mats, ms=ms, runs_ms=times, hbm_store_bound_ms=store,
                 fp64_bound_ms=flops, share_of_bound=bound / ms, binds="HBM store" if store >= flops else "fp64",
                 card=info)
        results.append(r)
        print("%-10s n=%-8d d=%-4d m=%-5d matrices=%-3d %9.3f ms   HBM-store bound %8.3f ms   fp64 bound %8.3f ms   "
              "%.0f%% of the larger" % (name, n, d, cols, mats, ms, store, flops, 100 * bound / ms))
        del A, B
        torch.cuda.empty_cache()
    eng.close()
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "time_kernel_eval.json"), "w") as f:
            json.dump(results, f, indent=1)


if __name__ == "__main__":
    main()
