"""GPU timing of the K-means active-set provider (`sgp_kmeans`, csrc/kmeans.cu) at the benchmark's shapes, beside the
scikit-learn provider on the same machine.  Run on an H100 from the repository root:

    python tools/time_kmeans.py [--out DIR] [--skip-sklearn]          (--out DIR: also write DIR/time_kmeans.json)

Per shape: the k-means|| initialisation (call with max_iter = 0 minus a call from given centres with max_iter = 0), one
Lloyd iteration (20 iterations from given centres with tol = 0, minus max_iter = 0, over 20), the whole provider call
(maxIter = 20), and the assignment kernel's device time per pass (torch.profiler) against the fp32 bound 2 n k d / 67
TFLOP/s.  Host clocks around calls that end in a device synchronise; the card and its power limit are read in the same
run."""
import argparse
import json
import os
import subprocess
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np  # noqa: E402

import spark_gp_b200 as sg  # noqa: E402

SHAPES = [(1_000_000, 16, 1000, "configs[1]"), (1_250_000, 32, 2000, "configs[3] per-GPU shard"),
          (1_000_000, 8, 4000, "k = 4000"), (11769, 784, 500, "mnist68 shape")]
FP32_PEAK = 67e12


def card():
    r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return r.stdout.strip()


def clock(fn, reps=3):
    best = float("inf")
    for _ in range(reps):
        t0 = time.perf_counter()
        fn()
        best = min(best, time.perf_counter() - t0)
    return best


def assign_kernel_ms(eng, X, k, C0):
    import torch
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        eng.kmeans(X, k, max_iter=5, tol=0.0, init_centers=C0)
        torch.cuda.synchronize()
    times = [e.device_time_total if hasattr(e, "device_time_total") else e.cuda_time_total
             for e in prof.key_averages() if "kmeans_assign_kernel" in e.key]
    counts = [e.count for e in prof.key_averages() if "kmeans_assign_kernel" in e.key]
    return (sum(times) / 1e3 / sum(counts)) if counts else float("nan")


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=None, help="directory for time_kmeans.json (default: print only)")
    ap.add_argument("--skip-sklearn", action="store_true")
    args = ap.parse_args()
    info = card()
    print("card:", info, flush=True)
    eng = sg.ProjectedProcessEngine(0)
    rng = np.random.default_rng(0)
    eng.kmeans(rng.random((4096, 8), dtype=np.float32), 64, max_iter=2)          # module load, first allocations
    rows = []
    for n, d, k, label in SHAPES:
        X = rng.random((n, d), dtype=np.float32)
        C0 = X[:k].astype(np.float64)
        eng.kmeans(X, k, max_iter=1, init_centers=C0)                           # workspaces at this shape
        t_pass0 = clock(lambda: eng.kmeans(X, k, max_iter=0, init_centers=C0))
        t_init = clock(lambda: eng.kmeans(X, k, max_iter=0, seed=1)) - t_pass0
        t_lloyd = (clock(lambda: eng.kmeans(X, k, max_iter=20, tol=0.0, init_centers=C0), reps=2) - t_pass0) / 20
        t_prov = clock(lambda: eng.kmeans(X, k, max_iter=20, tol=1e-4, seed=1), reps=2)
        ms_assign = assign_kernel_ms(eng, X, k, C0)
        bound_ms = 2.0 * n * k * d / FP32_PEAK * 1e3
        row = dict(shape=label, n=n, d=d, k=k, init_s=t_init, lloyd_iter_ms=1e3 * t_lloyd, provider_s=t_prov,
                   assign_ms=ms_assign, fp32_bound_ms=bound_ms, assign_share_of_fp32_peak=bound_ms / ms_assign)
        rows.append(row)
        print("%-26s n=%-8d d=%-4d k=%-5d init %.3f s  Lloyd %.2f ms/iter  provider(maxIter=20) %.3f s  "
              "assign %.3f ms/pass (fp32 bound %.3f ms, %.0f%%)" % (label, n, d, k, t_init, 1e3 * t_lloyd, t_prov,
                                                                   ms_assign, bound_ms, 100 * bound_ms / ms_assign),
              flush=True)
    sk = None
    if not args.skip_sklearn:
        X = np.random.default_rng(1).random((1_000_000, 16), dtype=np.float32)
        prov = sg.KMeansActiveSetProvider(maxIter=20)
        t0 = time.perf_counter()
        prov(1000, X, None, None, None, 0)
        sk = time.perf_counter() - t0
        gpu = sg.KMeansActiveSetProvider(maxIter=20, on_gpu=True)
        gpu(1000, X, None, None, None, 0)
        t_gpu = clock(lambda: gpu(1000, X, None, None, None, 0), reps=2)
        print("provider 1M x 16, k = 1000, maxIter = 20: scikit-learn %.1f s, GPU %.3f s (%.0fx)" % (sk, t_gpu, sk / t_gpu),
              flush=True)
        sk = dict(sklearn_s=sk, gpu_s=t_gpu)
    eng.close()
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "time_kmeans.json"), "w") as f:
            json.dump(dict(card=info, rows=rows, provider_1M_16_k1000=sk), f, indent=1)


if __name__ == "__main__":
    main()
