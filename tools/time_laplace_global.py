"""Times the Laplace objective across the on-chip / global-memory boundary (`sgp_laplace_nll_any_size`).

  python tools/time_laplace_global.py [--out DIR] [--reps R]

For each case: the time of one evaluation from zero modes (fresh upload) and of a warm one (the next evaluation, at the
same theta), median of R synchronised calls; which kernel ran; and, on the global path, the CTAs launched against the
SM count (min(E, resident CTAs, 4 GiB / workspace per CTA)).  Cases:
  - the mnist68 rows of tests/golden/mnist68_case.npz (1500 x 784, RBFKernel(10) + 1e-3 Eye) at n_e = 100 (on chip),
    117, 118, 200, 500 and 1000;
  - a 200 000 x 8 shard (seeded) at n_e = 200 and 500;
  - held-out accuracy of GaussianProcessClassifier at fixed theta on a fixed 80/20 split of the mnist68 rows, n_e = 100
    and 500.
Prints the card's name and power limit beside the numbers.  Needs a GPU; there is no CPU fallback."""
from __future__ import annotations

import argparse
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import spark_gp_b200 as sg                           # noqa: E402
from spark_gp_b200.regression import ExplicitActiveSetProvider   # noqa: E402

LAPLACE_GLOBAL_CAP = 4 << 30


def card():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                              capture_output=True, text=True, timeout=60).stdout.strip()
    except Exception as e:                            # noqa: BLE001
        return "unknown (%s)" % e


def cta_bytes(n_max):
    ld = (n_max + 31) // 32 * 32
    return 8 * ld * (2 * ld + 44)


def time_case(eng, X, y, n_e, kernel, tol, reps):
    cold, warm = [], []
    for _ in range(reps):
        eng.experts_upload_grouped(X, y, n_e)
        t0 = time.perf_counter(); eng.laplace_nll_any_size(kernel, tol); cold.append(time.perf_counter() - t0)
        t0 = time.perf_counter(); eng.laplace_nll_any_size(kernel, tol); warm.append(time.perf_counter() - t0)
    E = int(np.floor(len(X) / n_e + 0.5))
    n_max = -(-len(X) // E)
    return np.median(cold), np.median(warm), eng.last_laplace_path(), E, n_max


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=None)
    ap.add_argument("--reps", type=int, default=3)
    a = ap.parse_args()
    lines = ["card: " + card()]
    eng = sg.ProjectedProcessEngine(0)
    import torch
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    c = np.load(os.path.join(ROOT, "tests", "golden", "mnist68_case.npz"))
    n = int(c["n_rows"])
    X = (c["pixels"].astype(np.float64) - c["mean"]) / c["std"]
    y = c["y01"].astype(np.float64)
    sigma, sigma2 = float(c["sigma"]), float(c["sigma2"])
    kern = sg.RBFKernel(sigma) + sg.const(sigma2) * sg.EyeKernel()
    eng.experts_upload_grouped(X[:n], y[:n], 100)
    eng.laplace_nll_any_size(kern, 1e-3)                  # warm-up: module load
    for n_e in (100, 117, 118, 200, 500, 1000):
        cold, warm, path, E, n_max = time_case(eng, X[:n], y[:n], n_e, kern, 1e-3, a.reps)
        ctas = min(E, sms, LAPLACE_GLOBAL_CAP // cta_bytes(n_max)) if path == 1 else E
        lines.append("mnist68 %d x 784 n_e=%4d (E=%3d, n_max=%4d) path=%d  zero modes %8.2f ms  warm %8.2f ms  CTAs %d / %d SMs"
                     % (n, n_e, E, n_max, path, cold * 1e3, warm * 1e3, ctas, sms))
        print(lines[-1], flush=True)
    rng = np.random.default_rng(0)
    Xs = rng.standard_normal((200000, 8))
    ys = (np.sin(2 * Xs[:, 0]) + Xs[:, 1:].sum(1) / np.sqrt(7) + 0.3 * rng.standard_normal(len(Xs)) > 0).astype(np.float64)
    ks = 1.2 * sg.ARDRBFKernel(np.full(8, 0.5)) + sg.const(1e-2) * sg.EyeKernel()
    for n_e in (200, 500):
        cold, warm, path, E, n_max = time_case(eng, Xs, ys, n_e, ks, 1e-6, a.reps)
        ctas = min(E, sms, LAPLACE_GLOBAL_CAP // cta_bytes(n_max))
        lines.append("shard 200000 x 8 n_e=%d (E=%d) path=%d  zero modes %8.2f ms  warm %8.2f ms  CTAs %d / %d SMs"
                     % (n_e, E, path, cold * 1e3, warm * 1e3, ctas, sms))
        print(lines[-1], flush=True)
    eng.close()
    split = np.random.default_rng(68).permutation(len(X))
    cut = int(0.8 * len(X))
    tr, te = split[:cut], split[cut:]
    for n_e in (100, 500):
        gp = (sg.GaussianProcessClassifier().setDatasetSizeForExpert(n_e).setActiveSetSize(500).setSigma2(sigma2)
              .setKernel(lambda: sg.RBFKernel(sigma)).setTol(1e-3)
              .setActiveSetProvider(ExplicitActiveSetProvider(X[tr][:500])))
        model = gp.fit(X[tr], y[tr], hyperparameters=np.array([sigma]))
        acc = float(np.mean(model.predict(X[te]) == y[te]))
        lines.append("mnist68 held-out accuracy (80/20 split of %d rows, fixed theta) n_e=%d: %.4f" % (len(X), n_e, acc))
        print(lines[-1], flush=True)
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        with open(os.path.join(a.out, "time_laplace_global.txt"), "w") as f:
            f.write("\n".join(lines) + "\n")


if __name__ == "__main__":
    main()
