"""Whole `fit` from a CUDA tensor against the same fit from a numpy array (GPU box), alternating in one process.

    python tools/time_fit_device.py [reps=3] [out.json]

Cases: `GaussianProcessRegression.fit` at maxIter = 10 on the benchmark's 1M x 16 fp32 shape, and
`GaussianProcessClassifier.fit` on the mnist68 fixture rows.  Prints the wall time of every fit (host clock around a call
that ends in a device synchronise), whether the two paths gave the same theta bit for bit, and the card's name and power
limit read in the same run."""
import json
import os
import subprocess
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
import torch

import spark_gp_b200 as sg

reps = int(sys.argv[1]) if len(sys.argv) > 1 else 3
out_path = sys.argv[2] if len(sys.argv) > 2 else None
card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"],
                      capture_output=True, text=True).stdout.strip()
print("card: %s" % card, flush=True)


def regression_case():
    n, d, m, n_e = 1_000_000, 16, 1000, 100
    rng = np.random.default_rng(13)
    X = rng.random((n, d), dtype=np.float32)
    y = np.sin(X.astype(np.float64).sum(1)) + 0.1 * rng.standard_normal(n)
    make = lambda: (sg.GaussianProcessRegression()
                    .setKernel(lambda: 1 * sg.ARDRBFKernel(np.full(d, np.sqrt(18.0 / d))) + sg.const(1) * sg.EyeKernel())
                    .setDatasetSizeForExpert(n_e).setActiveSetSize(m).setSigma2(1e-4).setMaxIter(10).setSeed(13))
    return "regression 1M x 16 fp32, maxIter 10", make, X, y


def classifier_case():
    c = np.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), "..", "tests", "golden", "mnist68_case.npz"))
    n = int(c["n_rows"])
    X = (c["pixels"].astype(np.float64) - c["mean"]) / c["std"]
    make = lambda: (sg.GaussianProcessClassifier().setDatasetSizeForExpert(100).setActiveSetSize(100)
                    .setKernel(lambda: sg.RBFKernel(10.0)).setTol(1e-3).setMaxIter(10))
    return "classifier mnist68 rows (%d x 784 fp64), maxIter 10" % n, make, X[:n], c["y01"][:n]


results = []
for name, make, X, y in (regression_case(), classifier_case()):
    dX, dy = torch.as_tensor(X, device="cuda:0"), torch.as_tensor(y, device="cuda:0")
    torch.cuda.synchronize()
    make().fit(X, y)                        # warm-up of both paths: contexts, workspaces, first launches
    make().fit(dX, dy)
    times = {"numpy": [], "cuda": []}
    thetas = {}
    for r in range(reps):
        for kind, args in (("numpy", (X, y)), ("cuda", (dX, dy))):
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            model = make().fit(*args)
            torch.cuda.synchronize()
            times[kind].append(time.perf_counter() - t0)
            thetas[kind] = np.asarray(model.hyperparameters, dtype=np.float64)
            del model
    same = bool(np.array_equal(thetas["numpy"].view(np.int64), thetas["cuda"].view(np.int64)))
    row = dict(case=name, card=card, numpy_s=times["numpy"], cuda_s=times["cuda"], theta_bit_identical=same)
    results.append(row)
    print("%s: numpy %s s, cuda %s s, theta bit-identical: %s"
          % (name, " ".join("%.3f" % t for t in times["numpy"]), " ".join("%.3f" % t for t in times["cuda"]), same),
          flush=True)
if out_path:
    with open(out_path, "w") as f:
        json.dump(results, f, indent=1)
