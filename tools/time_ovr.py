"""One-vs-rest fit against C independent binary fits, in the same process: wall time, optimisation rounds, objective
launches (sgp_launch_count over the hyper-parameter optimisation), held-out accuracy, and a check that both ways give
the same models (hyper-parameters and raw test predictions, bit for bit).

  python tools/time_ovr.py [--reps 3] [--out DIR]

Shapes:
  iris       classification/examples/Iris.scala: the reference's iris.csv (tests/golden/iris_case.npz split), C = 3,
             datasetSizeForExpert 20, activeSetSize 30, default maxIter (100)
  synthetic  a 10-class shard, 200 000 x 8 (+ 20 000 held out), datasetSizeForExpert 100, activeSetSize 500, maxIter 10,
             RBFKernel(2.0), sigma2 1
The two ways alternate; each time is the median of --reps runs."""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import spark_gp_b200 as sg                          # noqa: E402


def card():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                              capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
    except Exception as exc:                        # noqa: BLE001
        return "nvidia-smi unavailable (%s)" % exc


def iris():
    c = np.load(os.path.join(ROOT, "tests", "golden", "iris_case.npz"))
    tr, te = c["train_idx"], c["test_idx"]
    gp = lambda: sg.GaussianProcessClassifier().setDatasetSizeForExpert(20).setActiveSetSize(30)
    return c["X"][tr], c["y"][tr], c["X"][te], c["y"][te], gp


def synthetic(n=200_000, n_test=20_000, d=8, C=10):
    rng = np.random.default_rng(10)
    centres = 1.5 * rng.standard_normal((C, d))
    lab = rng.integers(0, C, n + n_test)
    X = centres[lab] + rng.standard_normal((n + n_test, d))
    y = lab.astype(np.float64)
    # sigma2 = 1: at the default 1e-3 the tail (sgp_magic) refused a class of this shard as not positive definite
    gp = lambda: (sg.GaussianProcessClassifier().setDatasetSizeForExpert(100).setActiveSetSize(500).setMaxIter(10)
                  .setKernel(lambda: sg.RBFKernel(2.0)).setSigma2(1.0))
    return X[:n], y[:n], X[n:], y[n:], gp


def fit_ovr(X, y, Xte, gp):
    t = time.perf_counter()
    ovr = sg.OneVsRest().setClassifier(gp())
    model = ovr.fit(X, y)
    wall = time.perf_counter() - t
    raw = model.predictRaw(Xte)
    thetas = np.array([m.hyperparameters for m in model.models])
    return wall, raw, thetas, ovr.last_objective["rounds"], ovr.last_objective["launches"]


def fit_binary(X, y, Xte, gp, C):
    t = time.perf_counter()
    models, rounds, launches = [], 0, 0
    for c in range(C):
        g = gp()
        models.append(g.fit(X, (y == c).astype(np.float64)))
        rounds += g.last_objective["evaluations"]
        launches += g.last_objective["launches"]
    wall = time.perf_counter() - t
    raw = np.stack([m.predictRaw(Xte)[:, 1] for m in models], axis=-1)
    thetas = np.array([m.hyperparameters for m in models])
    return wall, raw, thetas, rounds, launches


def run(name, data, reps):
    X, y, Xte, yte, gp = data
    C = int(y.max()) + 1
    ovr_t, bin_t = [], []
    for _ in range(reps):
        o = fit_ovr(X, y, Xte, gp)
        b = fit_binary(X, y, Xte, gp, C)
        assert np.array_equal(o[2], b[2]), "hyper-parameters differ"
        assert np.array_equal(o[1], b[1]), "raw predictions differ"
        ovr_t.append(o[0])
        bin_t.append(b[0])
    acc = float(np.mean(np.argmax(o[1], axis=1) == yte))
    res = dict(shape=name, n=len(X), d=X.shape[1], classes=C, ovr_s=float(np.median(ovr_t)),
               binary_s=float(np.median(bin_t)), speedup=float(np.median(bin_t) / np.median(ovr_t)),
               ovr_rounds=o[3], binary_evaluations=b[3], ovr_launches=o[4], binary_launches=b[4],
               heldout_accuracy=acc, identical_outputs=True)
    print(json.dumps(res))
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--out", help="directory for the report")
    a = ap.parse_args()
    report = dict(card=card(), results=[run("iris", iris(), a.reps), run("synthetic", synthetic(), a.reps)])
    print("card:", report["card"])
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        with open(os.path.join(a.out, "time_ovr.json"), "w") as fh:
            json.dump(report, fh, indent=1)


if __name__ == "__main__":
    main()
