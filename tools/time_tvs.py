"""TrainValidationSplit.fit against the P independent fit + predict + metric loops it replaces, alternated in one process:
wall time, optimisation rounds against evaluations, objective launches (sgp_launch_count over the optimisation),
validationMetrics, and a check that both ways give the same validation predictions, bit for bit.

  python tools/time_tvs.py [--reps 3] [--out DIR] [--workloads mnist68 ovr10 reg8]

Workloads:
  mnist68    the 1600 rows of tests/golden/mnist68_case.npz (784 features, classification/examples/MNIST.scala's 6-vs-8
             set), binary, RBFKernel(sigma) for sigma in 8, 10, 12, tol 1e-3, datasetSizeForExpert 100, activeSetSize
             100, default maxIter (100), trainRatio 0.8, accuracy
  ovr10      a 10-class one-vs-rest shard, 200 000 x 8, sigma2 in 1, 2, RBFKernel(2.0), datasetSizeForExpert 100,
             activeSetSize 500, maxIter 10 (as tools/time_ovr.py), trainRatio 0.8, f1
  reg8       a regression shard, 200 000 x 8, sigma2 in 0.5, 1, 2, 1.0 * ARDRBFKernel(8), datasetSizeForExpert
             100, activeSetSize 500, maxIter 10, trainRatio 0.8, rmse
Both sides run the whole selection except the refit of the best map on all rows, which is the same call on both.  After
one untimed run of each, each time is the median of --reps runs, the two ways alternated."""
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
from spark_gp_b200.utils import train_validation_assignment   # noqa: E402


def card():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                              capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
    except Exception as exc:                        # noqa: BLE001
        return "nvidia-smi unavailable (%s)" % exc


def mnist68():
    c = np.load(os.path.join(ROOT, "tests", "golden", "mnist68_case.npz"))
    X = (c["pixels"].astype(np.float64) - c["mean"]) / c["std"]
    est = (sg.GaussianProcessClassifier().setDatasetSizeForExpert(100).setActiveSetSize(100)
           .setKernel(lambda: sg.RBFKernel(10.0)).setTol(1e-3))
    maps = sg.ParamGridBuilder().addGrid("kernel", [(lambda s: lambda: sg.RBFKernel(s))(s) for s in (8.0, 10.0, 12.0)]).build()
    return X, c["y01"], est, maps, sg.MulticlassClassificationEvaluator("accuracy")


def ovr10(n=200_000, d=8, C=10):
    rng = np.random.default_rng(10)
    centres = 1.5 * rng.standard_normal((C, d))
    lab = rng.integers(0, C, n)
    X = centres[lab] + rng.standard_normal((n, d))
    gp = (sg.GaussianProcessClassifier().setDatasetSizeForExpert(100).setActiveSetSize(500).setMaxIter(10)
          .setKernel(lambda: sg.RBFKernel(2.0)).setSigma2(1.0))
    maps = sg.ParamGridBuilder().addGrid("sigma2", [1.0, 2.0]).build()
    return X, lab.astype(np.float64), sg.OneVsRest().setClassifier(gp), maps, sg.MulticlassClassificationEvaluator("f1")


def reg8(n=200_000, d=8):
    rng = np.random.default_rng(8)
    X = rng.standard_normal((n, d))
    y = np.sin(X[:, 0]) + 0.5 * X[:, 1] * X[:, 2] + 0.1 * rng.standard_normal(n)
    gp = (sg.GaussianProcessRegression().setDatasetSizeForExpert(100).setActiveSetSize(500).setMaxIter(10)
          .setKernel(lambda: 1.0 * sg.ARDRBFKernel(d)))
    maps = sg.ParamGridBuilder().addGrid("sigma2", [0.5, 1.0, 2.0]).build()
    return X, y, gp, maps, sg.RegressionEvaluator("rmse")


def batched(X, y, est, maps, ev, mask):
    """TrainValidationSplit's selection without the final refit."""
    tvs = sg.TrainValidationSplit().setEstimator(est).setEvaluator(ev).setEstimatorParamMaps(maps)
    ests = [est.copy(m) for m in maps]
    t = time.perf_counter()
    if isinstance(est, sg.GaussianProcessRegression):
        preds, objective = tvs._fit_regression(ests, X, y, mask)
    else:
        preds, _, objective = tvs._fit_classifiers(ests, isinstance(est, sg.OneVsRest), X, y, mask)
    metrics = [ev.evaluate(y[~mask], p) for p in preds]
    wall = time.perf_counter() - t
    g = objective["groups"]
    return wall, preds, metrics, sum(x["rounds"] for x in g), sum(x["launches"] for x in g)


def independent(X, y, est, maps, ev, mask):
    t = time.perf_counter()
    preds, metrics, evaluations, launches = [], [], 0, 0
    for m in maps:
        e = est.copy(m)
        model = e.fit(X[mask], y[mask])
        preds.append(model.predict(X[~mask]))
        metrics.append(ev.evaluate(y[~mask], preds[-1]))
        if isinstance(e, sg.OneVsRest):
            evaluations += e.last_objective["rounds"]
            launches += e.last_objective["launches"]
        else:
            evaluations += e.last_objective["evaluations"]
            launches += e.last_objective["launches"]
        del model
    return time.perf_counter() - t, preds, metrics, evaluations, launches


def run(name, data, reps):
    X, y, est, maps, ev = data
    mask = train_validation_assignment(len(X), 0.8, 0)
    batched(X, y, est, maps, ev, mask)               # warm-up: contexts, modules and workspaces of both ways
    independent(X, y, est, maps, ev, mask)
    bt, it, identical = [], [], True
    for _ in range(reps):
        b = batched(X, y, est, maps, ev, mask)
        i = independent(X, y, est, maps, ev, mask)
        identical &= all(np.array_equal(p, q) for p, q in zip(b[1], i[1])) and b[2] == i[2]
        bt.append(b[0])
        it.append(i[0])
    res = dict(workload=name, n=len(X), d=X.shape[1], maps=len(maps), train_rows=int(mask.sum()),
               tvs_s=float(np.median(bt)), independent_s=float(np.median(it)),
               speedup=float(np.median(it) / np.median(bt)), tvs_rounds=b[3], independent_evaluations=i[3],
               tvs_launches=b[4], independent_launches=i[4], validationMetrics=b[2], identical_outputs=bool(identical))
    print(json.dumps(res))
    sys.stdout.flush()
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--out", help="directory for the report")
    ap.add_argument("--workloads", nargs="+", choices=("mnist68", "ovr10", "reg8"), default=["mnist68", "ovr10", "reg8"])
    a = ap.parse_args()
    report = dict(card=card())
    print("card:", report["card"])
    workloads = dict(mnist68=mnist68, ovr10=ovr10, reg8=reg8)
    report["results"] = [run(name, workloads[name](), a.reps) for name in a.workloads]
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        with open(os.path.join(a.out, "time_tvs.json"), "w") as fh:
            json.dump(report, fh, indent=1)


if __name__ == "__main__":
    main()
