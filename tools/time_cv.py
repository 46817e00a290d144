"""CrossValidator.fit against the K x P independent fit + predict + metric loop it replaces, in the same process: wall
time, optimisation rounds against summed evaluations, objective launches (sgp_launch_count over the hyper-parameter
optimisation, uploads excluded), avgMetrics, and a check that both ways give the same fold models (hyper-parameters and
validation predictions, bit for bit) and the same avgMetrics.  Both ways end with the refit of the best map on all rows.

  python tools/time_cv.py [--reps 3] [--out DIR]

Shapes:
  airfoil    regression/examples/Airfoil.scala's configuration on tests/golden/airfoil_cv_case.npz (1503 rows, its
             10-fold split): datasetSizeForExpert 100, activeSetSize 1000, 1*ARDRBFKernel(5) + 1.const*EyeKernel,
             sigma2 1e-4, default maxIter (100)
  synthetics regression/examples/Synthetics.scala's recipe (2000 points of sin(x) + N(0, 0.01)), 10 folds,
             datasetSizeForExpert 100, activeSetSize 100, the K-means provider on the GPU, seed 13, sigma2 1e-3
  shard      200 000 x 8 synthetic points, 5 folds x 2 sigma2 values (1e-3, 1e-2), RBFKernel(2.0), datasetSizeForExpert
             100, activeSetSize 500, maxIter 10
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
from spark_gp_b200.regression import KMeansActiveSetProvider   # noqa: E402
from spark_gp_b200.tuning import best_index         # noqa: E402
from spark_gp_b200.utils import kfold_assignment    # noqa: E402


def card():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                              capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
    except Exception as exc:                        # noqa: BLE001
        return "nvidia-smi unavailable (%s)" % exc


def airfoil():
    z = np.load(os.path.join(ROOT, "tests", "golden", "airfoil_cv_case.npz"))
    gp = (sg.GaussianProcessRegression().setDatasetSizeForExpert(100).setActiveSetSize(1000).setSigma2(1e-4)
          .setKernel(lambda: 1 * sg.ARDRBFKernel(5) + sg.const(1.0) * sg.EyeKernel()))
    return z["X"], z["y"], z["fold_of"].astype(np.int32), 10, gp, [{}]


def synthetics():
    rng = np.random.default_rng(13)
    X = np.linspace(0, 1, 2000)[:, None]
    y = np.sin(X[:, 0]) + np.sqrt(0.01) * rng.standard_normal(2000)
    gp = (sg.GaussianProcessRegression()
          .setKernel(lambda: 1 * sg.RBFKernel(0.1, 1e-6, 10) + sg.WhiteNoiseKernel(0.5, 0, 1))
          .setDatasetSizeForExpert(100).setActiveSetProvider(KMeansActiveSetProvider(on_gpu=True))
          .setActiveSetSize(100).setSeed(13).setSigma2(1e-3))
    return X, y, kfold_assignment(len(X), 10, 13), 10, gp, [{}]


def shard(n=200_000, d=8):
    rng = np.random.default_rng(20)
    X = rng.standard_normal((n, d))
    y = np.sin(X[:, 0]) + 0.5 * X[:, 1] * X[:, 2] + 0.1 * rng.standard_normal(n)
    gp = (sg.GaussianProcessRegression().setDatasetSizeForExpert(100).setActiveSetSize(500).setMaxIter(10)
          .setKernel(lambda: sg.RBFKernel(2.0)))
    return X, y, kfold_assignment(n, 5, 3), 5, gp, sg.ParamGridBuilder().addGrid("sigma2", [1e-3, 1e-2]).build()


def cross_validate(X, y, folds, K, gp, maps):
    t = time.perf_counter()
    cv = sg.CrossValidator().setEstimator(gp).setEstimatorParamMaps(maps).setNumFolds(K)
    model = cv.fit(X, y, folds=folds)
    wall = time.perf_counter() - t
    groups = model.last_objective["groups"]
    out = {pk: (f["theta"], f["prediction"]) for pk, f in cv.last_folds.items()}
    return (wall, out, model.avgMetrics, sum(g["rounds"] for g in groups), sum(g["launches"] for g in groups),
            model.bestModel.hyperparameters)


def independent(X, y, folds, K, gp, maps):
    t = time.perf_counter()
    ev = sg.RegressionEvaluator()
    out, avg, evaluations, launches = {}, [], 0, 0
    for p, m in enumerate(maps):
        metrics = []
        for k in range(K):
            tr, va = folds != k, folds == k
            g = gp.copy(m)
            model = g.fit(X[tr], y[tr])
            pred = model.predict(X[va])
            out[p, k] = (model.hyperparameters, pred)
            metrics.append(ev.evaluate(y[va], pred))
            evaluations += g.last_objective["evaluations"]
            launches += g.last_objective["launches"]
            del model
        avg.append(sum(metrics) / K)
    best = gp.copy(maps[best_index(avg, ev.isLargerBetter())]).fit(X, y)
    wall = time.perf_counter() - t
    return wall, out, avg, evaluations, launches, best.hyperparameters


def run(name, data, reps):
    X, y, folds, K, gp, maps = data
    cv_t, ind_t = [], []
    for _ in range(reps):
        c = cross_validate(X, y, folds, K, gp, maps)
        i = independent(X, y, folds, K, gp, maps)
        for pk in i[1]:
            assert np.array_equal(c[1][pk][0], i[1][pk][0]), ("hyper-parameters differ", pk)
            assert np.array_equal(c[1][pk][1], i[1][pk][1]), ("validation predictions differ", pk)
        assert c[2] == i[2], "avgMetrics differ"
        assert np.array_equal(c[5], i[5]), "best models differ"
        cv_t.append(c[0])
        ind_t.append(i[0])
    res = dict(shape=name, n=len(X), d=X.shape[1], folds=K, maps=len(maps), cv_s=float(np.median(cv_t)),
               independent_s=float(np.median(ind_t)), speedup=float(np.median(ind_t) / np.median(cv_t)),
               cv_rounds=c[3], independent_evaluations=i[3], cv_launches=c[4], independent_launches=i[4],
               avgMetrics=c[2], identical_outputs=True)
    print(json.dumps(res), flush=True)
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--out", help="directory for the report")
    a = ap.parse_args()
    report = dict(card=card(), results=[run("airfoil", airfoil(), a.reps), run("synthetics", synthetics(), a.reps),
                                        run("shard", shard(), a.reps)])
    print("card:", report["card"])
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        with open(os.path.join(a.out, "time_cv.json"), "w") as fh:
            json.dump(report, fh, indent=1)


if __name__ == "__main__":
    main()
