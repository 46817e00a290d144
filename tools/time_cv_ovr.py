"""CrossValidator.fit over one-vs-rest against the K x P independent OneVsRest.fit + predict + metric loop it replaces, in
the same process: wall time, optimisation rounds against summed evaluations, objective launches (sgp_launch_count over
the hyper-parameter optimisation, uploads excluded; the selector's count includes its call at the optima), avgMetrics, and a check that both ways give the same fold models
(class hyper-parameters and validation predictions, bit for bit) and the same avgMetrics.  Both ways end with the refit of
the best map on all rows.

  python tools/time_cv_ovr.py [--reps 3] [--cases iris,shard] [--out DIR]

Shapes:
  iris   classification/examples/Iris.scala's configuration on the 150 rows of tests/golden/iris_case.npz: 10 folds,
         datasetSizeForExpert 20, activeSetSize 30, the default kernel, accuracy
  shard  tools/time_tvs.py's 10-class 200 000 x 8 shard and classifier (RBFKernel(2.0), datasetSizeForExpert 100,
         activeSetSize 500, maxIter 10), 5 folds x 2 sigma2 values (1, 2), accuracy
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
from spark_gp_b200.tuning import best_index         # noqa: E402
from spark_gp_b200.utils import kfold_assignment    # noqa: E402


def card():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                              capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
    except Exception as e:                          # noqa: BLE001
        return "unknown (%s)" % e


def iris_case():
    c = np.load(os.path.join(ROOT, "tests", "golden", "iris_case.npz"))
    ovr = sg.OneVsRest().setClassifier(sg.GaussianProcessClassifier().setDatasetSizeForExpert(20).setActiveSetSize(30))
    return c["X"], c["y"], ovr, [{}], 10, 0


def shard_case():
    """tools/time_tvs.py's 10-class shard and classifier, with 5 folds."""
    rng = np.random.default_rng(10)
    n, d, C = 200_000, 8, 10
    centres = 1.5 * rng.standard_normal((C, d))
    lab = rng.integers(0, C, n)
    X = centres[lab] + rng.standard_normal((n, d))
    gp = (sg.GaussianProcessClassifier().setDatasetSizeForExpert(100).setActiveSetSize(500).setMaxIter(10)
          .setKernel(lambda: sg.RBFKernel(2.0)).setSigma2(1.0))
    maps = sg.ParamGridBuilder().addGrid("sigma2", [1.0, 2.0]).build()
    return X, lab.astype(np.float64), sg.OneVsRest().setClassifier(gp), maps, 5, 3


def batched(X, y, ovr, maps, K, seed):
    cv = (sg.CrossValidator().setEstimator(ovr).setEvaluator(sg.MulticlassClassificationEvaluator("accuracy"))
          .setEstimatorParamMaps(maps).setNumFolds(K).setSeed(seed))
    model = cv.fit(X, y)
    groups = model.last_objective["groups"]
    return dict(avg=model.avgMetrics, best=model.bestIndex,
                thetas={key: out["theta"] for key, out in cv.last_folds.items()},
                preds={key: out["prediction"] for key, out in cv.last_folds.items()},
                rounds=sum(g["rounds"] for g in groups), launches=sum(g["launches"] for g in groups),
                evaluations=sum(s.get("evaluations", 0) for g in groups for s in g["slots"]))


def independent(X, y, ovr, maps, K, seed):
    fold_of = kfold_assignment(len(X), K, seed)
    ev = sg.MulticlassClassificationEvaluator("accuracy")
    thetas, preds, metrics, launches, evaluations = {}, {}, np.empty((len(maps), K)), 0, 0
    for p, m in enumerate(maps):
        for k in range(K):
            tr = fold_of != k
            est = ovr.copy(m)
            model = est.fit(X[tr], y[tr])
            thetas[p, k] = model.hyperparameters
            preds[p, k] = model.predict(X[~tr])
            metrics[p, k] = ev.evaluate(y[~tr], preds[p, k])
            if est.last_objective is not None:
                launches += est.last_objective["launches"]
                evaluations += sum(c["evaluations"] for c in est.last_objective["classes"])
            del model
    avg = [sum(metrics[p, k] for k in range(K)) / K for p in range(len(maps))]
    best = best_index(avg, True)
    ovr.copy(maps[best]).fit(X, y)
    return dict(avg=avg, best=best, thetas=thetas, preds=preds, launches=launches, evaluations=evaluations)


def same(a, b):
    eq = lambda u, v: np.array_equal(np.asarray(u, dtype=np.float64).view(np.int64),
                                     np.asarray(v, dtype=np.float64).view(np.int64))
    return (a["avg"] == b["avg"] and a["best"] == b["best"] and set(a["thetas"]) == set(b["thetas"])
            and all(eq(a["thetas"][key], b["thetas"][key]) and eq(a["preds"][key], b["preds"][key]) for key in a["thetas"]))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--cases", default="iris,shard")
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    report = dict(card=card(), cases={})
    print("card:", report["card"])
    for name in args.cases.split(","):
        X, y, ovr, maps, K, seed = {"iris": iris_case, "shard": shard_case}[name]()
        batched(X, y, ovr, maps, K, seed)               # warm-up: module loads, pooled contexts, workspaces
        tb, ti, rb, ri = [], [], None, None
        for _ in range(args.reps):
            for way, times in ((batched, tb), (independent, ti)):
                eng = sg.ProjectedProcessEngine.acquire(0)
                eng.sync()
                eng.release()
                t0 = time.perf_counter()
                r = way(X, y, ovr, maps, K, seed)
                times.append(time.perf_counter() - t0)
                if way is batched:
                    rb = r
                else:
                    ri = r
        row = dict(cv_s=float(np.median(tb)), independent_s=float(np.median(ti)), rounds=rb["rounds"],
                   evaluations=rb["evaluations"], launches_cv=rb["launches"], launches_independent=ri["launches"],
                   avgMetrics=rb["avg"], identical=bool(same(rb, ri)))
        report["cases"][name] = row
        print(name, json.dumps(row))
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "time_cv_ovr.json"), "w") as f:
            json.dump(report, f, indent=1)


if __name__ == "__main__":
    main()
