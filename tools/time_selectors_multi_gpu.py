"""Model selection over a process group, one process per GPU (GPU box):

    python -m torch.distributed.run --nproc_per_node N tools/time_selectors_multi_gpu.py [reps=3] [out.json]

Three workloads, every rank passing its own shard:
  * cv_regression: CrossValidator over GaussianProcessRegression on a 200 000 x 8 host shard per rank (the seeded
    synthetic rows of `tools/time_cv.py`'s kind: y = sin(sum x) + noise), 5 folds x 2 sigma2 values, RBFKernel(1.0),
    datasetSizeForExpert 100, activeSetSize 200, maxIter 5, random provider;
  * cv_ovr_iris: CrossValidator over OneVsRest on Iris (every rank passes the 150 rows, so the concatenation holds
    150 R rows), 10 folds x 2 sigma2 values, datasetSizeForExpert 20, activeSetSize 30, scored by accuracy;
  * tvs_binary_mnist68: TrainValidationSplit over the binary classifier on the 1500 mnist68 rows (every rank passes
    them), 2 sigma2 values, trainRatio 0.75, scored by areaUnderROC.
Each is timed as whole `fit` calls with a host clock around calls that end in a device synchronise, after one untimed
fit; medians over reps.  At world 1 each alternates with the plain selector on the same rows and checks that both give
the same bits (metrics, bestIndex, every fold or map record, the best model's predictions).  The communicator set-up
(`sgp_comm_init` on a fresh context) and the regression's fold shuffle (one `all_to_all_single`, `exchange_sets`) are
timed apart.  Rank 0 prints one JSON line, with every rank's card name and power limit read in the same run."""
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import numpy as np                                  # noqa: E402
import torch                                        # noqa: E402
import torch.distributed as dist                    # noqa: E402

import spark_gp_b200 as sg                          # noqa: E402
from spark_gp_b200 import distributed as D          # noqa: E402
from spark_gp_b200.utils import kfold_assignment    # noqa: E402

reps = int(sys.argv[1]) if len(sys.argv) > 1 else 3
out_path = sys.argv[2] if len(sys.argv) > 2 else None
rank, world = int(os.environ.get("RANK", 0)), int(os.environ.get("WORLD_SIZE", 1))
local = int(os.environ.get("LOCAL_RANK", rank))
torch.cuda.set_device(local)
dist.init_process_group("nccl", init_method=None if "MASTER_ADDR" in os.environ else "tcp://127.0.0.1:29563",
                        rank=rank, world_size=world, device_id=torch.device("cuda", local))
group = dist.group.WORLD
dev = torch.device("cuda", local)
card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", str(local)],
                      capture_output=True, text=True).stdout.strip()
cards = [None] * world
dist.all_gather_object(cards, card)
GOLD = os.path.join(ROOT, "tests", "golden")


def regression_shard():
    rng = np.random.default_rng(1000 + rank)
    X = rng.random((200_000, 8))
    return X, np.sin(X.sum(1)) + 0.1 * rng.standard_normal(len(X)), rng.random((256, 8))


def iris():
    c = np.load(os.path.join(GOLD, "iris_case.npz"))
    return c["X"], c["y"], c["X"][c["test_idx"]]


def mnist68():
    c = np.load(os.path.join(GOLD, "mnist68_case.npz"))
    n = int(c["n_rows"])
    X = (c["pixels"].astype(np.float64) - c["mean"]) / c["std"]
    return X[:n], c["y01"][:n], X[n:n + 100]


def cv_regression(pg):
    gp = (sg.GaussianProcessRegression(device=local, process_group=pg).setKernel(lambda: sg.RBFKernel(1.0))
          .setDatasetSizeForExpert(100).setActiveSetSize(200).setMaxIter(5).setSeed(3))
    maps = sg.ParamGridBuilder().addGrid("sigma2", [1e-2, 1e-1]).build()
    return sg.CrossValidator().setEstimator(gp).setEstimatorParamMaps(maps).setNumFolds(5).setSeed(1)


def cv_ovr_iris(pg):
    gp = (sg.GaussianProcessClassifier(device=local, process_group=pg).setDatasetSizeForExpert(20)
          .setActiveSetSize(30).setKernel(lambda: sg.RBFKernel(1.0)))
    maps = sg.ParamGridBuilder().addGrid("sigma2", [1e-3, 1e-1]).build()
    return (sg.CrossValidator().setEstimator(sg.OneVsRest().setClassifier(gp)).setEstimatorParamMaps(maps)
            .setEvaluator(sg.MulticlassClassificationEvaluator("accuracy")).setNumFolds(10).setSeed(1))


def tvs_binary_mnist68(pg):
    gp = (sg.GaussianProcessClassifier(device=local, process_group=pg).setDatasetSizeForExpert(100)
          .setActiveSetSize(100).setKernel(lambda: sg.RBFKernel(10.0)).setTol(1e-3).setMaxIter(5))
    maps = sg.ParamGridBuilder().addGrid("sigma2", [1e-3, 1e-1]).build()
    return (sg.TrainValidationSplit().setEstimator(gp).setEstimatorParamMaps(maps)
            .setEvaluator(sg.BinaryClassificationEvaluator()).setSeed(1))


WORKLOADS = [("cv_regression", cv_regression, regression_shard), ("cv_ovr_iris", cv_ovr_iris, iris),
             ("tvs_binary_mnist68", tvs_binary_mnist68, mnist68)]


def timed(fn):
    torch.cuda.synchronize()
    dist.barrier(group)
    t = time.perf_counter()
    out = fn()
    torch.cuda.synchronize()
    return time.perf_counter() - t, out


def outputs(selector, model, Xte):
    """The bits a selector's result is compared on."""
    out = [np.asarray(getattr(model, "avgMetrics", None) or model.validationMetrics), np.array([model.bestIndex], float)]
    folds = getattr(selector, "last_folds", None)
    if folds is not None:
        for key in sorted(folds):
            out += [np.asarray(folds[key]["theta"], float), np.asarray(folds[key]["prediction"], float)]
    else:
        out += [np.asarray(p, float) for p in selector.last_predictions]
    return out + [np.asarray(model.predict(Xte), float)]


def same_bits(a, b):
    return len(a) == len(b) and all(np.array_equal(np.ascontiguousarray(x).view(np.int64),
                                                   np.ascontiguousarray(y).view(np.int64)) for x, y in zip(a, b))


rec = dict(world=world, cards=cards, comm_init_s=[], shuffle_s=[])
for name, make, data in WORKLOADS:
    X, y, Xte = data()
    r = rec[name] = dict(rows_per_rank=len(X), fit_s=[], plain_fit_s=[], identical=[])
    sel = make(group)
    sel.fit(X, y)                                                   # warm-up: every shape once
    if world == 1:
        make(None).fit(X, y)
    for _ in range(reps):
        sel = make(group)
        t, md = timed(lambda: sel.fit(X, y))
        r["fit_s"].append(t)
        if world == 1:
            plain = make(None)
            t, mp_ = timed(lambda: plain.fit(X, y))
            r["plain_fit_s"].append(t)
            r["identical"].append(same_bits(outputs(sel, md, Xte), outputs(plain, mp_, Xte)))
    r["bestIndex"] = md.bestIndex
    for k in ("fit_s", "plain_fit_s"):
        r[k.replace("_s", "_median_s")] = float(np.median(r[k])) if r[k] else None

X, y, _ = regression_shard()
sizes = [None] * world
dist.all_gather_object(sizes, len(X))
offset = sum(sizes[:rank])
fold = kfold_assignment(len(X), 5, 1, offset)
members = [fold != k for k in range(5)]
set_sizes = [None] * world
dist.all_gather_object(set_sizes, [int(m.sum()) for m in members])
plans = [D.ShardPlan([s[k] for s in set_sizes], rank, 100) for k in range(5)]
Xd, yd = torch.as_tensor(X, device=dev), torch.as_tensor(y, device=dev)
for _ in range(reps):
    eng = sg.ProjectedProcessEngine(local)
    try:
        rec["comm_init_s"].append(timed(lambda: D.attach_communicator(eng, group, dev))[0])
    finally:
        eng.close()
    rec["shuffle_s"].append(timed(lambda: D.exchange_sets(plans, members, Xd, yd, group))[0])
for k in ("comm_init_s", "shuffle_s"):
    rec[k.replace("_s", "_median_s")] = float(np.median(rec[k]))
if rank == 0:
    print(json.dumps(rec), flush=True)
    if out_path:
        with open(out_path, "w") as f:
            json.dump(rec, f, indent=1)
dist.destroy_process_group()
