"""One-vs-rest over a process group, one process per GPU (GPU box):

    python -m torch.distributed.run --nproc_per_node N tools/time_ovr_multi_gpu.py [reps=3] [out.json]

The workload is the 10-class 200 000 x 8 shard of `tools/time_ovr.py` (datasetSizeForExpert 100, activeSetSize 500,
maxIter 10, RBFKernel(2.0), sigma2 1, host input), on every rank: 200 000 rows per rank.  It times whole
`OneVsRest.fit` calls with a host clock around calls that end in a device synchronise, and reports medians over reps.
At world 1 it alternates the group fit with the plain `OneVsRest.fit` of the same rows, after one untimed fit of each,
so the difference is the cost of the group, and checks that both give the same bits (every class's theta and magic
pair, raw predictions of the held-out rows).  It also times apart the communicator set-up (`sgp_comm_init` on a fresh
context) and the shuffle of the rows to their experts' owners (one all-to-all).  Rank 0 prints one JSON line, with
every rank's card name and power limit read in the same run."""
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))
import numpy as np                                  # noqa: E402
import torch                                        # noqa: E402
import torch.distributed as dist                    # noqa: E402

import spark_gp_b200 as sg                          # noqa: E402
from spark_gp_b200 import distributed as D          # noqa: E402
from time_ovr import synthetic                      # noqa: E402

reps = int(sys.argv[1]) if len(sys.argv) > 1 else 3
out_path = sys.argv[2] if len(sys.argv) > 2 else None
rank, world = int(os.environ.get("RANK", 0)), int(os.environ.get("WORLD_SIZE", 1))
local = int(os.environ.get("LOCAL_RANK", rank))
torch.cuda.set_device(local)
dist.init_process_group("nccl", init_method=None if "MASTER_ADDR" in os.environ else "tcp://127.0.0.1:29562",
                        rank=rank, world_size=world, device_id=torch.device("cuda", local))
group = dist.group.WORLD
dev = torch.device("cuda", local)
card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", str(local)],
                      capture_output=True, text=True).stdout.strip()
cards = [None] * world
dist.all_gather_object(cards, card)


def make(process_group):
    gp = (sg.GaussianProcessClassifier(device=local, process_group=process_group).setDatasetSizeForExpert(100)
          .setActiveSetSize(500).setMaxIter(10).setKernel(lambda: sg.RBFKernel(2.0)).setSigma2(1.0))
    return sg.OneVsRest().setClassifier(gp)


def timed(fn):
    torch.cuda.synchronize()
    dist.barrier(group)
    t = time.perf_counter()
    out = fn()
    torch.cuda.synchronize()
    return time.perf_counter() - t, out


def outputs(model, Xte):
    return [np.asarray(model.hyperparameters)] + [m.rawPredictor.magicVector for m in model.models] + \
        [m.rawPredictor.magicMatrix for m in model.models] + [model.predictRaw(Xte)]


def same_bits(a, b):
    return all(np.array_equal(np.asarray(x).view(np.int64), np.asarray(y).view(np.int64)) for x, y in zip(a, b))


X, y, Xte, yte, _ = synthetic()
sizes = [None] * world
dist.all_gather_object(sizes, len(X))
plan = D.ShardPlan(sizes, rank, 100)
rec = dict(workload="10-class 200 000 x 8 per rank, n_e 100, m 500, maxIter 10", world=world, rows_per_rank=sizes,
           cards=cards, fit_s=[], plain_fit_s=[], comm_init_s=[], shuffle_s=[], identical=[])
make(group).fit(X, y)                                               # warm-up: every shape once
if world == 1:
    make(None).fit(X, y)
for _ in range(reps):
    t, md = timed(lambda: make(group).fit(X, y))
    rec["fit_s"].append(t)
    if world == 1:
        t, mp_ = timed(lambda: make(None).fit(X, y))
        rec["plain_fit_s"].append(t)
        rec["identical"].append(same_bits(outputs(md, Xte), outputs(mp_, Xte)))
    eng = sg.ProjectedProcessEngine(local)
    try:
        rec["comm_init_s"].append(timed(lambda: D.attach_communicator(eng, group, dev))[0])
    finally:
        eng.close()
    Xd, yd = torch.as_tensor(X, device=dev), torch.as_tensor(y, device=dev)
    rec["shuffle_s"].append(timed(lambda: D.exchange(plan, Xd, yd, group))[0])
rec["accuracy"] = float(np.mean(md.predict(Xte) == yte))
for k in ("fit_s", "plain_fit_s", "comm_init_s", "shuffle_s"):
    rec[k.replace("_s", "_median_s")] = float(np.median(rec[k])) if rec[k] else None
if rank == 0:
    print(json.dumps(rec), flush=True)
    if out_path:
        with open(out_path, "w") as f:
            json.dump(rec, f, indent=1)
dist.destroy_process_group()
