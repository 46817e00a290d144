"""The data-parallel regression fit over a process group, one process per GPU (GPU box):

    python -m torch.distributed.run --nproc_per_node N tools/time_fit_multi_gpu.py [reps=3] [out.json]

Two workloads, `GaussianProcessRegression.fit` at maxIter = 10 on fp32 CUDA shards of 16 features (the benchmark's
shape): 1M rows per rank, and 1M rows in total.  For each it times, with a host clock around calls that end in a device
synchronise, the whole fit and separately its parts: the communicator set-up (`sgp_comm_init` on a fresh context), the
shuffle of the rows to their experts' owners (one all-to-all), and the sharded GPU K-means (`sgp_kmeans_sharded`, k =
the active-set size).  At world 1 it also times the plain fit of the same shard, alternating with the distributed one,
so the difference is the cost of the group.  Rank 0 prints one JSON line per workload, with every rank's card name and
power limit read in the same run."""
import json
import os
import subprocess
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
import torch
import torch.distributed as dist

import spark_gp_b200 as sg
from spark_gp_b200 import distributed as D

reps = int(sys.argv[1]) if len(sys.argv) > 1 else 3
out_path = sys.argv[2] if len(sys.argv) > 2 else None
rank, world = int(os.environ.get("RANK", 0)), int(os.environ.get("WORLD_SIZE", 1))
local = int(os.environ.get("LOCAL_RANK", rank))
torch.cuda.set_device(local)
dist.init_process_group("nccl", init_method=None if "MASTER_ADDR" in os.environ else "tcp://127.0.0.1:29561",
                        rank=rank, world_size=world, device_id=torch.device("cuda", local))
group = dist.group.WORLD
dev = torch.device("cuda", local)
card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", str(local)],
                      capture_output=True, text=True).stdout.strip()
cards = [None] * world
dist.all_gather_object(cards, card)

d, m, n_e = 16, 1000, 100


def make(process_group):
    return (sg.GaussianProcessRegression(device=local, process_group=process_group)
            .setKernel(lambda: 1 * sg.ARDRBFKernel(np.full(d, np.sqrt(18.0 / d))) + sg.const(1) * sg.EyeKernel())
            .setDatasetSizeForExpert(n_e).setActiveSetSize(m).setSigma2(1e-4).setMaxIter(10).setSeed(13)
            .setActiveSetProvider(sg.KMeansActiveSetProvider(maxIter=10, on_gpu=True)))


def timed(fn):
    torch.cuda.synchronize()
    dist.barrier(group)
    t = time.perf_counter()
    out = fn()
    torch.cuda.synchronize()
    return time.perf_counter() - t, out


def workload(name, n_local):
    rng = np.random.default_rng(13 + rank)
    X = torch.as_tensor(rng.random((n_local, d), dtype=np.float32), device=dev)
    y = torch.as_tensor(np.sin(X.double().sum(1).cpu().numpy()) + 0.1 * rng.standard_normal(n_local), device=dev)
    sizes = [None] * world
    dist.all_gather_object(sizes, n_local)
    plan = D.ShardPlan(sizes, rank, n_e)
    rec = dict(workload=name, world=world, rows_per_rank=sizes, cards=cards, fit_s=[], plain_fit_s=[], comm_init_s=[],
               shuffle_s=[], kmeans_s=[])
    make(group).fit(X, y)                                           # warm-up: every shape once
    if world == 1:
        make(None).fit(X, y)
    for _ in range(reps):
        rec["fit_s"].append(timed(lambda: make(group).fit(X, y))[0])
        if world == 1:
            rec["plain_fit_s"].append(timed(lambda: make(None).fit(X, y))[0])
        eng = sg.ProjectedProcessEngine(local)
        try:
            rec["comm_init_s"].append(timed(lambda: D.attach_communicator(eng, group, dev))[0])
            rec["shuffle_s"].append(timed(lambda: D.exchange(plan, X, y, group))[0])
            rec["kmeans_s"].append(timed(lambda: eng.kmeans_sharded(X, plan.offset, plan.N, m, max_iter=10, seed=13))[0])
        finally:
            eng.close()
    return rec


records = [workload("1M x 16 fp32 per rank", 1_000_000),
           workload("1M x 16 fp32 in total", 1_000_000 // world + (1 if rank < 1_000_000 % world else 0))]
if rank == 0:
    for r in records:
        print(json.dumps(r), flush=True)
    if out_path:
        with open(out_path, "w") as f:
            json.dump(records, f, indent=1)
dist.destroy_process_group()
