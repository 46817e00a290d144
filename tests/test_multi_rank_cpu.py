"""world_size-2 `gloo` test of the multi-GPU decomposition (CPU, no GPU needed).

The statistics are sums over points (PGPH:25-35: treeAggregate seqOp/combOp are plain sums), so ranks hold disjoint
point shards, each computes its partial (G, b) -- here with the oracle standing in for the per-rank kernel -- and ONE
all-reduce(sum) of the packed [G;b] buffer gives every rank the full statistics.  This is the exact host-side logic
bench.py / the C-ABI use (sgp_comm_init + sgp_stats_finish), with gloo in place of NCCL."""
import os
import socket

import numpy as np
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

import oracle
from oracle.regression import bcm_objective


def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    p = s.getsockname()[1]
    s.close()
    return p


def _worker(rank, world, port, ret):
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    rng = np.random.default_rng(3)
    N, d, m = 4000, 6, 64
    X = rng.random((N, d)); y = np.sin(X.sum(1)); Z = X[:m]
    fac = lambda: 1.3 * oracle.ARDRBFKernel(np.full(d, 1.1)) + oracle.const(1) * oracle.EyeKernel()
    theta = fac().get_hyperparameters()
    lo, hi = rank * N // world, (rank + 1) * N // world          # contiguous point shard of this rank
    experts = oracle.get_expert_labels_and_kernels(X[lo:hi], y[lo:hi], fac, 100)
    for _, k in experts:
        k.set_hyperparameters(theta)
    G, b = oracle.get_matrix_kmn_knm_and_vector_kmny(experts, Z)
    packed = torch.from_numpy(np.concatenate([G.ravel(), b]))     # the packed [G;b] buffer of sgp_stats_finish
    dist.all_reduce(packed, op=dist.ReduceOp.SUM)
    if rank == 0:
        full = oracle.get_expert_labels_and_kernels(X, y, fac, 100)
        for _, k in full:
            k.set_hyperparameters(theta)
        G0, b0 = oracle.get_matrix_kmn_knm_and_vector_kmny(full, Z)
        out = packed.numpy()
        ret["dG"] = float(np.abs(out[:m * m].reshape(m, m) - G0).max() / np.abs(G0).max())
        ret["db"] = float(np.abs(out[m * m:] - b0).max() / np.abs(b0).max())
    # the hyper-parameter objective (GPC:73-78) is a sum over EXPERTS: rank r owns experts r, r+world, ... of the
    # reference's grouping (point i -> expert i % E) and one all-reduce of the packed [nll; grad] row gives the total --
    # the contract of sgp_experts_upload + sgp_bcm_nll / sgp_laplace_nll (tests/test_gpu_multi_rank.py runs it on GPUs)
    full = oracle.get_expert_labels_and_kernels(X, y, fac, 100)
    mine = full[rank::world]
    v, g = bcm_objective(mine, theta)
    row = torch.from_numpy(np.concatenate([[v], g]))
    dist.all_reduce(row, op=dist.ReduceOp.SUM)
    if rank == 0:
        v0, g0 = bcm_objective(full, theta)
        ret["dnll"] = float(abs(row[0].item() - v0) / abs(v0))
        ret["dgrad"] = float(np.abs(row[1:].numpy() - g0).max() / np.abs(g0).max())
    dist.destroy_process_group()


def test_two_rank_allreduce_of_shard_statistics():
    ctx = mp.get_context("spawn")
    with ctx.Manager() as mgr:
        ret = mgr.dict()
        port = _free_port()
        procs = [ctx.Process(target=_worker, args=(r, 2, port, ret)) for r in range(2)]
        for p in procs:
            p.start()
        for p in procs:
            p.join(timeout=300)
            assert p.exitcode == 0
        # expert boundaries differ between the sharded and the unsharded run, which is irrelevant to G and b
        assert ret["dG"] < 1e-13 and ret["db"] < 1e-13
        assert ret["dnll"] < 1e-13 and ret["dgrad"] < 1e-12
