"""CPU checks of feature scaling (`spark_gp_b200.scale`, commons/util/Scaling.scala:10-25) off the GPU:
  * the device rule of oracle/scaling_model.py (exact column sums, the reference's formula) against the reference's
    formula as `scale` computes it on the host, on the airfoil, mnist 6-vs-8 and iris fixtures: within the rounding of
    the host's sums;
  * a zero-variance column is divided by 1;
  * the protocol of `scale` over a process group, on two and three gloo ranks with a stand-in engine that sums exactly:
    uneven shards and an empty shard of another width, the same mean and sd on every rank, every rank's own rows back,
    and the refusals -- one rank's own, and every shard empty -- raised on every rank before any engine exists."""
import multiprocessing as mp
import os
import queue
import socket

import numpy as np
import pytest

import oracle
from oracle import scaling_model as SM

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
DEADLINE = 240.0


def fixtures():
    air = np.load(os.path.join(GOLD, "airfoil_case.npz"))
    mn = np.load(os.path.join(GOLD, "mnist68_case.npz"))
    iris = np.load(os.path.join(GOLD, "iris_case.npz"))
    return {"airfoil": air["X"], "mnist68": mn["pixels"].astype(np.float64), "iris": iris["X"]}


def host_bound(X, Y, sd):
    """How far the host formula may lie from the rule, element by element: numpy sums the rows of a column one after
    the other (a reduction over the outer axis), within (n - 1) 2^-53 sum|terms| of the exact sum; that moves the mean by
    dm and the variance by dv, so an output moves by dm / sd + |y| (dv / (2 var) + 2^-53) plus its own two roundings."""
    n = len(X)
    g = n * SM.U
    dm = g * np.abs(X).sum(0) / n + SM.U * np.abs(X.mean(0))
    var = sd * sd
    dv = g * ((X - X.mean(0)) ** 2).sum(0) / n + 2 * dm * np.abs(X - X.mean(0)).sum(0) / n + 2 * SM.U * var
    return (dm / sd + np.abs(Y) * (dv / (2 * var) + SM.U)) * 1.01 + 4 * SM.U * np.abs(Y)


@pytest.mark.parametrize("name", ["airfoil", "mnist68", "iris"])
def test_the_device_rule_gives_the_reference_formula_within_rounding(name):
    from spark_gp_b200.utils import scale
    X = fixtures()[name]
    ref = scale(X)
    assert scale(X).tobytes() == oracle.scale(X).tobytes()        # the host path is the oracle's formula, bit for bit
    mean, sd = SM.moments(X)
    Y = SM.scale(X)
    err = np.abs(Y - ref)
    assert (err <= host_bound(X, Y, sd)).all(), err.max()


def test_a_zero_variance_column_is_divided_by_one():
    rng = np.random.default_rng(3)
    X = np.column_stack([rng.standard_normal(500), np.full(500, 7.25), np.zeros(500)])
    mean, sd = SM.moments(X)
    assert sd[1] == 1.0 and sd[2] == 1.0 and mean[1] == 7.25 and mean[2] == 0.0
    Y = SM.scale(X)
    assert (Y[:, 1] == 0.0).all() and (Y[:, 2] == 0.0).all()
    from spark_gp_b200.utils import scale
    assert (scale(X)[:, 1:] == 0.0).all()


def test_the_sum_bound_counts_blocks():
    assert SM.blocks(1) == 1 and SM.blocks(SM.ROWS_PER_BLOCK) == 1 and SM.blocks(SM.ROWS_PER_BLOCK + 1) == 2
    assert SM.sum_bound(5000, [1.0])[0] == (SM.ROWS_PER_BLOCK + 3) * SM.U


# ---------------- the group protocol over gloo, with a stand-in engine ------------------------------------------------
class StandIn:
    """The engine calls of `scale` in numpy: exact column sums of the rank's rows, and the host formula.  It records the
    mean and sd it is asked to apply."""
    made = 0

    def __init__(self, device):
        StandIn.made += 1

    def column_sums(self, X, center=None):
        T = X.cpu().numpy().astype(np.float64)
        if center is not None:
            T = SM.centred_squares(T, center)
        return SM.exact_sums(T) if len(T) else np.zeros(T.shape[1])

    def scale_apply(self, X, mean, sd):
        import torch
        self.applied = (mean.copy(), sd.copy())
        return torch.from_numpy((X.cpu().numpy().astype(np.float64) - mean) / sd)

    def release(self):
        StandIn.last = self


def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    p = s.getsockname()[1]
    s.close()
    return p


def data(N=2000, d=4):
    rng = np.random.default_rng(8)
    X = rng.standard_normal((N, d)) * np.array([1.0, 1e-3, 5.0, 2.0])[:d] + np.array([0.0, 1e6, -3.0, 0.5])[:d]
    X[:, 3] = 2.0                                                    # a constant column
    return X


def _worker(rank, world, port, sizes, case, outq):
    try:
        import torch.distributed as dist

        from spark_gp_b200 import distributed as D
        os.environ["MASTER_ADDR"] = "127.0.0.1"
        os.environ["MASTER_PORT"] = str(port)
        dist.init_process_group("gloo", rank=rank, world_size=world)
        X = data()
        off = np.concatenate([[0], np.cumsum(sizes)])
        Xl = X[off[rank]:off[rank + 1]]
        if len(Xl) == 0:                     # an empty shard of another width than the others: it takes theirs
            Xl = np.empty((0, 7))
        if case == "bad" and rank == world - 1:
            Xl = Xl[:, 0]                    # one rank's shard is not n x d
        try:
            Y = D.scale(Xl, dist.group.WORLD, engine_factory=StandIn)
            out = dict(error=None, Y=Y, applied=StandIn.last.applied)
        except Exception as e:                                      # noqa: BLE001 -- compared in the parent
            out = dict(error=(type(e).__name__, str(e)))
        out["made"] = StandIn.made
        dist.destroy_process_group()
        outq.put((rank, "ok", out))
    except Exception:                                               # noqa: BLE001
        import traceback
        outq.put((rank, "error", traceback.format_exc()))


def run(sizes, case="scale"):
    ctx = mp.get_context("spawn")
    outq = ctx.Queue()
    port = _free_port()
    world = len(sizes)
    procs = [ctx.Process(target=_worker, args=(r, world, port, list(sizes), case, outq), daemon=True)
             for r in range(world)]
    for p in procs:
        p.start()
    got = {}
    try:
        for _ in range(world):
            rank, status, out = outq.get(timeout=DEADLINE)
            assert status == "ok", out
            got[rank] = out
    except queue.Empty:
        pytest.fail("the gloo workers passed their deadline")
    finally:
        for p in procs:
            p.join(timeout=30)
            if p.is_alive():
                p.kill()
                p.join()
    return got


@pytest.mark.parametrize("sizes", [(1200, 800), (0, 2000), (2000, 0), (1, 1500, 499), (700, 0, 1300)])
def test_every_rank_scales_its_rows_with_the_mean_and_sd_of_the_concatenation(sizes):
    got = run(sizes)
    X = data()
    mean0, sd0 = SM.moments(X)
    off = np.concatenate([[0], np.cumsum(sizes)])
    ref_mean, ref_sd = got[0]["applied"]
    # the rank sums of exact partials are within the sum bound of the exact sums of the concatenation
    S_bound = SM.sum_bound(len(X), np.abs(X).sum(0)) / len(X)
    assert (np.abs(ref_mean - mean0) <= S_bound + SM.U * np.abs(mean0)).all()
    assert ref_sd[3] == 1.0 and np.allclose(ref_sd, sd0, rtol=1e-12)
    for r in range(len(sizes)):
        o = got[r]
        assert o["error"] is None and o["made"] == 1
        mean, sd = o["applied"]
        assert mean.tobytes() == ref_mean.tobytes() and sd.tobytes() == ref_sd.tobytes()
        Xl = X[off[r]:off[r + 1]]
        assert isinstance(o["Y"], np.ndarray) and o["Y"].dtype == np.float64 and o["Y"].shape == (len(Xl), 4)
        assert o["Y"].tobytes() == ((Xl - mean) / sd).tobytes()


def test_a_refusal_on_one_rank_raises_on_every_rank_before_any_engine_exists():
    got = run((1000, 600, 400), "bad")
    for r in range(3):
        assert got[r]["error"] == ("ValueError", "rank 2: scale: X must be n x d") and got[r]["made"] == 0


def test_every_shard_empty_is_refused_on_every_rank():
    got = run((0, 0))
    for r in range(2):
        assert got[r]["error"] == ("ValueError", "every rank's shard is empty") and got[r]["made"] == 0
