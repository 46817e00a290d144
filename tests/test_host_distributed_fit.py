"""The data-parallel fit's host logic (`spark_gp_b200.distributed`), no GPU needed.

  * the shuffle plan: for ragged N, 1..8 ranks, uneven and empty shards, the rows a rank receives, grouped as the strided
    upload groups them, are its block of `group_for_experts` on the concatenation, expert for expert and row for row;
  * the agreement step's verdicts;
  * a two-rank gloo run of the whole estimator path with a stand-in engine: the objective is all-reduced as the library's
    reducing entries do, so both ranks' L-BFGS-B runs take the same steps; the random provider's active set is the
    single-GPU draw; and a refusal computed on one rank raises on both before any engine exists."""
import os
import queue
import socket

import numpy as np
import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

import spark_gp_b200 as sg
from spark_gp_b200 import distributed as D
from spark_gp_b200.hyperopt import group_for_experts
from spark_gp_b200.regression import ExplicitActiveSetProvider

DEADLINE = 120.0


def shards(N, R, rng, empty=None):
    """R shard sizes summing to N, uneven; rank `empty` gets none."""
    cuts = np.sort(rng.integers(0, N + 1, size=R - 1))
    sizes = np.diff(np.concatenate([[0], cuts, [N]]))
    if empty is not None and R > 1:
        other = (empty + 1) % R
        sizes[other] += sizes[empty]
        sizes[empty] = 0
    return sizes


@pytest.mark.parametrize("R", range(1, 9))
@pytest.mark.parametrize("N,n_e", [(1000, 100), (1037, 100), (999, 37), (2503, 250), (161, 16)])
@pytest.mark.parametrize("empty", [None, 0, "last"])
def test_shuffle_plan_gives_every_rank_its_block_of_the_reference_grouping(R, N, n_e, empty):
    rng = np.random.default_rng(N * 13 + R)
    sizes = shards(N, R, rng, None if empty is None else (R - 1 if empty == "last" else 0))
    reference = group_for_experts(N, n_e)
    E = len(reference)
    plans = [D.ShardPlan(sizes, r, n_e) for r in range(R)]
    assert all(p.E == E and p.N == N for p in plans)
    if E < R:
        assert D.group_refusal(plans[0], [(int(s), 3, "float64", None) for s in sizes], False, True)[0] == "ValueError"
        return
    # the all-to-all: rank s sends its rows to each destination in its row order, rank r concatenates in rank order
    sent = {}
    for s, p in enumerate(plans):
        dest = p.destinations()
        rows = np.arange(p.offsets[s], p.offsets[s + 1])
        order = np.argsort(dest, kind="stable")
        counts = p.send_counts()
        assert counts.sum() == sizes[s]
        parts = np.split(rows[order], np.cumsum(counts)[:-1])
        for r in range(R):
            sent[s, r] = parts[r]
    experts = []
    for r, p in enumerate(plans):
        recv = p.recv_counts()
        assert [len(sent[s, r]) for s in range(R)] == recv.tolist()
        got = np.concatenate([sent[s, r] for s in range(R)])
        np.testing.assert_array_equal(got, p.expert_rows())
        assert p.local_experts >= 1
        # the strided upload: local row i -> local expert i % E_r
        local = [got[q::p.local_experts] for q in range(p.local_experts)]
        assert np.concatenate(local).tolist() == got[p.local_order()].tolist()
        experts += local
    assert len(experts) == E
    for e in range(E):
        np.testing.assert_array_equal(experts[e], reference[e])
    # about E / R experts each, in rank order
    per = np.diff(plans[0].first)
    assert per.max() - per.min() <= 1 and plans[0].first[0] == 0 and plans[0].first[-1] == E


def info(n, d=4, dtype="float64", err=None):
    return (n, d, dtype, err)


def test_agreement_verdicts():
    plan = lambda sizes, n_e=100: D.ShardPlan(sizes, 0, n_e)
    ok = [info(500), info(0), info(700)]
    assert D.group_refusal(plan([500, 0, 700]), ok, False, True) is None
    # a rank's own refusal, named with its rank, wins over everything else
    bad = [info(500), info(0, err=("RuntimeError", "Only 0 and 1 labels are supported.")), info(700, d=5)]
    assert D.group_refusal(plan([500, 0, 700]), bad, True, True) == \
        ("RuntimeError", "rank 1: Only 0 and 1 labels are supported.")
    # shapes and dtypes must agree (empty shards do not count)
    assert "features" in D.group_refusal(plan([500, 0, 700]), [info(500), info(0, d=9), info(700, d=5)], False, True)[1]
    assert D.group_refusal(plan([500, 0, 700]), [info(500), info(0, d=9), info(700)], False, True) is None   # takes d = 4
    assert "dtypes" in D.group_refusal(plan([5, 7]), [info(5), info(7, dtype="float32")], False, False)[1]
    assert D.group_refusal(plan([0, 0]), [info(0), info(0)], False, False)[0] == "ValueError"
    # the expert grouping's limits only where experts are grouped
    three = [info(100), info(50), info(0)]                                  # E = round(1.5) = 2 experts, 3 ranks
    assert "2 experts for 3 ranks" in D.group_refusal(plan([100, 50, 0]), three, False, True)[1]
    assert D.group_refusal(plan([100, 50, 0]), three, False, False) is None
    assert D.group_refusal(plan([120, 130, 0]), [info(120), info(130), info(0)], False, True) is None
    assert D.group_refusal(plan([20, 20], 100), [info(20), info(20)], False, True)[0] == "ZeroDivisionError"
    big = [info(47000), info(47000)]
    assert "46340" in D.group_refusal(plan([47000, 47000], 47000), big, False, True)[1]
    assert "46336" in D.group_refusal(plan([47000, 47000], 47000), big, True, True)[1]
    edge = [info(46340), info(46340)]
    assert D.group_refusal(plan([46340, 46340], 46340), edge, False, True) is None
    assert D.group_refusal(plan([46340, 46340], 46340), edge, True, True) is not None


def test_providers_that_cannot_run_over_a_group_are_refused():
    D.check_provider(sg.RandomActiveSetProvider)
    D.check_provider(ExplicitActiveSetProvider(np.zeros((2, 2))))
    D.check_provider(sg.KMeansActiveSetProvider(on_gpu=True))
    class Derived(ExplicitActiveSetProvider):             # could derive Z from the rank's own shard
        pass
    for p in (sg.KMeansActiveSetProvider(), sg.GreedilyOptimizingActiveSetProvider(), Derived(np.zeros((2, 2)))):
        with pytest.raises(ValueError):
            D.check_provider(p)


# ---------------- two ranks over gloo with a stand-in engine ----------------------------------------------------------
class StandIn:
    """The engine calls of the distributed fit, in numpy, with the library's reductions as gloo all-reduces.  Its
    objective is a convex quadratic in theta over the rank's expert rows, summed over the ranks; its statistics are the
    rows' linear-kernel sums, summed over the ranks."""
    made = 0

    def __init__(self, device):
        StandIn.made += 1
        self.trace = []

    @staticmethod
    def comm_unique_id():
        return bytes(128)

    def comm_init(self, uid, rank, world):
        self.trace.append(("comm_init", rank, world))

    def launch_count(self):
        return len(self.trace)

    def experts_upload_strided(self, X, y, E):
        self.X, self.y, self.E = X.numpy(), y.numpy(), E
        return E

    def bcm_nll(self, kernel):
        theta = kernel.getHyperparameters()
        r = theta[None, :] - self.y[:, None] / 10.0
        row = torch.from_numpy(np.concatenate([[0.5 * (r * r).sum()], r.sum(0)]))
        dist.all_reduce(row)
        self.trace.append(("bcm_nll", theta.tobytes(), row.numpy().tobytes()))
        return float(row[0]), row[1:].numpy()

    def statistics(self, kernel, Z, X, y, shard_points):
        K = np.asarray(X, dtype=np.float64) @ Z.T
        packed = torch.from_numpy(np.concatenate([(K.T @ K).ravel(), K.T @ y]))
        dist.all_reduce(packed)
        m = len(Z)
        self.G, self.b = packed[:m * m].numpy().reshape(m, m), packed[m * m:].numpy()
        return self.G, self.b

    def magic(self):
        return self.b.copy(), self.G.copy()

    def set_precision(self, mode):
        pass

    def begin(self, kernel, Z):
        self.Z = Z

    def set_magic(self, v, M):
        self.magic_pair = (v, M)

    def release(self):
        pass

    def close(self):
        pass


def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    p = s.getsockname()[1]
    s.close()
    return p


def data(N=1037, d=3):
    rng = np.random.default_rng(5)
    X = rng.standard_normal((N, d))
    return X, np.sin(X.sum(1)) + 10.0


def _worker(rank, world, port, sizes, case, outq):
    try:
        os.environ["MASTER_ADDR"] = "127.0.0.1"
        os.environ["MASTER_PORT"] = str(port)
        dist.init_process_group("gloo", rank=rank, world_size=world)
        group = dist.group.WORLD
        X, y = data()
        off = np.concatenate([[0], np.cumsum(sizes)])
        Xl, yl = X[off[rank]:off[rank + 1]], y[off[rank]:off[rank + 1]]
        if len(Xl) == 0:                     # an empty shard of another width than the others: it takes theirs
            Xl = np.empty((0, 5 if rank == 0 else 0))
        if case == "fit":
            gp = sg.GaussianProcessRegression(process_group=group).setMaxIter(20).setActiveSetSize(7).setSeed(3)
            out = {}
            for i in range(2):               # the second fit reuses the group's context and communicator
                model_eng, kernel, theta, Z, mv, mm, (G, b), _ = D.fit(gp, Xl, yl, None, False, engine_factory=StandIn)
                out[i] = dict(theta=theta, Z=Z, G=G, objective=gp.last_objective, model_Z=model_eng.Z,
                              model_magic=model_eng.magic_pair, mv=mv, mm=mm)
            comm = next(iter(D._COMM_ENGINES.values()))
            out.update(trace=comm.trace, X=comm.X, y=comm.y, E=comm.E, made=StandIn.made)
        else:
            gp = sg.GaussianProcessClassifier(process_group=group)
            labels = (yl > 10.0).astype(np.float64)
            if rank == 1:
                labels[-1] = 2.0
            try:
                D.fit(gp, Xl, labels, None, True, engine_factory=StandIn)
                out = dict(error=None)
            except Exception as e:                                      # noqa: BLE001 -- compared in the parent
                out = dict(error=(type(e).__name__, str(e)))
            out["made"] = StandIn.made
        dist.destroy_process_group()
        outq.put((rank, "ok", out))
    except Exception as e:                                              # noqa: BLE001
        import traceback
        outq.put((rank, "error", traceback.format_exc()))


def run_two(sizes, case):
    ctx = mp.get_context("spawn")
    outq = ctx.Queue()
    port = _free_port()
    procs = [ctx.Process(target=_worker, args=(r, 2, port, sizes, case, outq), daemon=True) for r in range(2)]
    for p in procs:
        p.start()
    got = {}
    try:
        for _ in range(2):
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


@pytest.mark.parametrize("sizes", [(600, 437), (0, 1037), (1037, 0), (1, 1036)])
def test_two_ranks_optimise_in_lock_step_and_draw_the_single_gpu_active_set(sizes):
    got = run_two(list(sizes), "fit")
    X, y = data()
    reference = group_for_experts(len(X), 100)
    E = len(reference)
    for r in (0, 1):
        o = got[r]
        # the rows the rank received and uploaded: its block of the reference grouping, row for row, X and y exactly
        first, last = r * E // 2, (r + 1) * E // 2
        assert o["E"] == last - first
        experts = [o["X"][q::o["E"]] for q in range(o["E"])]
        labels = [o["y"][q::o["E"]] for q in range(o["E"])]
        for q, e in enumerate(range(first, last)):
            assert experts[q].tobytes() == X[reference[e]].tobytes() and labels[q].tobytes() == y[reference[e]].tobytes()
        # one communicator for both fits; each model has a context of its own holding the active set and magic pair
        assert o["made"] == 3 and [t for t in o["trace"] if t[0] == "comm_init"] == [("comm_init", r, 2)]
        for i in (0, 1):
            assert o[i]["model_Z"] is o[i]["Z"] and o[i]["model_magic"][0] is o[i]["mv"]
    a, b = got[0], got[1]
    # the same evaluations, in the same order, with the same all-reduced values: the same trajectory on both ranks
    assert a["trace"][1:] == b["trace"][1:] and len(a["trace"]) > 2
    for i in (0, 1):
        assert a[i]["theta"].tobytes() == b[i]["theta"].tobytes() and a[i]["objective"] == b[i]["objective"]
        # the stand-in objective's minimum: theta = mean(y) / 10 over the concatenation
        assert abs(a[i]["theta"][0] - y.mean() / 10.0) < 1e-5
        # the random provider draws the single-GPU indices over N and gathers the rows exactly
        idx = np.random.default_rng(3).choice(len(X), size=7, replace=False)
        assert a[i]["Z"].tobytes() == X[idx].tobytes() == b[i]["Z"].tobytes()
        assert a[i]["G"].tobytes() == b[i]["G"].tobytes()


def test_a_refusal_on_one_rank_raises_on_every_rank_before_any_engine_exists():
    got = run_two([600, 437], "refuse")
    for r in (0, 1):
        assert got[r]["error"] == ("RuntimeError", "rank 1: Only 0 and 1 labels are supported.")
        assert got[r]["made"] == 0
