"""One-vs-rest over a process group (`spark_gp_b200.distributed.group_fit(..., "classes")`), host logic, no GPU needed.

  * the agreement step: numClasses from the ranks' largest labels (a rank without the top class, an empty rank), one
    rank's bad labels named on every rank, the expert limit and E < R;
  * two-rank gloo runs of the whole one-vs-rest path with a stand-in engine whose classes objective all-reduces every
    listed class's [value; gradient] as `sgp_laplace_nll_classes_any_size` does, and whose per-class modes follow each
    class's theta: every rank uploads exactly its block of `group_for_experts`, class indices included; the classes'
    L-BFGS-B runs go in lock step, the same on both ranks, each to the optimum of the concatenation; the modes come back
    in global row order; a binary fit and a one-vs-rest fit share one communicator; and a bad label on rank 1 raises on
    both ranks before any engine exists."""
import os
import queue
import socket

import numpy as np
import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

import spark_gp_b200 as sg
from spark_gp_b200 import _native as N
from spark_gp_b200 import distributed as D
from spark_gp_b200.hyperopt import group_for_experts

DEADLINE = 120.0
N_ROWS, N_E, TOP_ROW = 1037, 100, 5          # TOP_ROW holds the only row of the top class


def info(n, d=4, dtype="float64", err=None, top=-1):
    return (n, d, dtype, err, top)


def test_num_classes_is_one_more_than_the_largest_label_of_any_rank():
    assert D.num_classes([info(500, top=2), info(0), info(700, top=4)]) == 5      # an empty rank sends -1
    assert D.num_classes([info(500, top=4), info(700, top=1)]) == 5               # class 4 lives on rank 0 only
    assert D.num_classes([info(0), info(700, top=0)]) == 1
    # the agreement verdicts take the 5-entry form unchanged
    plan = D.ShardPlan([500, 0, 700], 0, 100)
    assert D.group_refusal(plan, [info(500, top=2), info(0), info(700, top=4)], True, True) is None


@pytest.mark.parametrize("labels,message", [([0.0, 1.5, 2.0], "non-negative integers"),
                                            ([0.0, -1.0, 2.0], "non-negative integers"),
                                            ([0.0, np.nan, 2.0], "non-negative integers")])
def test_bad_labels_of_one_rank_are_named_on_every_rank(labels, message):
    X = np.zeros((3, 4))
    with pytest.raises(ValueError, match=message):
        D._local_data(X, np.array(labels), 0, "classes", "OneVsRest.fit")
    try:
        D._local_data(X, np.array(labels), 0, "classes", "OneVsRest.fit")
    except ValueError as e:
        err = (type(e).__name__, str(e))
    plan = D.ShardPlan([3, 3], 0, 2)
    verdict = D.group_refusal(plan, [info(3, top=2), info(3, err=err)], True, True)
    assert verdict[0] == "ValueError" and verdict[1].startswith("rank 1: OneVsRest: labels must be non-negative")


def test_local_labels_give_the_largest_class_and_allow_an_empty_shard():
    X, y, top = D._local_data(np.zeros((4, 2)), np.array([0, 3, 1, 3]), 0, "classes", "OneVsRest.fit")
    assert top == 3 and y.dtype == np.float64
    assert D._local_data(np.zeros((0, 2)), np.zeros(0), 0, "classes", "OneVsRest.fit")[2] == -1
    assert D._local_data(np.zeros((4, 2)), np.array([0, 1, 1, 0]), 0, "binary", "GaussianProcessClassifier.fit")[2] == -1


def test_expert_limits_of_one_vs_rest():
    big = [info(47000, top=1), info(47000, top=2)]
    assert "46336" in D.group_refusal(D.ShardPlan([47000, 47000], 0, 47000), big, True, True)[1]
    edge = [info(46336, top=1), info(46336, top=2)]
    assert D.group_refusal(D.ShardPlan([46336, 46336], 0, 46336), edge, True, True) is None
    three = [info(100, top=1), info(50, top=1), info(0)]                  # E = round(1.5) = 2 experts, 3 ranks
    assert "2 experts for 3 ranks" in D.group_refusal(D.ShardPlan([100, 50, 0], 0, 100), three, True, True)[1]


# ---------------- two ranks over gloo with a stand-in engine ----------------------------------------------------------
def data():
    rng = np.random.default_rng(8)
    X = rng.standard_normal((N_ROWS, 3))
    y = rng.integers(0, 3, N_ROWS).astype(np.float64)
    y[TOP_ROW] = 3.0
    return X, y


def target(X, y, c):
    """The stand-in objective of class c is 1/2 sum over rows (theta - target)^2: its optimum is the target's mean."""
    return 1.0 + (y == c) + 0.1 * np.tanh(X[:, 0])


def modes(X, y, c, theta):
    """The stand-in's modes of class c at theta, per row."""
    return theta * (y == c) - X[:, 0]


class StandIn:
    """The engine calls of the group fit, in numpy, with the library's reductions as gloo all-reduces."""
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
        n = len(self.X)
        self.order = np.concatenate([np.arange(q, n, E) for q in range(E)])     # row i -> expert i % E, expert-major
        self.f = {}
        return E

    def laplace_nll_classes_any_size(self, n_classes, classes, kernels, tol):
        thetas = [k.getHyperparameters()[0] for k in kernels]
        rows = []
        for c, t in zip(classes, thetas):
            r = t - target(self.X, self.y, c)
            rows += [0.5 * (r * r).sum(), r.sum()]
            self.f[N.SGP_MODES_CLASS, c] = modes(self.X, self.y, c, t)[self.order]
        packed = torch.tensor(rows, dtype=torch.float64)
        dist.all_reduce(packed)
        self.trace.append(("classes", n_classes, list(classes), np.array(thetas).tobytes(), packed.numpy().tobytes()))
        out = packed.numpy().reshape(len(classes), 2)
        return out[:, 0].copy(), out[:, 1:].copy()

    def laplace_nll_any_size(self, kernel, tol):
        t = kernel.getHyperparameters()[0]
        r = t - target(self.X, self.y, 1)
        packed = torch.tensor([0.5 * (r * r).sum(), r.sum()], dtype=torch.float64)
        dist.all_reduce(packed)
        self.f[N.SGP_MODES_BINARY, 0] = modes(self.X, self.y, 1, t)[self.order]
        self.trace.append(("binary", np.float64(t).tobytes(), packed.numpy().tobytes()))
        return float(packed[0]), packed[1:].numpy()

    def experts_modes(self, store, index, n):
        assert n == len(self.X)
        return self.f[store, index].copy()

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
        self.trace.append(("precision", mode))

    def begin(self, kernel, Z):
        self.Z = Z

    def set_magic(self, v, M):
        self.magic_pair = (v, M)

    def close(self):
        pass


def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    p = s.getsockname()[1]
    s.close()
    return p


def classifier(group):
    return (sg.GaussianProcessClassifier(process_group=group).setKernel(lambda: sg.RBFKernel(1.0)).setMaxIter(20)
            .setActiveSetSize(7).setSeed(3))


def _worker(rank, world, port, sizes, case, outq):
    try:
        os.environ["MASTER_ADDR"] = "127.0.0.1"
        os.environ["MASTER_PORT"] = str(port)
        dist.init_process_group("gloo", rank=rank, world_size=world)
        group = dist.group.WORLD
        X, y = data()
        off = np.concatenate([[0], np.cumsum(sizes)])
        Xl, yl = X[off[rank]:off[rank + 1]], y[off[rank]:off[rank + 1]]
        gp = classifier(group)
        if case == "fit":
            # a binary fit first: the one-vs-rest fit after it reuses the group's communicator
            D.fit(gp, Xl, (yl == 1).astype(np.float64), None, True, engine_factory=StandIn)
            made_binary = StandIn.made
            models, record = D.group_fit(gp, Xl, yl, None, "classes", engine_factory=StandIn)
            comm = next(iter(D._COMM_ENGINES.values()))
            out = dict(trace=comm.trace, X=comm.X, y=comm.y, E=comm.E, made_binary=made_binary, made=StandIn.made,
                       thetas=[m[2] for m in models], Z=[m[3] for m in models], G=[m[6][0] for m in models],
                       f=[m[7] for m in models], model_Z=[m[0].Z for m in models], record=record)
        else:
            yl = yl.copy()
            if rank == 1:
                yl[-1] = -1.0
            try:
                D.group_fit(gp, Xl, yl, None, "classes", engine_factory=StandIn)
                out = dict(error=None)
            except Exception as e:                                      # noqa: BLE001 -- compared in the parent
                out = dict(error=(type(e).__name__, str(e)))
            out["made"] = StandIn.made
        dist.destroy_process_group()
        outq.put((rank, "ok", out))
    except Exception:                                                   # noqa: BLE001
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


@pytest.mark.parametrize("sizes", [(600, 437), (0, 1037), (1037, 0)])
def test_two_ranks_fit_every_class_in_lock_step_on_their_block_of_the_experts(sizes):
    got = run_two(list(sizes), "fit")
    X, y = data()
    C = 4                                       # the top class has one row, on one rank only (or on the only full one)
    reference = group_for_experts(N_ROWS, N_E)
    E = len(reference)
    for r in (0, 1):
        o = got[r]
        # the rank's block of the reference grouping, row for row: X and the class indices exactly
        first, last = r * E // 2, (r + 1) * E // 2
        assert o["E"] == last - first
        for q, e in enumerate(range(first, last)):
            assert o["X"][q::o["E"]].tobytes() == X[reference[e]].tobytes()
            assert o["y"][q::o["E"]].tobytes() == y[reference[e]].tobytes()
        # one communicator for the binary and the one-vs-rest fit; one model context per fit and per class
        assert [t for t in o["trace"] if t[0] == "comm_init"] == [("comm_init", r, 2)]
        assert o["made_binary"] == 2 and o["made"] == 2 + C
        assert len(o["thetas"]) == C and all(mz is z for mz, z in zip(o["model_Z"], o["Z"]))
        # every round lists the pending classes in class order, every round of the same fit has C numClasses
        rounds = [t for t in o["trace"] if t[0] == "classes"]
        assert all(t[1] == C and t[2] == sorted(t[2]) for t in rounds)
        assert rounds[0][2] == list(range(C)) and rounds[-1][2] == list(range(C))      # x0 together; the call at theta
        # the modes of the rank's expert rows, in global row order, at each class's theta
        rows = D.ShardPlan(list(sizes), r, N_E).expert_rows()
        for c in range(C):
            assert o["f"][c].tobytes() == modes(X[rows], y[rows], c, o["thetas"][c][0]).tobytes(), c
    a, b = got[0], got[1]
    # the same evaluations, in the same order, with the same all-reduced values: the same trajectories on both ranks
    assert a["trace"][1:] == b["trace"][1:] and len([t for t in a["trace"] if t[0] == "classes"]) > 2
    assert a["record"] == b["record"] and len(a["record"]["slots"]) == C
    assert a["record"]["rounds"] == max(s["evaluations"] for s in a["record"]["slots"])
    idx = np.random.default_rng(3).choice(N_ROWS, size=7, replace=False)
    for c in range(C):
        assert a["thetas"][c].tobytes() == b["thetas"][c].tobytes()
        # each class reaches the optimum of the concatenation
        assert abs(a["thetas"][c][0] - target(X, y, c).mean()) < 1e-5
        assert a["Z"][c].tobytes() == X[idx].tobytes() == b["Z"][c].tobytes()
        assert a["G"][c].tobytes() == b["G"][c].tobytes()


def test_a_bad_label_on_one_rank_raises_on_every_rank_before_any_engine_exists():
    got = run_two([600, 437], "refuse")
    for r in (0, 1):
        assert got[r]["error"] == ("ValueError",
                                   "rank 1: OneVsRest: labels must be non-negative integers (class indices)")
        assert got[r]["made"] == 0
