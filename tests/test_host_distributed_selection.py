"""Model selection over a process group (`CrossValidator` / `TrainValidationSplit` with a `process_group` estimator,
`spark_gp_b200.distributed.selection`), host logic, no GPU needed.

  * set plans: for 1..8 ranks with uneven shards and an empty one, every fold's training set and the train/validation
    split's training set, the rows a rank receives, grouped row i -> expert i % E_k,r, are its block of
    `group_for_experts` on the plain set, expert for expert and row for row; one gloo run checks `exchange_sets` itself;
  * the seeded splits of the ranks, numbered from their offsets, concatenate to the plain splits;
  * every refusal of the agreement, including one that only one rank sees, which a two-rank gloo run raises on both ranks
    before any engine exists;
  * two-rank gloo runs with a stand-in engine whose objectives all-reduce as the library's do: both ranks take the same
    lock-step trajectories, gather the same validation arrays, compute the same metrics and bestIndex, refit the same
    map, and one communicator serves a CrossValidator and a TrainValidationSplit after it."""
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
from spark_gp_b200.utils import kfold_assignment, train_validation_assignment

DEADLINE = 120.0
N_E = 10


def shard_sizes(N, R, seed):
    """Uneven sizes of R shards of N rows, one of them empty when R > 1."""
    if R == 1:
        return [N]
    cuts = np.sort(np.random.default_rng(seed).choice(np.arange(1, N), size=R - 2, replace=False))
    sizes = list(np.diff(np.concatenate([[0], cuts, [N]])))
    return sizes[:seed % R] + [0] + sizes[seed % R:]


def received(plans, members_of, r):
    """What rank r receives of every set, as `exchange_sets` orders it: by set, then source rank, then row (global row
    indices)."""
    out = []
    for k, plan in enumerate(plans):
        rows = []
        for s in range(plan.R):
            mine = members_of[s][k]
            dest = D.ShardPlan(plan.sizes, s, N_E).destinations()
            rows.append(mine[dest == r])
        out.append(np.concatenate(rows))
    return out


def check_blocks(masks_global, sizes):
    """For every set (a global bool mask), every rank's received rows grouped i % E_k,r are its block of the plain
    grouping of the set."""
    R = len(sizes)
    off = np.concatenate([[0], np.cumsum(sizes)])
    members_of = [[np.arange(off[s], off[s + 1])[m[off[s]:off[s + 1]]] for m in masks_global] for s in range(R)]
    set_sizes = [[len(members_of[s][k]) for k in range(len(masks_global))] for s in range(R)]
    for r in range(R):
        plans = [D.ShardPlan([set_sizes[s][k] for s in range(R)], r, N_E) for k in range(len(masks_global))]
        got = received(plans, members_of, r)
        for k, m in enumerate(masks_global):
            rows = np.flatnonzero(m)
            reference = group_for_experts(len(rows), N_E)
            plan = plans[k]
            assert plan.E == len(reference)
            E_r = plan.local_experts
            assert E_r >= 1 and len(got[k]) == sum(len(reference[e]) for e in range(plan.first[r], plan.first[r + 1]))
            for q, e in enumerate(range(plan.first[r], plan.first[r + 1])):
                assert np.array_equal(got[k][q::E_r], rows[reference[e]]), (r, k, e)


@pytest.mark.parametrize("R", range(1, 9))
@pytest.mark.parametrize("N", [161, 999, 1037, 2503])
def test_every_rank_receives_its_block_of_every_training_set(R, N):
    sizes = shard_sizes(N, R, N + R)
    for K in (2, 3, 5, 10):
        if N // K < N_E * R:                    # E_k < R: refused by the agreement, covered below
            continue
        fold = kfold_assignment(N, K, 7)
        check_blocks([fold != k for k in range(K)], sizes)
    check_blocks([train_validation_assignment(N, 0.75, 7)], sizes)


@pytest.mark.parametrize("N", [161, 1037, 2503])
def test_seeded_splits_of_the_ranks_concatenate_to_the_plain_splits(N):
    for R in (1, 3, 8):
        sizes = shard_sizes(N, R, N)
        off = np.concatenate([[0], np.cumsum(sizes)])
        for K in (2, 5, 10):
            parts = [kfold_assignment(sizes[r], K, 11, off[r]) for r in range(R)]
            assert np.concatenate(parts).tobytes() == kfold_assignment(N, K, 11).tobytes()
        parts = [train_validation_assignment(sizes[r], 0.6, 11, off[r]) for r in range(R)]
        assert np.concatenate(parts).tobytes() == train_validation_assignment(N, 0.6, 11).tobytes()


# ---------------- the agreement's verdicts ---------------------------------------------------------------------------
def entry(n, rows, err=None, tops=None, d=3):
    return (n, d, "float64", err, -1, rows, tops or [-1] * len(rows))


CV = sg.CrossValidator._empty_fold
TVS = sg.TrainValidationSplit._empty_side


def test_verdicts_of_the_selection_agreement():
    ok = [entry(600, [400, 420, 380]), entry(500, [330, 340, 330])]
    assert D.selection_refusal(ok, False, [50], CV) is None
    # a bad given split (or bad data, or a refused provider) on one rank is named on every rank
    bad = [ok[0], entry(0, [], err=("ValueError", "CrossValidator: folds must hold one integer in [0, numFolds) per row"))]
    assert D.selection_refusal(bad, False, [50], CV) == (
        "ValueError", "rank 1: CrossValidator: folds must hold one integer in [0, numFolds) per row")
    # a fold without validation rows over the whole group (its rows are all on other ranks' training sets)
    empty = [entry(600, [600, 400, 200]), entry(500, [500, 250, 250])]
    assert D.selection_refusal(empty, False, [50], CV) == ("ValueError", "CrossValidator: fold 0 has no rows to "
                                                                         "validate on")
    for rows, side in (([0], "training"), ([600], "validation")):
        v = D.selection_refusal([entry(600, rows), entry(0, [0])], True, [50], TVS)
        assert v == ("ValueError", "TrainValidationSplit: the %s side of the split is empty" % side)
    # the expert grouping of every set, for every datasetSizeForExpert that groups experts
    assert D.selection_refusal(ok, False, [50, 2000], CV)[0] == "ZeroDivisionError"
    assert D.selection_refusal(ok, False, [600], CV) == (
        "ValueError", "training set 0: 1 experts for 2 ranks: every rank needs at least one expert (lower "
                      "datasetSizeForExpert or use fewer ranks)")
    big = [entry(46400, [46338]), entry(46400, [46338])]                           # 2 experts of 46338 points
    assert "training set 0: datasetSizeForExpert above 46336" in D.selection_refusal(big, True, [46338], TVS)[1]
    assert D.selection_refusal(big, False, [46338], TVS) is None                  # the BCM limit is 46340
    # maps that group no experts (regression with maxIter <= 0) set no expert limit
    assert D.selection_refusal(ok, False, [], CV) is None


def test_a_refused_provider_in_any_param_map_is_a_local_refusal():
    gp = sg.GaussianProcessRegression().setActiveSetProvider(sg.GreedilyOptimizingActiveSetProvider())
    with pytest.raises(ValueError, match="cannot run over a process group"):
        D.check_provider(gp._activeSetProvider)


# ---------------- two ranks over gloo with a stand-in engine ----------------------------------------------------------
N_ROWS = 1037


def data():
    rng = np.random.default_rng(8)
    X = rng.standard_normal((N_ROWS, 3))
    y = np.where(X[:, 0] + 0.3 * rng.standard_normal(N_ROWS) > 0, 1.0, 0.0)
    return X, y


def target(X, y):
    """The stand-in objective of a set is 1/2 sum over its rows (theta - target)^2: its optimum is the target's mean."""
    return 1.0 + y + 0.1 * np.tanh(X[:, 0])


class StandIn:
    """The engine calls of the selectors over a group, in numpy, with the library's reductions as gloo all-reduces."""
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

    def _reduce(self, rows):
        packed = torch.tensor(rows, dtype=torch.float64)
        dist.all_reduce(packed)
        return packed.numpy().reshape(-1, 2)

    def experts_upload_fold_sets(self, X, y, rows, experts):
        X, y = X.numpy(), y.numpy()
        cut = np.cumsum(rows)[:-1]
        self.sets = list(zip(np.split(X, cut), np.split(y, cut)))
        self.trace.append(("fold_sets", [int(r) for r in rows], [int(e) for e in experts], X.tobytes()))
        return experts

    def experts_upload_strided(self, X, y, E):
        X, y = X.numpy(), y.numpy()
        self.sets, self.f = [(X, y)], {}
        self.order = np.concatenate([np.arange(q, len(X), E) for q in range(E)])
        self.trace.append(("strided", int(E), X.tobytes()))
        return E

    def _values(self, sets, kernels, what, labels=lambda y, i: y):
        thetas = [k.getHyperparameters()[0] for k in kernels]
        rows = []
        for i, (s, t) in enumerate(zip(sets, thetas)):
            X, y = self.sets[s]
            r = t - target(X, labels(y, i))
            rows += [0.5 * (r * r).sum(), r.sum()]
        out = self._reduce(rows)
        self.trace.append((what, list(sets), np.array(thetas).tobytes(), out.tobytes()))
        return out[:, 0].copy(), out[:, 1:].copy()

    def bcm_nll_folds(self, sets, kernels):
        return self._values(sets, kernels, "bcm_folds")

    def bcm_nll_slots(self, kernels):
        return self._values([0] * len(kernels), kernels, "bcm_slots")

    def laplace_nll_slots_any_size(self, n_mode_slots, modes, classes, kernels, tol):
        out = self._values([0] * len(kernels), kernels, "laplace_slots", lambda y, i: (y == classes[i]) * 1.0)
        X, y = self.sets[0]
        for m, c, k in zip(modes, classes, kernels):
            self.f[m] = (k.getHyperparameters()[0] * (y == c) - X[:, 0])[self.order]
        return out

    def experts_modes(self, store, index, n):
        return self.f[index].copy()

    def statistics(self, kernel, Z, X, y, shard_points):
        K = np.asarray(X, dtype=np.float64) @ Z.T
        packed = torch.from_numpy(np.concatenate([(K.T @ K).ravel(), K.T @ np.asarray(y)]))
        dist.all_reduce(packed)
        m = len(Z)
        self.Z, self.G, self.b = Z, packed[:m * m].numpy().reshape(m, m), packed[m * m:].numpy()
        self.trace.append(("stats", Z.tobytes(), packed.numpy().tobytes()))
        return self.G, self.b

    def magic(self):
        return self.b.copy(), self.G.copy()

    def predict(self, X, with_variance=True):
        return np.tanh(np.asarray(X) @ self.Z.T @ self.b * 1e-3), None

    def set_precision(self, mode):
        pass

    def close(self):
        pass


def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    p = s.getsockname()[1]
    s.close()
    return p


def _refit(self, X, y, hyperparameters=None):
    """The refit, recorded: the group fit itself is pinned by the distributed fit's tests."""
    return ("refit", type(self).__name__, self._activeSetSize, np.asarray(X).tobytes(), np.asarray(y).tobytes())


def _worker(rank, world, port, sizes, case, outq):
    try:
        os.environ["MASTER_ADDR"] = "127.0.0.1"
        os.environ["MASTER_PORT"] = str(port)
        dist.init_process_group("gloo", rank=rank, world_size=world)
        group = dist.group.WORLD
        made = D.comm_engine
        D.comm_engine = lambda g, i, dev, factory: made(g, i, dev, StandIn)
        sg.GaussianProcessRegression.fit = _refit
        sg.GaussianProcessClassifier.fit = _refit
        X, y = data()
        off = np.concatenate([[0], np.cumsum(sizes)])
        Xl, yl = X[off[rank]:off[rank + 1]], y[off[rank]:off[rank + 1]]
        maps = sg.ParamGridBuilder().addGrid("activeSetSize", [5, 7]).build()
        if case == "select":
            gpr = (sg.GaussianProcessRegression(process_group=group).setKernel(lambda: sg.RBFKernel(1.0))
                   .setDatasetSizeForExpert(50).setMaxIter(20).setSeed(3))
            cv = sg.CrossValidator().setEstimator(gpr).setEstimatorParamMaps(maps).setNumFolds(3).setSeed(5)
            cvm = cv.fit(Xl, yl)
            gpc = (sg.GaussianProcessClassifier(process_group=group).setKernel(lambda: sg.RBFKernel(1.0))
                   .setDatasetSizeForExpert(50).setMaxIter(20).setSeed(3))
            tvs = (sg.TrainValidationSplit().setEstimator(gpc).setEstimatorParamMaps(maps).setSeed(5)
                   .setEvaluator(sg.BinaryClassificationEvaluator()))
            tvm = tvs.fit(Xl, yl)
            comm = next(iter(D._COMM_ENGINES.values()))
            out = dict(trace=comm.trace, made=StandIn.made, cv_avg=cvm.avgMetrics, cv_best=cvm.bestIndex,
                       cv_refit=cvm.bestModel, cv_objective=cvm.last_objective,
                       cv_folds={k: (v["prediction"].tobytes(), v["theta"].tobytes()) for k, v in cv.last_folds.items()},
                       tvs_metrics=tvm.validationMetrics, tvs_best=tvm.bestIndex, tvs_refit=tvm.bestModel,
                       tvs_predictions=[p.tobytes() for p in tvs.last_predictions], tvs_objective=tvm.last_objective)
        else:
            folds = kfold_assignment(len(Xl), 3, 5, off[rank])
            if rank == 1:
                folds[-1] = 3
            gpr = sg.GaussianProcessRegression(process_group=group).setDatasetSizeForExpert(50)
            cv = sg.CrossValidator().setEstimator(gpr).setEstimatorParamMaps(maps).setNumFolds(3)
            try:
                cv.fit(Xl, yl, folds=folds)
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


@pytest.mark.parametrize("sizes", [(600, 437), (0, 1037)])
def test_two_ranks_select_in_lock_step_on_gathered_validation_arrays(sizes):
    got = run_two(list(sizes), "select")
    a, b = got[0], got[1]
    X, y = data()
    # one communicator for the CrossValidator and the TrainValidationSplit after it
    assert [t for t in a["trace"] if t[0] == "comm_init"] == [("comm_init", 0, 2)]
    assert a["made"] == 1 and b["made"] == 1
    # the same evaluations, in the same order, with the same all-reduced values on both ranks
    rounds = lambda o, what: [t[1:] for t in o["trace"] if t[0] == what]
    for what in ("bcm_folds", "laplace_slots", "stats"):
        assert rounds(a, what) == rounds(b, what) and len(rounds(a, what)) > 2, what
    # each (map, fold) slot reaches the optimum of its training set of the concatenation
    fold = kfold_assignment(N_ROWS, 3, 5)
    for (p, k), (_, theta) in a["cv_folds"].items():
        t = np.frombuffer(theta)[0]
        assert abs(t - target(X[fold != k], y[fold != k]).mean()) < 1e-5
    # the gathered predictions, the metrics, bestIndex and the refitted map agree on both ranks
    for key in ("cv_avg", "cv_best", "cv_folds", "tvs_metrics", "tvs_best", "tvs_predictions"):
        assert a[key] == b[key], key
    assert all(len(np.frombuffer(v[0])) == np.count_nonzero(fold == k) for (p, k), v in a["cv_folds"].items())
    assert a["cv_refit"][:3] == b["cv_refit"][:3] == ("refit", "GaussianProcessRegression", [5, 7][a["cv_best"]])
    assert a["tvs_refit"][2] == b["tvs_refit"][2] == [5, 7][a["tvs_best"]]
    # each rank refits on its own shard
    off = np.concatenate([[0], np.cumsum(sizes)])
    for r, o in got.items():
        assert o["cv_refit"][3] == X[off[r]:off[r + 1]].tobytes()
    # the records have the plain selectors' shape
    assert [sorted(g) for g in a["cv_objective"]["groups"]] == [["launches", "rounds", "slots"]]
    assert a["cv_objective"]["fold_metrics"].shape == (2, 3)
    assert len(a["tvs_objective"]["groups"]) == 1 and len(a["tvs_objective"]["groups"][0]["slots"]) == 2
    assert a["tvs_objective"]["groups"][0]["calls"] == a["tvs_objective"]["groups"][0]["rounds"] + 1


def test_a_bad_split_on_one_rank_raises_on_every_rank_before_any_engine_exists():
    got = run_two([600, 437], "refuse")
    for r in (0, 1):
        assert got[r]["error"] == ("ValueError",
                                   "rank 1: CrossValidator: folds must hold one integer in [0, numFolds) per row")
        assert got[r]["made"] == 0


def _exchange_worker(rank, world, port, sizes, outq):
    try:
        os.environ["MASTER_ADDR"] = "127.0.0.1"
        os.environ["MASTER_PORT"] = str(port)
        dist.init_process_group("gloo", rank=rank, world_size=world)
        X, y = data()
        off = np.concatenate([[0], np.cumsum(sizes)])
        fold = kfold_assignment(N_ROWS, 4, 9)
        members = [(fold != k)[off[rank]:off[rank + 1]] for k in range(4)]
        plans = [D.ShardPlan([int((fold != k)[off[s]:off[s + 1]].sum()) for s in range(world)], rank, N_E)
                 for k in range(4)]
        Xe, ye, rows = D.exchange_sets(plans, members, torch.from_numpy(X[off[rank]:off[rank + 1]]),
                                       torch.from_numpy(y[off[rank]:off[rank + 1]]), dist.group.WORLD)
        dist.destroy_process_group()
        outq.put((rank, "ok", (Xe.numpy(), ye.numpy(), list(rows), [p.local_experts for p in plans],
                               [p.first for p in plans])))
    except Exception:                                                   # noqa: BLE001
        import traceback
        outq.put((rank, "error", traceback.format_exc()))


def test_exchange_sets_moves_every_row_once_per_set_to_its_block():
    sizes, world = [400, 0, 637], 3
    ctx = mp.get_context("spawn")
    outq = ctx.Queue()
    port = _free_port()
    procs = [ctx.Process(target=_exchange_worker, args=(r, world, port, sizes, outq), daemon=True) for r in range(world)]
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
    X, y = data()
    fold = kfold_assignment(N_ROWS, 4, 9)
    for r, (Xe, ye, rows, experts, firsts) in got.items():
        at = np.concatenate([[0], np.cumsum(rows)])
        for k in range(4):
            set_rows = np.flatnonzero(fold != k)
            reference = group_for_experts(len(set_rows), N_E)
            block_X, block_y = Xe[at[k]:at[k + 1]], ye[at[k]:at[k + 1]]
            for q, e in enumerate(range(firsts[k][r], firsts[k][r + 1])):
                assert block_X[q::experts[k]].tobytes() == X[set_rows[reference[e]]].tobytes()
                assert block_y[q::experts[k]].tobytes() == y[set_rows[reference[e]]].tobytes()
