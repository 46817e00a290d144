"""The NCCL communicator on real GPUs: every all-reducing entry of sgp.h across ranks (run on an H100 box: `pytest -m gpu`).

A module-scoped pool of `world` spawned workers runs each case, worker r on cuda:r.  Rank 0 makes the communicator id,
the parent hands it to every worker, and each worker attaches it with `comm_init` to one context.  Each worker also keeps
a second context on the same device without a communicator: on it the worker computes its rank-local result for the
same inputs.  A case is a module-level scenario function; the workers send back numpy outputs, the errors they met (class
and message) and launch counts.  Every scenario makes the same sequence of collective calls on every rank: a rank's bad
input appears only where the library carries it in the reduced status word, never as a refusal that returns before the
all-reduce (those leave the peers blocked in ncclAllReduce; sgp.h makes avoiding them the caller's obligation).

Three checks for every reducing call, each sharp for a different mistake:
  1. the same bits on every rank (the status decision and the per-rank tails rest on it);
  2. each rank's output against the element-wise sum of the no-communicator results, within
     (world - 1) 2^-53 sum_r |out_r| (at two ranks both sides are one correctly rounded addition): this catches packing,
     count and offset slips that an oracle tolerance hides;
  3. the fp64 oracle on the union of the ranks' data, at the tolerances of the single-context tests
     (test_gpu_entry_points.py, test_gpu_objectives.py).
With a communicator and world > 1 each reducing call makes exactly one launch more than the same call without one.

On one GPU the same scenarios run on a communicator of one rank (the no-communicator bits and launch counts), and the
constructions that give one rank a bad shard run with that rank's data alone, so their premises are checked too.  The
cases of two or more ranks are skipped when fewer GPUs are visible.  A case that passes its deadline kills the pool and
fails; no worker outlives the module.
"""
import multiprocessing as mp
import queue
import time
import traceback

import numpy as np
import pytest

import oracle
import oracle.regression
import spark_gp_b200 as sg
from spark_gp_b200 import _native as N
from oracle.classification import classification_likelihood_and_gradient
from test_gpu_entry_points import TiledOracle, oracle_rows
from test_gpu_objectives import check_components, laplace_atol, oracle_bcm
from test_host_logic import bcm_variant

pytestmark = pytest.mark.gpu

DEADLINE = 240.0                        # seconds for one case on every rank
TOL_STATS, TOL_PRED, TOL_NLL, RTOL_G, RTOL_LAP = 1e-6, 1e-5, 1e-9, 1e-12, 1e-9
TOL_LAP = 1e-6                          # the Newton loop's tolerance
U = 2.0 ** -53


def visible_gpus():
    import torch
    return torch.cuda.device_count() if torch.cuda.is_available() else 0


GPUS = visible_gpus()
BIG_WORLD = max(1, min(GPUS, 8))
STATS_WORLDS = sorted({1, 2, BIG_WORLD})     # the statistics cases also run on every visible GPU (up to 8)


def bits(a):
    return np.ascontiguousarray(a, dtype=np.float64).view(np.int64)


# ---------------- the rank harness ---------------------------------------------------------------------------------------
class Rank:
    """What a scenario sees: its rank, the world, the context with the communicator and the one without, and the rank
    whose data it uses (its own, unless a one-GPU case runs another rank's shard)."""

    def __init__(self, rank, world, eng, solo, data_rank):
        self.rank, self.world, self.eng, self.solo, self.data_rank = rank, world, eng, solo, data_rank


def attempt(fn, *args):
    """("ok", result) or (exception class name, message): the scenarios report the errors they expect."""
    try:
        return "ok", fn(*args)
    except Exception as ex:                                     # noqa: BLE001 -- compared by name in the parent
        return type(ex).__name__, str(ex)


def _serve(rank, world, inq, outq):
    """A worker: one communicator context and one plain context on cuda:rank, serving requests until None arrives."""
    eng = solo = None
    try:
        import torch
        torch.cuda.set_device(rank)
        eng, solo = sg.ProjectedProcessEngine(rank), sg.ProjectedProcessEngine(rank)
        while True:
            msg = inq.get()
            if msg is None:
                break
            kind, arg = msg
            try:
                if kind == "uid":
                    out = sg.ProjectedProcessEngine.comm_unique_id()
                elif kind == "init":
                    eng.comm_init(arg, rank, world)
                    out = None
                else:
                    name, data_rank, kw = arg
                    out = globals()[name](Rank(rank, world, eng, solo, data_rank), **kw)
                outq.put((rank, "ok", out))
            except Exception:                                   # noqa: BLE001 -- reported to the parent
                outq.put((rank, "error", traceback.format_exc()))
    except BaseException:                                       # noqa: BLE001 -- start-up failure, reported
        outq.put((rank, "error", traceback.format_exc()))
    finally:
        for e in (eng, solo):
            if e is not None:
                e.close()


class RankPool:
    def __init__(self, world):
        ctx = mp.get_context("spawn")
        self.world, self.broken = world, None
        self.outq = ctx.Queue()
        self.inq = [ctx.Queue() for _ in range(world)]
        self.procs = [ctx.Process(target=_serve, args=(r, world, self.inq[r], self.outq), daemon=True)
                      for r in range(world)]
        try:
            for p in self.procs:
                p.start()
            uid = self._ask([0], [("uid", None)], "communicator id")[0]
            self._ask(range(world), [("init", uid)] * world, "comm_init")
        except BaseException:
            self.kill()
            raise

    def _ask(self, ranks, msgs, what):
        """Sends msgs[i] to rank ranks[i] and waits for every answer, at most DEADLINE seconds in all."""
        if self.broken:
            pytest.fail("the rank pool is unusable: " + self.broken)
        ranks = list(ranks)
        for r, m in zip(ranks, msgs):
            self.inq[r].put(m)
        got, end = {}, time.monotonic() + DEADLINE
        while len(got) < len(ranks):
            try:
                r, status, out = self.outq.get(timeout=1.0)
            except queue.Empty:
                dead = [r for r, p in enumerate(self.procs) if not p.is_alive()]
                late = time.monotonic() > end
                if dead or late:
                    self.broken = "%s: %s (ranks that answered: %s)" % (
                        what, "workers %s exited" % dead if dead else "past the %.0f s deadline" % DEADLINE, sorted(got))
                    self.kill()
                    pytest.fail(self.broken + "; every worker was killed")
                continue
            if status != "ok":
                # the other ranks may be blocked in a collective this rank never reached: do not wait for them
                self.broken = "%s: rank %d raised" % (what, r)
                self.kill()
                pytest.fail("%s:\n%s" % (self.broken, out))
            got[r] = out
        return [got[r] for r in ranks]

    def run(self, scenario, as_ranks=None, **kw):
        """Runs `scenario` on every rank; rank r uses the data of rank as_ranks[r] (default: its own)."""
        as_ranks = list(range(self.world)) if as_ranks is None else as_ranks
        return self._ask(range(self.world), [("run", (scenario, as_ranks[r], kw)) for r in range(self.world)], scenario)

    def kill(self):
        for p in self.procs:
            if p.is_alive():
                p.kill()
        for p in self.procs:
            p.join(timeout=30)

    def close(self):
        for q, p in zip(self.inq, self.procs):
            if p.is_alive():
                q.put(None)
        for p in self.procs:
            p.join(timeout=60)
        self.kill()


@pytest.fixture(scope="module")
def pools():
    made = {}

    def get(world):
        if world > GPUS:
            pytest.skip("needs %d GPUs, %d visible" % (world, GPUS))
        if world not in made:
            made[world] = RankPool(world)
        return made[world]

    yield get
    for p in made.values():
        p.close()


# ---------------- the checks -------------------------------------------------------------------------------------------
def check_reduced(what, outs, locs):
    """Checks 1 and 2 on one output: outs[r] rank r's reduced array, locs[r] its no-communicator array.  Returns the
    largest deviation from the sum in ulps of the sum."""
    world = len(outs)
    outs = [np.asarray(o, dtype=np.float64) for o in outs]
    locs = [np.asarray(l, dtype=np.float64) for l in locs]
    for r in range(1, world):
        assert np.array_equal(bits(outs[r]), bits(outs[0])), "%s: rank %d's bits differ from rank 0's" % (what, r)
    ref = locs[0].copy()
    for l in locs[1:]:
        ref = ref + l
    bound = (world - 1) * U * sum(np.abs(l) for l in locs)
    dev = np.abs(outs[0] - ref)
    worst = int(np.argmax(dev - bound))
    assert np.all(dev <= bound), "%s: element %d deviates from sum_r out_r by %.3e > %.3e" % (
        what, worst, dev.flat[worst], bound.flat[worst])
    ulps = float(np.max(dev / np.spacing(np.maximum(np.abs(ref), np.finfo(float).tiny))))
    return ulps, bool(np.array_equal(bits(outs[0]), bits(ref)))


def check_launches(what, extra):
    """Launches of ONE reducing call with the communicator minus without, per rank."""
    world = len(extra)
    assert extra == [1 if world > 1 else 0] * world, "%s: launch-count differences %s" % (what, extra)


def report(what, world, ulps, exact, err, extra):
    print("%-34s world=%d: max |out - sum_r out_r| = %.1f ulp (bits %s), oracle err %s, launches +%d" % (
        what, world, ulps, "equal" if exact else "differ", err, extra[0]))


def rel(a, b):
    return float(np.abs(np.asarray(a) - np.asarray(b)).max() / max(np.abs(np.asarray(b)).max(), 1e-300))


# ---------------- statistics: data ---------------------------------------------------------------------------------------
MODES = {"auto": N.SGP_PREC_AUTO, "i8": N.SGP_PREC_I8, "i8_direct": N.SGP_PREC_I8_DIRECT, "f64": N.SGP_PREC_F64,
         "f64_strict": N.SGP_PREC_F64_STRICT}
ST_N, ST_D, ST_M = 150_037, 16, 256       # 2344 units of 64 points and a partial one
AUTO_MIN_POINTS = 32768                   # AUTO runs the int8 Gram on an accumulate call of at least this many points


def stats_points(world):
    """Points of an every-mode case: ST_N, or enough that every rank of the uneven plans still holds more than
    AUTO_MIN_POINTS (the "tiny" rank aside), so that AUTO's int8 path runs at every world."""
    return max(ST_N, (world - 1) * 45_000 + 37)


def ard_stats(d):
    beta = np.full(d, np.sqrt(18.0 / d))
    return (1.0 * sg.ARDRBFKernel(beta) + sg.const(1.0) * sg.EyeKernel() + sg.const(1e-4) * sg.EyeKernel(),
            lambda: 1.0 * oracle.ARDRBFKernel(beta) + oracle.const(1.0) * oracle.EyeKernel()
            + oracle.const(1e-4) * oracle.EyeKernel())


def stats_data(seed, n, d, m):
    """Bench-like points X ~ U[0,1)^d (fp32), labels, an active set drawn from X, held-out points."""
    rng = np.random.default_rng(seed)
    X = rng.random((n, d), dtype=np.float32)
    y = np.sin(X.astype(np.float64).sum(1)) + 0.1 * rng.standard_normal(n)
    Z = X[rng.permutation(n)[:m]].astype(np.float64)
    return X, y, Z, rng.random((400, d))


def shard_bounds(plan, n, world):
    """(lo, hi) of every rank.  even: equal cuts; ragged: cuts 37 points past a unit edge; empty: the last rank holds no
    point; tiny: rank 0 holds 50 points, less than one unit."""
    if world == 1:
        return [(0, n)]
    if plan == "even":
        cuts = [r * n // world for r in range(world + 1)]
    elif plan == "ragged":
        cuts = [0] + [(r * n // world) // 64 * 64 + 37 for r in range(1, world)] + [n]
    elif plan == "empty":
        cuts = [r * n // (world - 1) for r in range(world)] + [n]
    elif plan == "tiny":
        cuts = [0] + [50 + (r - 1) * (n - 50) // (world - 1) for r in range(1, world)] + [n]
    else:
        raise ValueError(plan)
    return list(zip(cuts[:-1], cuts[1:]))


_ORACLE = {}


def stats_oracle(seed, n, d, m):
    """(G0, b0, mean0, var0) of the oracle on every point of stats_data(seed, n, d, m)."""
    key = (seed, n, d, m)
    if key not in _ORACLE:
        X, y, Z, Xt = stats_data(seed, n, d, m)
        _, ok = ard_stats(d)
        K = oracle_rows(ok, Z, X)
        _ORACLE[key] = (K.T @ K, K.T @ y) + posterior(ok, Z, K.T @ K, K.T @ y, Xt)
    return _ORACLE[key]


def posterior(ok, Z, G0, b0, Xt):
    k0 = ok().set_hyperparameters(ok().get_hyperparameters()).set_training_vectors(Z)
    mv0, mm0 = oracle.get_magic_vector(k0, G0, b0)
    return oracle.GaussianProjectedProcessRawPredictor(mv0, mm0, k0).predict_many(Xt)


# ---------------- statistics: scenario -----------------------------------------------------------------------------------
def _window(e, k, Z, X, y, mode, entry, rank):
    """One begin .. finish window on context e: (G, b, path, launches)."""
    import torch
    e.set_precision(mode)
    before = e.launch_count()
    e.begin(k, Z)
    if entry == "host":
        e.accumulate(X, y)
    elif len(X) > 0:
        cuda = torch.device("cuda", rank)
        Xd, yd = torch.from_numpy(np.ascontiguousarray(X)).to(cuda), torch.from_numpy(y).to(cuda)
        torch.cuda.current_stream(cuda).synchronize()
        e.accumulate_ptr(Xd.data_ptr(), Xd.dtype == torch.float32, yd.data_ptr(), len(X), device=True)
    path = e.last_path()
    G, b = e.finish()
    return G, b, path, e.launch_count() - before


def sc_stats(w, windows, tail=True):
    """Each window (a dict of stats_data's arguments, mode, entry, dtype, shard plan) on the communicator context and
    on the plain one; after the last, the tail and a prediction on the communicator context."""
    out = []
    for win in windows:
        X, y, Z, Xt = stats_data(win["seed"], win["n"], win["d"], win["m"])
        lo, hi = shard_bounds(win["plan"], win["n"], w.world)[w.data_rank]
        Xs, ys = X[lo:hi].astype(win["dtype"]), y[lo:hi]
        k, _ = ard_stats(win["d"])
        mode = MODES[win["mode"]]
        G, b, path, launches = _window(w.eng, k, Z, Xs, ys, mode, win["entry"], w.rank)
        Gl, bl, path_l, launches_l = _window(w.solo, k, Z, Xs, ys, mode, win["entry"], w.rank)
        out.append(dict(G=G, b=b, Gl=Gl, bl=bl, path=path, path_l=path_l, extra=launches - launches_l, n=hi - lo))
    res = dict(windows=out)
    if tail:
        mv, mm = w.eng.magic()
        mean, var = w.eng.predict(Xt)
        res.update(mv=mv, mm=mm, mean=mean, var=var, tail_path=w.eng.last_tail_path())
    return res


def check_stats(res, windows, label):
    world = len(res)
    for i, win in enumerate(windows):
        what = "stats %s %s/%s %s m=%d" % (win["mode"], win["entry"], np.dtype(win["dtype"]).name, win["plan"], win["m"])
        rs = [r["windows"][i] for r in res]
        for r in rs:
            if r["n"] == 0:
                continue                                     # no launch: last_path() is the previous window's
            assert r["path"] == r["path_l"], what
            if win["mode"] == "auto" and r["n"] >= AUTO_MIN_POINTS:
                assert r["path"] == N.SGP_PREC_I8, "%s: AUTO took path %d" % (what, r["path"])
            elif win["mode"] != "auto" and r["n"] > 0:
                assert r["path"] == MODES[win["mode"]], what
        ug, eg = check_reduced(what + " G", [r["G"] for r in rs], [r["Gl"] for r in rs])
        ub, eb = check_reduced(what + " b", [r["b"] for r in rs], [r["bl"] for r in rs])
        check_launches(what, [r["extra"] for r in rs])
        G0, b0, _, _ = stats_oracle(win["seed"], win["n"], win["d"], win["m"])
        dG, db = rel(rs[0]["G"], G0), rel(rs[0]["b"], b0)
        report("%s [%s]" % (what, label), world, max(ug, ub), eg and eb, "dG=%.1e db=%.1e" % (dG, db), [rs[0]["extra"]])
        assert dG < TOL_STATS and db < TOL_STATS, what
        assert np.array_equal(rs[0]["G"], rs[0]["G"].T)
    if "mv" in res[0]:
        for key in ("mv", "mm", "mean", "var"):
            for r in range(1, world):
                assert np.array_equal(bits(res[r][key]), bits(res[0][key])), "tail %s: rank %d differs" % (key, r)
        win = windows[-1]
        _, _, mean0, var0 = stats_oracle(win["seed"], win["n"], win["d"], win["m"])
        em, ev = rel(res[0]["mean"], mean0), float(np.abs(res[0]["var"] / var0 - 1).max())
        print("tail + predict world=%d: same bits on every rank, dmean=%.1e dvar=%.1e" % (world, em, ev))
        assert em < TOL_PRED and ev < TOL_PRED


def win(mode, entry="host", dtype=np.float32, plan="even", m=ST_M, seed=11, n=ST_N, d=ST_D):
    return dict(seed=seed, n=n, d=d, m=m, mode=mode, entry=entry, dtype=dtype, plan=plan)


ENTRIES = [("host", np.float32), ("device", np.float64), ("host", np.float64), ("device", np.float32)]


def _plans(world):
    return ["even"] if world == 1 else ["ragged", "empty", "tiny"]


@pytest.mark.parametrize("world", STATS_WORLDS)
@pytest.mark.parametrize("entry,dtype", ENTRIES, ids=["host-fp32", "device-fp64", "host-fp64", "device-fp32"])
@pytest.mark.parametrize("mode", list(MODES))
def test_stats_every_mode(pools, world, mode, entry, dtype):
    """sgp_stats_finish in every precision mode, host and device entry, fp32 and fp64 points, on uneven shards (a
    partial unit at the end of a shard, a rank with no point, a rank with fewer points than one unit), then the tail."""
    pool = pools(world)
    for plan in _plans(world):
        windows = [win(mode, entry, dtype, plan, n=stats_points(world))]
        check_stats(pool.run("sc_stats", windows=windows), windows, plan)


@pytest.mark.parametrize("world", STATS_WORLDS)
def test_stats_windows_with_changing_m(pools, world):
    """Several windows on one communicator, m = 64 -> 1000 -> 129: the reduced count mm + m + 1 follows m."""
    windows = [win("f64", m=64, plan="ragged"), win("i8", "device", m=1000, plan="tiny", seed=12),
               win("f64_strict", m=129, plan="empty", seed=13)]
    check_stats(pools(world).run("sc_stats", windows=windows), windows, "sequence")


# ---------------- statistics: bench-like shards ----------------------------------------------------------------------------
BENCH = {"configs1": (20480, 16, 1000, 49), "configs3": (20480, 32, 2000, 61)}   # block, d, m, copies per rank


def bench_block(name, rank):
    """Rank r's base block; Z is drawn from rank 0's block, so every rank has the same active set."""
    nb, d, m, reps = BENCH[name]
    rng = np.random.default_rng(1000 + rank)
    Xb = rng.random((nb, d), dtype=np.float32)
    yb = np.sin(Xb.astype(np.float64).sum(1)) + 0.1 * rng.standard_normal(nb)
    Z = np.random.default_rng(1000).random((nb, d), dtype=np.float32)[:m].astype(np.float64)
    return Xb, yb, Z


def sc_bench(w, name, mode):
    import torch
    nb, d, m, reps = BENCH[name]
    Xb, yb, Z = bench_block(name, w.data_rank)
    order = np.random.default_rng(7 + w.data_rank).permutation(nb * reps)
    X, y = np.tile(Xb, (reps, 1))[order], np.tile(yb, reps)[order]
    k, _ = ard_stats(d)
    out = {}
    for tag, e in (("", w.eng), ("l", w.solo)):
        G, b, path, launches = _window(e, k, Z, X, y, MODES[mode], "device", w.rank)
        out.update({"G" + tag: G, "b" + tag: b, "path" + tag: path, "launches" + tag: launches})
    torch.cuda.empty_cache()
    return out


@pytest.mark.parametrize("name,world", [("configs1", BIG_WORLD), ("configs3", 8)])
def test_stats_bench_shards(pools, name, world):
    """bench.py's per-GPU shard on every visible GPU (configs3: 1.25M x 32, m = 2000, two int8 plane windows, with 8
    GPUs): AUTO through the device entry, each shard 49 / 61 shuffled copies of its rank's block (TiledOracle)."""
    pool = pools(world)
    res = pool.run("sc_bench", name=name, mode="auto")
    nb, d, m, reps = BENCH[name]
    assert all(r["path"] == r["pathl"] == N.SGP_PREC_I8 for r in res)
    ug, eg = check_reduced(name + " G", [r["G"] for r in res], [r["Gl"] for r in res])
    ub, eb = check_reduced(name + " b", [r["b"] for r in res], [r["bl"] for r in res])
    check_launches(name, [r["launches"] - r["launchesl"] for r in res])
    _, ok = ard_stats(d)
    G0, b0 = 0.0, 0.0
    for r in range(world):
        Xb, yb, Z = bench_block(name, r)
        Gr, br = TiledOracle(ok, Xb, yb, Z).stats(nb * reps)
        G0, b0 = G0 + Gr, b0 + br
    dG, db = rel(res[0]["G"], G0), rel(res[0]["b"], b0)
    report(name, world, max(ug, ub), eg and eb, "dG=%.1e db=%.1e" % (dG, db), [res[0]["launches"] - res[0]["launchesl"]])
    assert dG < TOL_STATS and db < TOL_STATS


# ---------------- statistics: one status on every rank ---------------------------------------------------------------------
def status_data(case, rank):
    """(X, y, Z, d) of one rank.  Rank 1 holds the shard only it cannot take on the int8 path:
    range: coordinates around 1e4, outside the fp16 operand range (forced I8);
    budget: a benign first staged chunk of 65536 points, later chunks x 12, over AUTO's magnitude budget;
    mixed: points x 6, whose scaled norms send AUTO's gate to the fp64 kernel."""
    d, m = {"range": (8, 256), "budget": (32, 128), "mixed": (8, 256)}[case]
    base = np.random.default_rng(500)
    Xa = base.random((65_536, d), dtype=np.float32)
    Z = Xa[:m].astype(np.float64)
    rng = np.random.default_rng(600 + rank)
    if rank != 1:
        X = rng.random((100_000, d), dtype=np.float32)
    elif case == "range":
        X = (rng.standard_normal((100_000, d)) * 1e4).astype(np.float32)
    elif case == "budget":
        X = np.vstack([Xa, rng.random((234_464, d), dtype=np.float32) * np.float32(12.0)])
    else:
        X = rng.random((100_000, d), dtype=np.float32) * np.float32(6.0)
    return X, rng.standard_normal(len(X)), Z, d


def sc_status(w, case):
    X, y, Z, d = status_data(case, w.data_rank)
    k, _ = ard_stats(d)
    e = w.eng
    out = {}
    mode = N.SGP_PREC_I8 if case == "range" else N.SGP_PREC_AUTO
    e.set_precision(mode)
    e.begin(k, Z)
    e.accumulate(X, y)
    out["path"] = e.last_path()
    out["finish"] = attempt(e.finish)
    out["finish_again"] = attempt(e.finish)
    out["magic"] = attempt(e.magic)
    if case == "range":
        out["f64"] = _window(e, k, Z, X, y, N.SGP_PREC_F64, "host", w.rank)
        out["f64_local"] = _window(w.solo, k, Z, X, y, N.SGP_PREC_F64, "host", w.rank)
    w.solo.set_precision(mode)
    w.solo.begin(k, Z)
    w.solo.accumulate(X, y)
    out["local_finish"] = attempt(w.solo.finish)
    return out


def status_oracle(case, ranks):
    G0, b0 = 0.0, 0.0
    for r in ranks:
        X, y, Z, d = status_data(case, r)
        K = oracle_rows(ard_stats(d)[1], Z, X)
        G0, b0 = G0 + K.T @ K, b0 + K.T @ y
    return G0, b0


@pytest.mark.parametrize("case", ["range", "budget"])
def test_one_rank_out_of_range_fails_every_rank(pools, case):
    """Only rank 1's shard is outside what the int8 path takes (forced I8: operand range; AUTO: the magnitude budget
    over the whole window).  Every rank raises OperandRangeError at finish, again at a repeated finish, and magic()
    without G_in is SGP_E_STATE on every rank.  A following F64 window on the same communicator matches the oracle."""
    res = pools(2).run("sc_status", case=case)
    assert [r["local_finish"][0] for r in res] == ["ok", "OperandRangeError"]      # the rank-local statuses differ
    for r in res:
        assert r["finish"][0] == r["finish_again"][0] == "OperandRangeError"
        assert r["magic"][0] == "TrainingVectorsNotInitializedException"
    assert res[0]["finish"][1] == res[1]["finish"][1]
    if case == "range":
        check_range_f64(res, [0, 1])


def check_range_f64(res, ranks):
    G, b = [r["f64"][0] for r in res], [r["f64"][1] for r in res]
    ug, eg = check_reduced("f64 after a range failure G", G, [r["f64_local"][0] for r in res])
    ub, eb = check_reduced("f64 after a range failure b", b, [r["f64_local"][1] for r in res])
    extra = [r["f64"][3] - r["f64_local"][3] for r in res]
    check_launches("f64 after a range failure", extra)
    G0, b0 = status_oracle("range", ranks)
    report("f64 window after SGP_E_RANGE", len(res), max(ug, ub), eg and eb,
           "dG=%.1e db=%.1e" % (rel(G[0], G0), rel(b[0], b0)), extra)
    assert rel(G[0], G0) < TOL_STATS and rel(b[0], b0) < TOL_STATS


@pytest.mark.parametrize("case,data_rank,status", [("range", 0, "ok"), ("range", 1, "OperandRangeError"),
                                                   ("budget", 0, "ok"), ("budget", 1, "OperandRangeError"),
                                                   ("mixed", 1, "ok")])
def test_status_constructions_on_one_rank(pools, case, data_rank, status):
    """The premises of the status cases, on a communicator of one rank: rank 1's shard alone fails (or, mixed, takes the
    fp64 kernel) and rank 0's does not; the status is the plain context's."""
    r = pools(1).run("sc_status", as_ranks=[data_rank], case=case)[0]
    assert r["finish"][0] == r["finish_again"][0] == r["local_finish"][0] == status
    if case == "mixed":
        assert r["path"] == N.SGP_PREC_F64
    elif data_rank == 0:
        assert r["path"] == N.SGP_PREC_I8
    if status != "ok":
        assert r["magic"][0] == "TrainingVectorsNotInitializedException"
    if case == "range":
        check_range_f64([r], [data_rank])


def test_mixed_int8_and_fp64_ranks_add_up(pools):
    """AUTO with rank 0 on the int8 path and rank 1's gate on the fp64 kernel: no error, last_path() differs between
    the ranks, and the summed G matches the oracle on the union."""
    res = pools(2).run("sc_stats_mixed")
    assert [r["path"] for r in res] == [N.SGP_PREC_I8, N.SGP_PREC_F64]
    ug, eg = check_reduced("mixed paths G", [r["G"] for r in res], [r["Gl"] for r in res])
    ub, eb = check_reduced("mixed paths b", [r["b"] for r in res], [r["bl"] for r in res])
    check_launches("mixed paths", [r["extra"] for r in res])
    G0, b0 = status_oracle("mixed", [0, 1])
    report("AUTO, int8 + fp64 ranks", 2, max(ug, ub), eg and eb,
           "dG=%.1e db=%.1e" % (rel(res[0]["G"], G0), rel(res[0]["b"], b0)), [res[0]["extra"]])
    assert rel(res[0]["G"], G0) < TOL_STATS and rel(res[0]["b"], b0) < TOL_STATS


def sc_stats_mixed(w):
    X, y, Z, d = status_data("mixed", w.data_rank)
    k, _ = ard_stats(d)
    G, b, path, launches = _window(w.eng, k, Z, X, y, N.SGP_PREC_AUTO, "host", w.rank)
    Gl, bl, _, launches_l = _window(w.solo, k, Z, X, y, N.SGP_PREC_AUTO, "host", w.rank)
    return dict(G=G, b=b, Gl=Gl, bl=bl, path=path, extra=launches - launches_l)


# ---------------- objectives ------------------------------------------------------------------------------------------------
def ard_obj(d, scale=1.3, eye=1e-2):
    """(library kernel factory, oracle kernel factory): setHyperparameters changes a kernel in place, so every slot
    gets a kernel of its own."""
    beta = np.linspace(0.6, 1.4, d) / np.sqrt(d)
    return (lambda: scale * sg.ARDRBFKernel(beta.copy()) + sg.const(eye) * sg.EyeKernel(),
            lambda: scale * oracle.ARDRBFKernel(beta.copy()) + oracle.const(eye) * oracle.EyeKernel())


def rbf_obj(eye):
    return (lambda: 1.0 * sg.RBFKernel(1.0) + sg.const(eye) * sg.EyeKernel(),
            lambda: 1.0 * oracle.RBFKernel(1.0) + oracle.const(eye) * oracle.EyeKernel())


# name: (entry, points per expert, experts per rank, d).  The BCM sizes pick the register (<= 128), shared-memory
# (<= 168) and LU variants; the Laplace ones the on-chip (<= 117) and global-memory kernels.
OBJ = {
    "bcm_register": ("bcm", 64, 3, 3), "bcm_shared": ("bcm", 150, 3, 3), "bcm_lu": ("bcm", 200, 3, 3),
    "bcm_breakdown": ("bcm", 40, 4, 2), "bcm_slots": ("bcm_slots", 60, 4, 3), "bcm_folds": ("bcm_folds", 50, 4, 3),
    "laplace": ("laplace", 40, 4, 3), "laplace_any_size": ("laplace_any_size", 200, 3, 3),
    "laplace_classes": ("classes", 40, 4, 3), "laplace_classes_any_size": ("classes_any_size", 150, 3, 3),
    "laplace_slots_any_size": ("slots_any_size", 60, 4, 3), "laplace_fold_slots": ("fold_slots", 117, 0, 3),
}
FOLD_SETS = [0, 2, 1, 0]
SLOT_MODES, SLOT_CLASSES = [2, 0], [1, 2]
FOLD_SLOT_SETS = [0, 1, 2]
THETA_STEPS = [1.0, 1.1, 0.9, 1.2]


def fold_slot_folds(rank):
    """608 points in folds of 140, 100 and 368: the sets hold 468, 508 and 240 points, as experts of at most 117 (on
    chip), 127 and 120 points (global memory) at datasetSizeForExpert = 117 -- one call, two launches, one collective.
    Odd ranks swap the first two folds, so set 0 runs on chip on even ranks and in global memory on odd ones (and set 1
    the other way round): the library sets the slots up in a rank-local order, and the sum must still add slot to slot."""
    return np.repeat([0, 1, 2], [100, 140, 368] if rank % 2 else [140, 100, 368]).astype(np.int32)


def obj_data(name, rank):
    """(X, y, kernel factory, oracle kernel factory) of one rank: its own points, disjoint from every other rank's."""
    entry, n_e, E, d = OBJ[name]
    rng = np.random.default_rng(7000 + 100 * rank + len(name))
    N_ = 608 if name == "laplace_fold_slots" else n_e * E
    if name == "bcm_breakdown":
        # well-separated points; rank 1 also holds a point 1e-9 from its point 0, in the same expert, so that with an
        # Eye term of 1e-30 its on-chip Cholesky breaks down and it runs LU, while every other rank stays on chip
        X = 3.0 * rng.standard_normal((N_, d))
        if rank == 1:
            X[E] = X[0] + 1e-9
        mk, ok = rbf_obj(1e-30)
        return X, np.sin(X.sum(1)), mk, ok
    X = rng.standard_normal((N_, d))
    if entry.startswith("bcm"):
        y = np.sin(X.sum(1)) + 0.3 * rng.standard_normal(N_)
        mk, ok = ard_obj(d)
    else:
        s = np.sin(2 * X[:, 0]) + 0.5 * X.sum(1) / np.sqrt(d) + 0.3 * rng.standard_normal(N_)
        y = np.digitize(s, [-0.5, 0.5]).astype(np.float64) if "classes" in entry or "slots" in entry \
            else (s > 0).astype(np.float64)
        mk, ok = ard_obj(d, scale=1.2)
    return X, y, mk, ok


def kernels_at(mk, n):
    """n fresh kernels of factory mk, slot i at THETA_STEPS[i] times its hyper-parameters."""
    return [mk().setHyperparameters(mk().getHyperparameters() * THETA_STEPS[i]) for i in range(n)]


def run_objective(e, name, X, y, mk, data_rank):
    """One objective case on context e: (list of reduced outputs, list of mode vectors, launches of each reducing call,
    paths)."""
    entry, n_e, E, d = OBJ[name]
    outs, modes, paths, launches = [], [], [], []

    def call(fn, *args):
        before = e.launch_count()
        v, g = fn(*args)
        launches.append(e.launch_count() - before)
        outs.append(np.column_stack([np.atleast_1d(v), np.atleast_2d(g)]))

    if entry == "bcm_folds" or entry == "fold_slots":
        folds = np.arange(len(X)) % 3 if entry == "bcm_folds" else fold_slot_folds(data_rank)
        e.experts_upload_folds(X, y, folds, 3, n_e)
    else:
        assert e.experts_upload_grouped(X, y, n_e) == E
    if entry == "bcm":
        call(e.bcm_nll, mk())
        paths.append(e.last_bcm_path())
    elif entry == "bcm_slots":
        call(e.bcm_nll_slots, kernels_at(mk, 3))
        paths.append(e.last_bcm_path())
    elif entry == "bcm_folds":
        call(e.bcm_nll_folds, FOLD_SETS, kernels_at(mk, len(FOLD_SETS)))
        paths.append(e.last_bcm_path())
    elif entry in ("laplace", "laplace_any_size"):
        fn = e.laplace_nll if entry == "laplace" else e.laplace_nll_any_size
        for kk in kernels_at(mk, 2):                                  # the second call warm-starts from the first's modes
            call(fn, kk, TOL_LAP)
            paths.append(e.last_laplace_path())
            modes.append(e.experts_f(len(X)))
    elif entry in ("classes", "classes_any_size"):
        fn = e.laplace_nll_classes if entry == "classes" else e.laplace_nll_classes_any_size
        call(fn, 3, [0, 1, 2], kernels_at(mk, 3), TOL_LAP)
        paths.append(e.last_laplace_path())
        modes += [e.experts_f_class(c, len(X)) for c in range(3)]
    elif entry == "slots_any_size":
        call(e.laplace_nll_slots_any_size, 3, SLOT_MODES, SLOT_CLASSES, kernels_at(mk, 2), TOL_LAP)
        paths.append(e.last_laplace_path())
        modes += [e.experts_f_slot(s, len(X)) for s in SLOT_MODES]
    elif entry == "fold_slots":
        call(e.laplace_nll_fold_slots_any_size, 3, [0, 1, 2], FOLD_SLOT_SETS, [1, 1, 1], kernels_at(mk, 3), TOL_LAP)
        folds = fold_slot_folds(data_rank)
        modes += [e.experts_f_fold_slot(s, s, int(np.sum(folds != s))) for s in FOLD_SLOT_SETS]
    return outs, modes, launches, paths


def sc_objective(w, name):
    X, y, mk, _ = obj_data(name, w.data_rank)
    outs, modes, launches, paths = run_objective(w.eng, name, X, y, mk, w.data_rank)
    outs_l, modes_l, launches_l, paths_l = run_objective(w.solo, name, X, y, mk, w.data_rank)
    return dict(outs=outs, modes=modes, outs_l=outs_l, modes_l=modes_l, extra=[a - b for a, b in zip(launches, launches_l)],
                paths=paths,
                paths_l=paths_l, n_calls=len(outs))


def oracle_laplace(X, yb, n_e, ofac, theta, fs=None):
    experts = oracle.get_expert_labels_and_kernels(X, yb, ofac, n_e)
    fs = [np.zeros(len(ye)) for ye, _ in experts] if fs is None else fs
    v0, g0 = 0.0, np.zeros(len(theta))
    for (ye, ke), f in zip(experts, fs):
        v, g = classification_likelihood_and_gradient(ye, f, ke, theta, TOL_LAP)
        v0 += v
        g0 = g0 + g
    return v0, g0, laplace_atol(experts, theta), fs


def objective_oracle(name, ranks):
    """Per reducing call, per slot: (value, gradient, gradient atol, rtol) of the oracle over the union of the ranks'
    experts."""
    entry, n_e, E, d = OBJ[name]
    per_call = []
    for r in ranks:
        X, y, mk, ok = obj_data(name, r)
        thetas = [kk.getHyperparameters() for kk in kernels_at(mk, 4)]
        calls = []
        if entry == "bcm":
            calls.append([oracle_bcm(X, y, n_e, ok, thetas[0]) + (RTOL_G,)])
        elif entry == "bcm_slots":
            calls.append([oracle_bcm(X, y, n_e, ok, thetas[s]) + (RTOL_G,) for s in range(3)])
        elif entry == "bcm_folds":
            f = np.arange(len(X)) % 3
            calls.append([oracle_bcm(X[f != st], y[f != st], n_e, ok, thetas[s]) + (RTOL_G,)
                          for s, st in enumerate(FOLD_SETS)])
        elif entry in ("laplace", "laplace_any_size"):
            v, g, a, fs = oracle_laplace(X, y, n_e, ok, thetas[0])
            calls.append([(v, g, a, RTOL_LAP)])
            v, g, a, _ = oracle_laplace(X, y, n_e, ok, thetas[1], fs)
            calls.append([(v, g, a, RTOL_LAP)])
        elif entry in ("classes", "classes_any_size"):
            calls.append([oracle_laplace(X, (y == c).astype(np.float64), n_e, ok, thetas[c])[:3] + (RTOL_LAP,)
                          for c in range(3)])
        elif entry == "slots_any_size":
            calls.append([oracle_laplace(X, (y == c).astype(np.float64), n_e, ok, thetas[i])[:3] + (RTOL_LAP,)
                          for i, c in enumerate(SLOT_CLASSES)])
        elif entry == "fold_slots":
            f = fold_slot_folds(r)
            calls.append([oracle_laplace(X[f != st], (y[f != st] == 1).astype(np.float64), n_e, ok, thetas[i])[:3]
                          + (RTOL_LAP,) for i, st in enumerate(FOLD_SLOT_SETS)])
        per_call.append(calls)
    union = []
    for c in range(len(per_call[0])):
        slots = []
        for s in range(len(per_call[0][c])):
            parts = [per_call[r][c][s] for r in range(len(ranks))]
            slots.append((sum(p[0] for p in parts), sum(p[1] for p in parts), sum(p[2] for p in parts), parts[0][3]))
        union.append(slots)
    return union


def check_objective(name, res, ranks, with_oracle=True):
    world = len(res)
    for r in res:
        assert r["paths"] == r["paths_l"], name                     # the dispatch is rank-local and unchanged
        assert len(r["modes"]) == len(r["modes_l"])
        for f, fl in zip(r["modes"], r["modes_l"]):                # the latent modes stay rank-local: bit for bit
            assert np.array_equal(bits(f), bits(fl)), "%s: rank-local modes differ" % name
    union = objective_oracle(name, ranks) if with_oracle else None
    for c in range(res[0]["n_calls"]):
        what = "%s call %d" % (name, c)
        check_launches(what, [r["extra"][c] for r in res])
        ulps, exact = check_reduced(what, [r["outs"][c] for r in res], [r["outs_l"][c] for r in res])
        err = "not compared"
        if union is not None:
            out = res[0]["outs"][c]
            worst_v, worst_g = 0.0, 0.0
            for s, (v0, g0, atol, rtol) in enumerate(union[c]):
                assert abs(out[s, 0] - v0) <= TOL_NLL * abs(v0), "%s slot %d: value %r vs oracle %r" % (what, s,
                                                                                                          out[s, 0], v0)
                worst_v = max(worst_v, abs(out[s, 0] - v0) / abs(v0))
                worst_g = max(worst_g, check_components(out[s, 1:], g0, atol, rtol, "%s slot %d" % (what, s)))
            err = "dnll=%.1e grad err/bound=%.1e" % (worst_v, worst_g)
        report(what, world, ulps, exact, err, [res[0]["extra"][c]])


OBJ_CASES = [n for n in OBJ if n != "bcm_breakdown"]


@pytest.mark.parametrize("world", [1, 2])
@pytest.mark.parametrize("name", OBJ_CASES)
def test_objectives(pools, world, name):
    """Each of the nine reducing objective entries (and sgp_bcm_nll on all three variants), every rank on its own
    experts: same bits, the sum of the no-communicator rows, the oracle on the union of the experts, one more launch,
    and the latent modes of every store equal to the no-communicator context's, bit for bit."""
    res = pools(world).run("sc_objective", name=name)
    entry = OBJ[name][0]
    if name in ("bcm_register", "bcm_shared", "bcm_lu"):
        # last_bcm_path() tells on chip from LU only: the dispatch rule (pinned in test_host_logic.py) names the variant
        assert bcm_variant(OBJ[name][1], 1, OBJ[name][3]).startswith(
            {"bcm_register": "reg", "bcm_shared": "smem", "bcm_lu": "lu"}[name])
    want = {"bcm_lu": 1}.get(name, 0) if entry.startswith("bcm") else (0 if OBJ[name][1] <= 117 else 1)
    if entry != "fold_slots":
        assert all(p == want for r in res for p in r["paths"]), (name, [r["paths"] for r in res])
    check_objective(name, res, list(range(world)))


def test_fold_slots_of_an_odd_rank_alone(pools):
    """The premise of the fold-slot case's second rank, on a communicator of one rank: with its first two folds swapped,
    set 0 runs in global memory and set 1 on chip, and the slots still come back in list order, on the oracle."""
    res = pools(1).run("sc_objective", as_ranks=[1], name="laplace_fold_slots")
    check_objective("laplace_fold_slots", res, [1])


@pytest.mark.parametrize("world,as_ranks", [(1, [0]), (1, [1]), (2, None)])
def test_bcm_breakdown_on_one_rank(pools, world, as_ranks):
    """A Cholesky breakdown in rank 1's experts only: that rank runs LU, the others stay on chip, and the rows add up.
    (On one GPU: each rank's experts alone take the path the two-rank case relies on.)  Rank 1's kernel matrix has
    condition ~1e18, where neither LU nor the oracle's LU determines the objective to TOL_NLL, so the sum is pinned on
    the no-communicator results (check 2) and only the on-chip ranks' own results are compared with the oracle."""
    res = pools(world).run("sc_objective", as_ranks=as_ranks, name="bcm_breakdown")
    ranks = as_ranks or list(range(world))
    assert [r["paths"] for r in res] == [[1 if rk == 1 else 0] for rk in ranks]
    check_objective("bcm_breakdown", res, ranks, with_oracle=False)
    for r, rk in zip(res, ranks):
        if rk == 1:
            continue
        (v0, g0, atol, rtol), = objective_oracle("bcm_breakdown", [rk])[0]
        local = r["outs_l"][0][0]
        assert abs(local[0] - v0) <= TOL_NLL * abs(v0), (rk, local[0], v0)
        check_components(local[1:], g0, atol, rtol, "bcm_breakdown rank %d on chip" % rk)


# ---------------- objectives: one failure, every rank ---------------------------------------------------------------------
# case: (exception, the slots that fail on rank 1, the name in the message).  The "_last" cases fail only the last listed
# slot, whose status word is the last double the all-reduce carries: a count a few doubles short loses it.
FAILURES = {"singular": ("MatrixSingularException", [1], "slot 1:"),
            "singular_last": ("MatrixSingularException", [2], "slot 2:"),
            "not_pd": ("NotPositiveDefiniteException", [1, 2], "mode slot 3:"),
            "not_pd_last": ("NotPositiveDefiniteException", [2], "mode slot 1:")}


def sc_objective_failure(w, case):
    rng = np.random.default_rng(900 + w.data_rank)
    failing = FAILURES[case][1] if w.data_rank == 1 else []
    out = {}
    if case.startswith("singular"):
        # every point of rank 1 equal and no Eye term in a failing slot: an all-ones kernel matrix, singular on LU as well
        X = np.zeros((200, 2)) if w.data_rank == 1 else 3.0 * rng.standard_normal((200, 2))
        y = rng.standard_normal(200)
        mk = lambda c: 1.0 * sg.RBFKernel(1.0) + sg.const(c) * sg.EyeKernel()
        for tag, e in (("comm", w.eng), ("local", w.solo)):
            e.experts_upload_grouped(X, y, 50)
            out[tag] = attempt(e.bcm_nll_slots, [mk(0.0 if s in failing else 1e-2) for s in range(3)])
    else:
        # NaN hyper-parameters in the failing slots (mode slots 0, 3, 1 listed) on rank 1 only: B is not PD there
        X = rng.standard_normal((300, 3))
        y = (X[:, 0] > 0).astype(np.float64)
        mk, _ = ard_obj(3, scale=1.2)
        t = mk().getHyperparameters()
        bad = np.concatenate([t[:1], np.full(len(t) - 1, np.nan)])
        for tag, e in (("comm", w.eng), ("local", w.solo)):
            e.experts_upload_folds(X, y, np.arange(300) % 3, 3, 50)
            out[tag] = attempt(e.laplace_nll_fold_slots_any_size, 4, [0, 3, 1], [0, 1, 2], [1, 1, 1],
                               [mk().setHyperparameters(bad if s in failing else t * (1 + 0.1 * s)) for s in range(3)],
                               TOL_LAP)
    return out


@pytest.mark.parametrize("case", list(FAILURES))
def test_failure_on_one_rank_reaches_every_rank(pools, case):
    """A singular BCM slot, or a Laplace B that is not PD, on rank 1 only: every rank raises the same exception naming
    the same slot; rank 0's plain context does not."""
    exc, _, match = FAILURES[case]
    res = pools(2).run("sc_objective_failure", case=case)
    assert res[0]["local"][0] == "ok" and res[1]["local"][0] == exc
    for r in res:
        assert r["comm"][0] == exc and match in r["comm"][1], r["comm"]
    assert res[0]["comm"][1] == res[1]["comm"][1]


@pytest.mark.parametrize("data_rank", [0, 1])
@pytest.mark.parametrize("case", list(FAILURES))
def test_failure_constructions_on_one_rank(pools, case, data_rank):
    """The premises of the failure cases on a communicator of one rank: rank 1's data fail alone with the expected
    name, rank 0's do not."""
    exc, _, match = FAILURES[case]
    r = pools(1).run("sc_objective_failure", as_ranks=[data_rank], case=case)[0]
    want = "ok" if data_rank == 0 else exc
    assert r["comm"][0] == r["local"][0] == want
    if want != "ok":
        assert r["comm"][1] == r["local"][1] and match in r["comm"][1]


# ---------------- entries that ignore the communicator --------------------------------------------------------------------
def run_local_entries(e, rank, data_rank):
    """Every rank-local entry on this rank's own inputs: outputs and the launches each made."""
    rng = np.random.default_rng(3000 + data_rank)
    d, m = 8, 96
    X = rng.random((20_000, d), dtype=np.float32)
    y = np.sin(X.astype(np.float64).sum(1)) + 0.1 * rng.standard_normal(len(X))
    k, _ = ard_stats(d)
    out, launches = {}, {}

    def rec(key, fn, *args):
        before = e.launch_count()
        out[key] = fn(*args)
        launches[key] = e.launch_count() - before

    rec("kmeans", lambda: e.kmeans(X, 8, max_iter=5, seed=rank + 1)[:2])
    rec("greedy", e.greedy_active_set, k, X[:3000].astype(np.float64), y[:3000], 20, 3, 16)
    rec("kernel_eval", e.kernel_eval, k, X[:300], X[300:500].astype(np.float64), True)
    Z = X[:m].astype(np.float64)
    e.begin(k, Z)                          # a window opened and left open: no finish, no collective
    rec("cross_kernel", e.cross_kernel, X[500:900].astype(np.float64))
    rec("kmn_sweep", e.kmn_sweep, X[:5000])
    v = rng.standard_normal(m)
    A = rng.standard_normal((m, m))
    e.set_magic(v, -(A @ A.T) / m * 1e-3)
    rec("predict", e.predict, X[900:1400].astype(np.float64))
    return out, launches


def sc_local(w):
    out, launches = run_local_entries(w.eng, w.rank, w.data_rank)
    out_l, launches_l = run_local_entries(w.solo, w.rank, w.data_rank)
    return dict(out=out, launches=launches, out_l=out_l, launches_l=launches_l)


def _flat(x):
    if isinstance(x, (tuple, list)):
        return [y for v in x for y in _flat(v)]
    if x is None:
        return []
    return [np.ascontiguousarray(x)]


@pytest.mark.parametrize("world", [1, 2])
def test_rank_local_entries_ignore_the_communicator(pools, world):
    """sgp_kmeans, sgp_greedy_active_set, sgp_kernel_eval, sgp_cross_kernel, sgp_kmn_sweep and sgp_predict, with other
    inputs on every rank: the communicator context's outputs and launch counts equal the plain context's, bit for bit."""
    res = pools(world).run("sc_local")
    for rank, r in enumerate(res):
        assert r["launches"] == r["launches_l"], (rank, r["launches"], r["launches_l"])
        for key in r["out"]:
            got, want = _flat(r["out"][key]), _flat(r["out_l"][key])
            assert len(got) == len(want)
            for a, b in zip(got, want):
                assert a.dtype == b.dtype and a.shape == b.shape and a.tobytes() == b.tobytes(), (rank, key)


# ---------------- sgp_comm_init on one context ------------------------------------------------------------------------------
def small_window(eng):
    rng = np.random.default_rng(5)
    X = rng.random((4000, 4))
    k, _ = ard_stats(4)
    eng.set_precision(N.SGP_PREC_F64)
    eng.begin(k, X[:32])
    eng.accumulate(X, np.sin(X.sum(1)))
    return eng.finish()


def test_comm_init_refusals_leave_the_context_usable():
    """A null id, nranks < 1, rank < 0 and rank >= nranks: SGP_E_BADARG, no communicator, and the context still
    computes what a fresh one computes."""
    eng, ref = sg.ProjectedProcessEngine(0), sg.ProjectedProcessEngine(0)
    try:
        uid = sg.ProjectedProcessEngine.comm_unique_id()
        buf = N.ptr(np.frombuffer(uid, dtype=np.uint8).copy())
        for args in ((None, 0, 1), (buf, 0, 0), (buf, -1, 2), (buf, 2, 2), (buf, 1, 1)):
            assert eng._lib.sgp_comm_init(eng._h, *args) == N.SGP_E_BADARG, args
        G, b = small_window(eng)
        G0, b0 = small_window(ref)
        assert np.array_equal(bits(G), bits(G0)) and np.array_equal(bits(b), bits(b0))
    finally:
        eng.close()
        ref.close()


def test_second_comm_init_is_refused():
    """A context that has a communicator refuses a second one with SGP_E_STATE and keeps the first: the statistics of a
    communicator of one rank are still the plain context's bits, with the same launch count."""
    eng, ref = sg.ProjectedProcessEngine(0), sg.ProjectedProcessEngine(0)
    try:
        eng.comm_init(sg.ProjectedProcessEngine.comm_unique_id(), 0, 1)
        other = np.frombuffer(sg.ProjectedProcessEngine.comm_unique_id(), dtype=np.uint8).copy()
        assert eng._lib.sgp_comm_init(eng._h, N.ptr(other), 0, 1) == N.SGP_E_STATE
        assert "already has a communicator" in eng._lib.sgp_last_error(eng._h).decode()
        with pytest.raises(sg.TrainingVectorsNotInitializedException):
            eng.comm_init(bytes(other), 0, 1)
        before, before_ref = eng.launch_count(), ref.launch_count()
        G, b = small_window(eng)
        G0, b0 = small_window(ref)
        assert np.array_equal(bits(G), bits(G0)) and np.array_equal(bits(b), bits(b0))
        assert eng.launch_count() - before == ref.launch_count() - before_ref
    finally:
        eng.close()
        ref.close()
