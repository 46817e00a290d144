"""Model selection over a process group on the GPU: `sgp_experts_upload_fold_sets_device`, and `CrossValidator` /
`TrainValidationSplit` over estimators with a `process_group`.

  * the entry against the fold upload: with blocks equal to the plain fold sets, `sgp_bcm_nll_folds` values and
    gradients and `sgp_laplace_nll_fold_slots_any_size` values, gradients and modes are the fold upload's bit for bit,
    on both Laplace kernel families;
  * virtual ranks: the rank halves of 2-, 3- and 7-rank selections on one GPU without a communicator, each rank's set
    blocks through the new entry: per-slot objectives add up to the plain ones within DESIGN.md section 5's bounds, and
    with equal-size experts (every rank on the plain kernel family) the modes are the plain modes at the rank's rows;
  * every refusal of the entry returns its code with no launch;
  * over a one-rank NCCL group every selector combination equals the plain selector bit for bit;
  * with two or more GPUs every rank returns the same bits, and the best map is the plain selector's on data whose maps
    are well separated (skipped below two GPUs)."""
import multiprocessing as mp
import os
import queue
import socket
import traceback

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

DEADLINE = 600.0
GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
U = 2.0 ** -53


def visible_gpus():
    import torch
    return torch.cuda.device_count() if torch.cuda.is_available() else 0


GPUS = visible_gpus()
MULTI = sorted({w for w in (2, min(GPUS, 8)) if w >= 2})
need_two = pytest.mark.skipif(GPUS < 2, reason="needs two or more GPUs; this machine has %d" % GPUS)


def bits(a):
    return np.ascontiguousarray(np.asarray(a, dtype=np.float64)).view(np.int64)


def host(a):
    return a.cpu().numpy() if hasattr(a, "cpu") else np.asarray(a)


# ---------------- the entry on one context --------------------------------------------------------------------------
def fold_data(F, K=3, d=4, seed=5):
    """K folds of F rows each in a seeded order, binary labels."""
    rng = np.random.default_rng(seed)
    X = rng.standard_normal((K * F, d))
    y = (X[:, 0] + 0.5 * rng.standard_normal(K * F) > 0).astype(np.float64)
    fold_of = rng.permutation(np.repeat(np.arange(K), F)).astype(np.int32)
    return X, y, fold_of


def kernel(theta):
    import spark_gp_b200 as sg
    return (sg.RBFKernel(1.0) + sg.const(1e-3) * sg.EyeKernel()).setHyperparameters(np.array([theta]))


def run_sets(eng, K, sets_of_slots):
    """The BCM and Laplace fold-slot objectives over K sets (two slots per set, classes 1 and 0), and every mode slot's
    modes per set in row order."""
    sets = [k for k in range(K) for _ in range(2)]
    kernels = [kernel(1.0 + 0.1 * i) for i in range(len(sets))]
    vb, gb = eng.bcm_nll_folds(sets, kernels)
    modes = list(range(len(sets)))
    classes = [1, 0] * K
    vl, gl = eng.laplace_nll_fold_slots_any_size(len(sets), modes, sets, classes, kernels, 1e-6)
    vl2, gl2 = eng.laplace_nll_fold_slots_any_size(len(sets), modes, sets, classes, kernels, 1e-6)   # warm start
    path = eng.last_laplace_path()
    f = [host(eng.experts_f_fold_slot_rows(s, m, sets_of_slots[s])) for m, s in zip(modes, sets)]
    return dict(vb=vb, gb=gb, vl=vl, gl=gl, vl2=vl2, gl2=gl2, f=f, path=path)


@pytest.mark.parametrize("n_e,f32", [(50, False), (50, True), (150, False)])
def test_fold_sets_upload_equals_the_fold_upload(n_e, f32):
    import torch
    import spark_gp_b200 as sg
    X, y, fold_of = fold_data(700 if n_e == 50 else 1500)
    K = 3
    if f32:
        X = X.astype(np.float32)
    Xd, yd = torch.as_tensor(X, device="cuda:0"), torch.as_tensor(y, device="cuda:0")
    plain, new = sg.ProjectedProcessEngine(0), sg.ProjectedProcessEngine(0)
    try:
        E = plain.experts_upload_folds(Xd, yd, fold_of, K, n_e)
        N_k = [int(np.count_nonzero(fold_of != k)) for k in range(K)]
        idx = torch.as_tensor(np.concatenate([np.flatnonzero(fold_of != k) for k in range(K)]), device="cuda:0")
        got = new.experts_upload_fold_sets(Xd[idx], yd[idx], N_k, E)
        assert list(got) == list(E)
        a, b = run_sets(plain, K, N_k), run_sets(new, K, N_k)
    finally:
        plain.close()
        new.close()
    assert a["path"] == b["path"] == (0 if n_e <= 117 else 1)
    for key in ("vb", "gb", "vl", "gl", "vl2", "gl2"):
        assert np.array_equal(bits(a[key]), bits(b[key])), key
    for fa, fb in zip(a["f"], b["f"]):
        assert np.array_equal(bits(fa), bits(fb))


def test_refusals_of_the_fold_sets_upload_launch_nothing():
    import torch
    import spark_gp_b200 as sg
    from spark_gp_b200 import _native as N
    X = torch.zeros((10, 3), dtype=torch.float64, device="cuda:0")
    y = torch.zeros(10, dtype=torch.float64, device="cuda:0")
    eng = sg.ProjectedProcessEngine(0)
    lib, h = eng._lib, eng._h
    px, py = X.data_ptr(), y.data_ptr()
    rows = lambda *v: np.array(v, dtype=np.int64)

    def call(px=px, py=py, r=rows(6, 4), e=rows(2, 1), n=2, d=3, null_rows=False):
        return lib.sgp_experts_upload_fold_sets_device(h, px, 0, py, None if null_rows else N.ptr(r), N.ptr(e), n, d)

    try:
        before = eng.launch_count()
        host_X = np.zeros((10, 3))
        cases = dict(null_X=call(px=None), null_y=call(py=None), null_rows=call(null_rows=True), no_set=call(n=0),
                     no_feature=call(d=0), empty_set=call(r=rows(0, 10)), no_expert=call(e=rows(0, 1)),
                     empty_expert=call(r=rows(6, 4), e=rows(2, 5)), host_memory=call(px=host_X.ctypes.data))
        assert all(rc == N.SGP_E_BADARG for rc in cases.values()), cases
        huge = rows(1 << 40, 4)                                       # the sets' rows would need 2^40 (d + 2) doubles
        assert call(r=huge) == N.SGP_E_NOMEM
        assert eng.launch_count() == before
        assert call() == N.SGP_OK and eng.launch_count() == before + 4
    finally:
        eng.close()


# ---------------- virtual ranks on one GPU ----------------------------------------------------------------------------
def rank_blocks(fold_of, K, sizes, n_e, r):
    """The global rows of rank r's block of every training set, in the order the shuffle delivers them, and its local
    experts per set."""
    from spark_gp_b200.distributed import ShardPlan
    R = len(sizes)
    off = np.concatenate([[0], np.cumsum(sizes)])
    out, experts = [], []
    for k in range(K):
        member = [np.arange(off[s], off[s + 1])[fold_of[off[s]:off[s + 1]] != k] for s in range(R)]
        plan_sizes = [len(m) for m in member]
        rows = [member[s][ShardPlan(plan_sizes, s, n_e).destinations() == r] for s in range(R)]
        out.append(np.concatenate(rows))
        experts.append(ShardPlan(plan_sizes, r, n_e).local_experts)
    return out, experts


@pytest.mark.parametrize("R", [2, 3, 7])
@pytest.mark.parametrize("n_e", [100, 150])
def test_rank_halves_of_every_set_sum_to_the_plain_fold_upload(R, n_e):
    import torch
    import spark_gp_b200 as sg
    F = 21 * n_e // 2                                     # every set: 2F rows in 21 experts of n_e rows
    X, y, fold_of = fold_data(F)
    K, N = 3, len(X)
    sizes = [N // R + (1 if r < N % R else 0) for r in range(R)]
    sizes[0], sizes[-1] = sizes[0] + sizes[-1] // 2, sizes[-1] - sizes[-1] // 2          # uneven
    Xd, yd = torch.as_tensor(X, device="cuda:0"), torch.as_tensor(y, device="cuda:0")
    eng = sg.ProjectedProcessEngine(0)
    try:
        E = eng.experts_upload_folds(Xd, yd, fold_of, K, n_e)
        assert list(E) == [21] * K
        N_k = [2 * F] * K
        plain = run_sets(eng, K, N_k)
        parts = []
        for r in range(R):
            blocks, experts = rank_blocks(fold_of, K, sizes, n_e, r)
            idx = torch.as_tensor(np.concatenate(blocks), device="cuda:0")
            eng.experts_upload_fold_sets(Xd[idx], yd[idx], [len(b) for b in blocks], experts)
            parts.append(dict(run_sets(eng, K, [len(b) for b in blocks]), blocks=blocks))
    finally:
        eng.close()
    # every rank runs the plain upload's kernel family: on chip up to 117 points, global memory above
    assert plain["path"] == (0 if n_e <= 117 else 1) and all(q["path"] == plain["path"] for q in parts)
    set_pos = [np.cumsum(fold_of != k) - 1 for k in range(K)]          # global row -> its position in set k
    for s, k in enumerate(k for k in range(K) for _ in range(2)):
        for key in ("vl", "vl2"):
            v = [q[key][s] for q in parts]
            assert all(x > 0 for x in v)
            assert abs(sum(v) - plain[key][s]) <= 2 * (21 - 1) * U * sum(abs(x) for x in v), (key, s)
        for key in ("vb", "gb", "gl", "gl2"):
            got = sum(q[key][s] for q in parts)
            np.testing.assert_allclose(got, plain[key][s], rtol=1e-10, atol=1e-10 * np.abs(plain[key][s]).max())
        # every expert is the plain upload's: its modes are the plain modes at its rows, bit for bit
        F_ = np.full(2 * F, np.nan)
        for q in parts:
            F_[set_pos[k][q["blocks"][k]]] = q["f"][s]
        assert np.array_equal(bits(F_), bits(plain["f"][s])), s


# ---------------- selectors over NCCL groups (spawned workers) --------------------------------------------------------
def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    p = s.getsockname()[1]
    s.close()
    return p


def _worker(rank, world, port, name, kw, outq):
    try:
        import torch
        import torch.distributed as dist
        torch.cuda.set_device(rank)
        dist.init_process_group("nccl", init_method="tcp://127.0.0.1:%d" % port, rank=rank, world_size=world,
                                device_id=torch.device("cuda", rank))
        try:
            out = globals()[name](rank, world, dist.group.WORLD, **kw)
        finally:
            dist.destroy_process_group()
        outq.put((rank, "ok", out))
    except BaseException:                                       # noqa: BLE001 -- reported to the parent
        outq.put((rank, "error", traceback.format_exc()))


def run(name, world=1, **kw):
    ctx = mp.get_context("spawn")
    outq = ctx.Queue()
    port = _free_port()
    procs = [ctx.Process(target=_worker, args=(r, world, port, name, kw, outq), daemon=True) for r in range(world)]
    for p in procs:
        p.start()
    got = {}
    try:
        for _ in range(world):
            rank, status, out = outq.get(timeout=DEADLINE)
            assert status == "ok", "rank %d:\n%s" % (rank, out)
            got[rank] = out
    except queue.Empty:
        pytest.fail("the workers passed their deadline of %.0f s" % DEADLINE)
    finally:
        for p in procs:
            p.join(timeout=60)
            if p.is_alive():
                p.kill()
                p.join()
    return got


def shard(a, rank, world, sizes=None):
    n = len(a)
    cuts = [0] + [int(c) for c in np.cumsum(sizes)] if sizes else [r * n // world for r in range(world + 1)]
    return a[cuts[rank]:cuts[rank + 1]]


def airfoil():
    z = np.load(os.path.join(GOLD, "airfoil_cv_case.npz"))
    return z["X"], z["y"], z["X"][:50]


def regression_shard(N=2400, d=4):
    rng = np.random.default_rng(11)
    X = rng.standard_normal((N, d))
    y = np.sin(X.sum(1)) + 0.1 * rng.standard_normal(N)
    return X, y, rng.standard_normal((50, d))


def iris():
    c = np.load(os.path.join(GOLD, "iris_case.npz"))
    return c["X"], c["y"], c["X"][c["test_idx"]]


def mnist68():
    c = np.load(os.path.join(GOLD, "mnist68_case.npz"))
    n = int(c["n_rows"])
    X = (c["pixels"].astype(np.float64) - c["mean"]) / c["std"]
    return X[:n], c["y01"][:n], X[n:n + 100]


def provider(kind, X):
    import spark_gp_b200 as sg
    from spark_gp_b200.regression import ExplicitActiveSetProvider
    return {"random": sg.RandomActiveSetProvider, "explicit": ExplicitActiveSetProvider(np.asarray(X[5:45], np.float64)),
            "kmeans": sg.KMeansActiveSetProvider(maxIter=10, on_gpu=True)}[kind]


def estimator(case, device, group):
    """(estimator, param maps, evaluator, data) of a case."""
    import spark_gp_b200 as sg
    data, kind = case.split("/")[:2]
    if data in ("airfoil", "shard"):
        X, y, Xt = airfoil() if data == "airfoil" else regression_shard()
        kernel = (lambda: 1 * sg.ARDRBFKernel(5)) if data == "airfoil" else (lambda: sg.RBFKernel(1.0))
        est = (sg.GaussianProcessRegression(device=device, process_group=group).setKernel(kernel)
               .setDatasetSizeForExpert(100).setActiveSetSize(40).setMaxIter(5).setSeed(7)
               .setActiveSetProvider(provider(kind, X)))
        maps = sg.ParamGridBuilder().addGrid("sigma2", [1e-3, 1e-1]).build()
        return est, maps, sg.RegressionEvaluator(), (X, y, Xt)
    gp = (sg.GaussianProcessClassifier(device=device, process_group=group).setActiveSetSize(30).setTol(1e-3)
          .setMaxIter(3).setSeed(7))
    if data == "iris":
        est = sg.OneVsRest().setClassifier(gp.setDatasetSizeForExpert(20).setKernel(lambda: sg.RBFKernel(1.0)))
        maps = sg.ParamGridBuilder().addGrid("sigma2", [1e-3, 1e-1]).build()
        return est, maps, sg.MulticlassClassificationEvaluator("accuracy"), iris()
    est = gp.setDatasetSizeForExpert(100).setActiveSetSize(100).setKernel(lambda: sg.RBFKernel(10.0))
    maps = sg.ParamGridBuilder().addGrid("sigma2", [1e-3, 1e-1]).build()
    ev = sg.BinaryClassificationEvaluator() if kind == "auc" else sg.MulticlassClassificationEvaluator("accuracy")
    return est, maps, ev, mnist68()


def model_bits(model, Xt, on_cuda):
    """The best model's theta, active sets, magic pairs and predictions."""
    import torch
    Xq = torch.as_tensor(Xt, device="cuda:%d" % torch.cuda.current_device()) if on_cuda else Xt
    models = getattr(model, "models", [model])
    out = dict(theta=np.asarray(model.hyperparameters), pred=host(model.predict(Xq)))
    for c, m in enumerate(models):
        rp = m.rawPredictor
        out["Z%d" % c], out["mv%d" % c], out["mm%d" % c] = np.asarray(rp.activeSet), rp.magicVector, rp.magicMatrix
    return out


def objective_bits(obj):
    """rounds and launches of every group of a selector's record, and its slots' values."""
    return [(g.get("rounds"), g.get("launches"), [s.get("value") for s in g.get("slots", [])]) for g in obj["groups"]]


def select(case, on_cuda, given, rank, world, group):
    """One selector (CV or TVS, from the case) over the group on this rank's shard, or plain when group is None."""
    import torch
    import spark_gp_b200 as sg
    selector = case.split("/")[2]
    est, maps, ev, (X, y, Xt) = estimator(case, rank, group)
    N = len(X)
    dev = torch.device("cuda", rank)
    if group is not None:
        X, y = shard(X, rank, world), shard(y, rank, world)
    off = 0 if group is None else rank * N // world
    put = (lambda a: torch.as_tensor(a, device=dev)) if on_cuda else (lambda a: a)
    if selector == "cv":
        sel = sg.CrossValidator().setEstimator(est).setEstimatorParamMaps(maps).setEvaluator(ev).setNumFolds(3).setSeed(4)
        split = None if not given else dict(folds=(np.arange(N) % 3)[off:off + len(X)])
        m = sel.fit(put(X), put(y), **(split or {}))
        metrics = m.avgMetrics
        records = {k: (v["theta"], v["magicVector"], v["prediction"]) for k, v in sel.last_folds.items()}
    else:
        sel = (sg.TrainValidationSplit().setEstimator(est).setEstimatorParamMaps(maps).setEvaluator(ev)
               .setTrainRatio(0.7).setSeed(4))
        split = None if not given else dict(train=(np.arange(N) % 4 != 0)[off:off + len(X)])
        m = sel.fit(put(X), put(y), **(split or {}))
        metrics = m.validationMetrics
        records = [host(p) for p in sel.last_predictions]
    return dict(metrics=metrics, best=m.bestIndex, records=records, objective=objective_bits(m.last_objective),
                model=model_bits(m.bestModel, Xt, on_cuda))


WORLD_ONE = [("airfoil/random/cv", False, False), ("shard/explicit/cv", True, True),
             ("shard/kmeans/cv", False, True), ("shard/kmeans/cv", True, False), ("iris/ovr/cv", False, False),
             ("iris/ovr/cv", True, True), ("mnist68/acc/tvs", False, False), ("mnist68/auc/tvs", True, True),
             ("shard/random/tvs", False, True), ("shard/kmeans/tvs", True, False), ("iris/ovr/tvs", True, False)]


def world_one_cases(rank, world, group):
    out = {}
    for case, on_cuda, given in WORLD_ONE:
        out[case, on_cuda, given] = (select(case, on_cuda, given, rank, world, group),
                                     select(case, on_cuda, given, rank, world, None))
    return out


@pytest.fixture(scope="module")
def world_one():
    return run("world_one_cases")[0]


def assert_same_bits(a, b, where=""):
    if isinstance(a, dict):
        assert sorted(a, key=str) == sorted(b, key=str), where
        for k in a:
            assert_same_bits(a[k], b[k], "%s/%s" % (where, k))
    elif isinstance(a, (list, tuple)) and not (len(a) and isinstance(a[0], (int, float, np.floating)) and
                                               not isinstance(a[0], bool)):
        assert len(a) == len(b), where
        for i, (x, y) in enumerate(zip(a, b)):
            assert_same_bits(x, y, "%s[%d]" % (where, i))
    elif a is None or isinstance(a, (int, str, bool)):
        assert a == b, where
    else:
        assert np.array_equal(bits(a), bits(b)), where


@pytest.mark.parametrize("case,on_cuda,given", WORLD_ONE)
def test_world_one_selection_equals_the_plain_selector(world_one, case, on_cuda, given):
    group, plain = world_one[case, on_cuda, given]
    # the entries all-reduce through the communicator: one more launch per objective call than on a plain context
    for (rg, lg, vg), (rp, lp, vp) in zip(group.pop("objective"), plain.pop("objective")):
        assert rg == rp and np.array_equal(bits(vg), bits(vp)) and lg >= lp, (rg, lg, rp, lp)
    assert_same_bits(group, plain, case)


def test_greedy_provider_in_a_param_map_is_refused_on_every_rank():
    out = run("refused_provider")[0]
    assert "GreedilyOptimizingActiveSetProvider" in out and out.startswith("rank 0: ")


def refused_provider(rank, world, group):
    import spark_gp_b200 as sg
    est, _, ev, (X, y, _) = estimator("shard/random/cv", rank, group)
    maps = [{}, {"activeSetProvider": sg.GreedilyOptimizingActiveSetProvider()}]
    try:
        sg.CrossValidator().setEstimator(est).setEstimatorParamMaps(maps).fit(X, y)
    except ValueError as e:
        return str(e)
    return "no refusal"


def multi_rank(rank, world, group, case):
    return select(case, False, False, rank, world, group), select(case, False, False, rank, world, None)


@need_two
@pytest.mark.parametrize("world", MULTI)
@pytest.mark.parametrize("case", ["shard/random/cv", "mnist68/acc/tvs"])
def test_every_rank_selects_the_same_bits(world, case):
    got = run("multi_rank", world, case=case)
    first = got[0][0]
    for r in range(1, world):
        assert_same_bits(got[r][0], first, "rank %d" % r)
    # the metrics of the maps are well separated here: the best map is the plain selector's
    assert first["best"] == got[0][1]["best"]
