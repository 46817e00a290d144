"""One-vs-rest over a process group on GPUs (`OneVsRest().setClassifier(GaussianProcessClassifier(process_group=g))`).

Each scenario runs in spawned workers, worker r on cuda:r, joined in one NCCL process group; the parent compares what
they send back, within a deadline, and joins (or kills) every worker before the next scenario.  At world 1:
  * the group fit equals the plain `OneVsRest.fit` bit for bit -- every class's theta, active set and magic pair,
    predictRaw, predict, predictAveragedProbability, last_latent and last_objective -- on the Iris fixture (n_e = 20,
    m = 30) with the random, explicit and GPU K-means providers, host and CUDA input, and on a 4-class shard with
    150-point experts, where the global-memory Laplace kernel runs;
  * the rank halves of 2-, 3- and 7-rank fits, on one GPU without a communicator: each rank's expert rows through the
    strided upload and one `laplace_nll_classes_any_size` over every class at fixed per-class thetas.  Each class's
    modes are the plain upload's at those rows bit for bit (every rank runs the plain upload's kernel family), and its
    objectives and statistics add up to the plain ones;
  * the greedy and scikit-learn providers and bad labels are refused with ValueError.
With two or more GPUs: every rank returns the same model bits, and at fixed thetas the modes, G, b and predictions
match the plain one-vs-rest on the concatenation, with uneven splits and an empty rank 0."""
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


def visible_gpus():
    import torch
    return torch.cuda.device_count() if torch.cuda.is_available() else 0


GPUS = visible_gpus()
MULTI = sorted({w for w in (2, min(GPUS, 8)) if w >= 2})
need_two = pytest.mark.skipif(GPUS < 2, reason="needs two or more GPUs; this machine has %d" % GPUS)


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
    """Runs scenario `name` on `world` ranks; returns their outputs by rank."""
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


def bits(a):
    return np.ascontiguousarray(np.asarray(a, dtype=np.float64)).view(np.int64)


def host(a):
    return a.cpu().numpy() if hasattr(a, "cpu") else np.asarray(a)


# ---------------- scenarios (run in the workers) -------------------------------------------------------------------------
def iris():
    c = np.load(os.path.join(GOLD, "iris_case.npz"))
    return c["X"][c["train_idx"]], c["y"][c["train_idx"]], c["X"][c["test_idx"]]


def class_shard(N, d=3, C=4, seed=12):
    """N rows of C Gaussian blobs, labelled by blob, and 64 test rows."""
    rng = np.random.default_rng(seed)
    centres = 1.5 * rng.standard_normal((C, d))
    lab = rng.integers(0, C, N + 64)
    X = centres[lab] + rng.standard_normal((N + 64, d))
    return X[:N], lab[:N].astype(np.float64), X[N:]


# data set -> (rows, labels, test rows, classifier settings)
DATA = {
    "iris": lambda: iris() + (dict(n_e=20, m=30, kernel=None, sigma2=None, max_iter=None),),
    # 150-point experts: above the on-chip Laplace kernel's 117 points
    "global": lambda: class_shard(1500) + (dict(n_e=150, m=40, kernel=2.0, sigma2=1.0, max_iter=3),),
}


def classifier(settings, kind, X, device, group=None):
    import spark_gp_b200 as sg
    from spark_gp_b200.regression import ExplicitActiveSetProvider
    gp = (sg.GaussianProcessClassifier(device=device, process_group=group)
          .setDatasetSizeForExpert(settings["n_e"]).setActiveSetSize(settings["m"]))
    if settings["kernel"] is not None:
        gp = gp.setKernel(lambda: sg.RBFKernel(settings["kernel"])).setSigma2(settings["sigma2"])
    if settings["max_iter"] is not None:
        gp = gp.setMaxIter(settings["max_iter"])
    provider = {"random": sg.RandomActiveSetProvider,
                "explicit": ExplicitActiveSetProvider(np.asarray(X[5:5 + settings["m"]], np.float64)),
                "kmeans": sg.KMeansActiveSetProvider(maxIter=10, on_gpu=True),
                "sklearn": sg.KMeansActiveSetProvider(), "greedy": sg.GreedilyOptimizingActiveSetProvider()}[kind]
    return gp.setActiveSetProvider(provider)


def shard(a, rank, world, sizes=None):
    cuts = [0] + [int(c) for c in np.cumsum(sizes)] if sizes else [r * len(a) // world for r in range(world + 1)]
    return a[cuts[rank]:cuts[rank + 1]]


def ovr_out(ovr, model, Xt):
    rps = [m.rawPredictor for m in model.models]
    return dict(theta=np.asarray(model.hyperparameters), Z=[np.asarray(rp.activeSet) for rp in rps],
                mv=[rp.magicVector for rp in rps], mm=[rp.magicMatrix for rp in rps],
                raw=host(model.predictRaw(Xt)), pred=host(model.predict(Xt)),
                prob=host(model.predictAveragedProbability(Xt)), latent=host(ovr.last_latent),
                objective=ovr.last_objective)


def fit_pair(rank, world, group, data, kind, on_cuda, sizes=None, fixed=False):
    """The group one-vs-rest fit of this rank's shard and, on every rank, the plain fit of the concatenation."""
    import torch
    import spark_gp_b200 as sg
    from spark_gp_b200 import distributed as D
    X, y, Xt, settings = DATA[data]()
    put = (lambda a: torch.as_tensor(a, device=torch.device("cuda", rank))) if on_cuda else (lambda a: a)
    C = int(y.max()) + 1
    thetas = np.linspace(1.0, 2.0, C)[:, None] if fixed else None
    ovr_d = sg.OneVsRest().setClassifier(classifier(settings, kind, X, rank, group))
    md = ovr_d.fit(put(shard(X, rank, world, sizes)), put(shard(y, rank, world, sizes)), thetas)
    path = next(iter(D._COMM_ENGINES.values())).last_laplace_path()
    ovr_p = sg.OneVsRest().setClassifier(classifier(settings, kind, X, rank))
    mp_ = ovr_p.fit(put(X), put(y), thetas)
    n = [len(shard(X, r, world, sizes)) for r in range(world)]
    rows = D.ShardPlan(n, rank, settings["n_e"]).expert_rows()
    latent = ovr_d.last_latent
    out = dict(dist=ovr_out(ovr_d, md, put(Xt)), plain=ovr_out(ovr_p, mp_, put(Xt)), rows=rows, path=path,
               latent_type=(str(latent.device) if torch.is_tensor(latent) else "host", str(latent.dtype)))
    if fixed:
        # every class's statistics through the group path the estimator takes, and the binary fit's on (y == c)
        slots, _ = D.group_fit(classifier(settings, kind, X, rank, group), put(shard(X, rank, world, sizes)),
                               put(shard(y, rank, world, sizes)), thetas, "classes")
        out["stats"] = [s[6] for s in slots]
        out["stats_plain"] = []
        for c in range(C):
            gp_c = classifier(settings, kind, X, rank)
            gp_c.fit(X, (y == c).astype(np.float64), thetas[c])
            out["stats_plain"].append(gp_c.last_stats)
    return out


WORLD_ONE = [("iris", "random", False), ("iris", "random", True), ("iris", "explicit", False),
             ("iris", "explicit", True), ("iris", "kmeans", False), ("iris", "kmeans", True),
             ("global", "random", False), ("global", "kmeans", True)]


def world_one_all(rank, world, group):
    return {case: fit_pair(rank, world, group, *case) for case in WORLD_ONE}


def virtual_ranks(rank, world, group, Rs, n_es):
    """The rank halves of R-rank one-vs-rest fits on one GPU, without a communicator: for each rank of an uneven split,
    its expert rows (`ShardPlan.expert_rows`, the rows the shuffle delivers) through the strided upload (E_r < E
    experts), one `laplace_nll_classes_any_size` over every class at fixed per-class thetas, each class's modes ungrouped
    into row order, and the statistics over its rows with each class's modes as labels.  The parent sums them and
    compares with the plain upload of all rows.  21 experts of exactly n_e points each: every rank's largest expert is
    the plain upload's, so every rank runs its kernel family."""
    import torch
    import spark_gp_b200 as sg
    from spark_gp_b200 import _native as N
    from spark_gp_b200.distributed import ShardPlan
    dev = torch.device("cuda", rank)
    C = 4
    kernels = [(sg.RBFKernel(2.0) + sg.const(1.0) * sg.EyeKernel()).setHyperparameters(np.array([1.5 + 0.25 * c]))
               for c in range(C)]

    def halves(eng, Xd, yd, upload):
        upload()
        v, g = eng.laplace_nll_classes_any_size(C, list(range(C)), kernels, 1e-6)
        path = eng.last_laplace_path()
        fs = [eng.experts_modes_rows(N.SGP_MODES_CLASS, c, len(Xd)) for c in range(C)]
        eng.set_precision(N.SGP_PREC_F64_STRICT)
        stats = [eng.statistics(kernels[c], Z, Xd, fs[c]) for c in range(C)]
        eng.set_precision(N.SGP_PREC_AUTO)
        return dict(v=v, g=g, path=path, f=[f.cpu().numpy() for f in fs], G=[s[0] for s in stats],
                    b=[s[1] for s in stats])

    out = {}
    eng = sg.ProjectedProcessEngine(rank)
    try:
        for n_e in n_es:
            X, y, _ = class_shard(21 * n_e, seed=n_e)
            Z = X[::37][:60]
            Xd, yd = torch.as_tensor(X, device=dev), torch.as_tensor(y, device=dev)
            plain = halves(eng, Xd, yd, lambda: eng.experts_upload_grouped(Xd, yd, n_e))
            for R in Rs:
                rng = np.random.default_rng(R)
                cuts = np.sort(rng.integers(0, len(X) + 1, size=R - 1))
                sizes = np.diff(np.concatenate([[0], cuts, [len(X)]]))
                parts = []
                for r in range(R):
                    plan = ShardPlan(sizes, r, n_e)
                    rows = plan.expert_rows()
                    Xr, yr = Xd[torch.as_tensor(rows, device=dev)], yd[torch.as_tensor(rows, device=dev)]
                    part = halves(eng, Xr, yr, lambda: eng.experts_upload_strided(Xr, yr, plan.local_experts))
                    parts.append(dict(part, rows=rows, E=plan.local_experts))
                out[n_e, R] = dict(plain=plain, parts=parts, E=ShardPlan(sizes, 0, n_e).E, N=len(X))
        return out
    finally:
        eng.close()


def refusals(rank, world, group):
    import spark_gp_b200 as sg
    X, y, _, settings = DATA["iris"]()
    out = {}
    cases = [("sklearn", y), ("greedy", y), ("negative", np.where(np.arange(len(y)) == 7, -1.0, y)),
             ("fraction", np.where(np.arange(len(y)) == 7, 0.5, y))]
    for name, labels in cases:
        kind = name if name in ("sklearn", "greedy") else "random"
        try:
            sg.OneVsRest().setClassifier(classifier(settings, kind, X, rank, group)).fit(shard(X, rank, world),
                                                                                       shard(labels, rank, world))
            out[name] = None
        except ValueError as e:
            out[name] = str(e)
    return out


# ---------------- cases ------------------------------------------------------------------------------------------------
def same_model(a, b, keys=("theta", "Z", "mv", "mm")):
    for k in keys:
        assert np.array_equal(bits(a[k]), bits(b[k])), k


@pytest.fixture(scope="module")
def world_one():
    return run("world_one_all")[0]


@pytest.mark.parametrize("case", WORLD_ONE, ids=["-".join(map(str, c)) for c in WORLD_ONE])
def test_world_one_equals_the_plain_one_vs_rest(world_one, case):
    o = world_one[case]
    same_model(o["dist"], o["plain"], ("theta", "Z", "mv", "mm", "raw", "pred", "prob", "latent"))
    assert o["dist"]["objective"] == o["plain"]["objective"]
    assert o["path"] == (1 if case[0] == "global" else 0)
    assert o["latent_type"] == (("cuda:0", "torch.float64") if case[2] else ("host", "float64"))
    assert np.array_equal(o["rows"], np.arange(len(o["rows"])))


@pytest.fixture(scope="module")
def rank_halves():
    return run("virtual_ranks", Rs=[2, 3, 7], n_es=[100, 150])[0]


@pytest.mark.parametrize("R", [2, 3, 7])
@pytest.mark.parametrize("n_e", [100, 150])
def test_rank_halves_of_every_class_sum_to_the_plain_upload(rank_halves, R, n_e):
    o = rank_halves[n_e, R]
    p, parts = o["plain"], o["parts"]
    assert sum(q["E"] for q in parts) == o["E"] == 21 and all(q["E"] < o["E"] for q in parts)
    # every rank runs the plain upload's kernel family: on chip up to 117 points, global memory above
    assert p["path"] == (0 if n_e <= 117 else 1) and all(q["path"] == p["path"] for q in parts)
    u = 2.0 ** -53
    for c in range(4):
        # every expert is the plain upload's: its modes are the plain modes at its rows, bit for bit
        F = np.full(o["N"], np.nan)
        for q in parts:
            F[q["rows"]] = q["f"][c]
        assert np.array_equal(bits(F), bits(p["f"][c])), c
        # every expert's -log Z is non-negative, so any order of the E terms, the ranks' and the plain one, is within
        # (E - 1) u of the sum of their magnitudes
        v = [q["v"][c] for q in parts]
        assert all(x > 0 for x in v)
        assert abs(sum(v) - p["v"][c]) <= 2 * (o["E"] - 1) * u * sum(abs(x) for x in v), c
        g = sum(q["g"][c] for q in parts)
        np.testing.assert_allclose(g, p["g"][c], rtol=1e-10, atol=1e-10 * np.abs(p["g"][c]).max())
        # G sums non-negative kernel products over the rows; b has terms of both signs
        G = [q["G"][c] for q in parts]
        assert np.all(np.abs(sum(G) - p["G"][c]) <= 2 * o["N"] * u * sum(np.abs(x) for x in G)), c
        b = sum(q["b"][c] for q in parts)
        assert np.abs(b - p["b"][c]).max() <= 1e-11 * np.abs(p["b"][c]).max(), c


def test_greedy_scikit_learn_and_bad_labels_are_refused():
    out = run("refusals")[0]
    assert "on_gpu=True" in out["sklearn"] and "GreedilyOptimizingActiveSetProvider" in out["greedy"]
    for name in ("negative", "fraction"):
        assert out[name] == "rank 0: OneVsRest: labels must be non-negative integers (class indices)"


@need_two
@pytest.mark.parametrize("world", MULTI)
@pytest.mark.parametrize("data,kind,on_cuda", [("iris", "random", False), ("iris", "kmeans", True),
                                               ("global", "explicit", True)])
def test_every_rank_returns_the_same_one_vs_rest_model(world, data, kind, on_cuda):
    got = run("fit_pair", world, data=data, kind=kind, on_cuda=on_cuda)
    for r in range(1, world):
        same_model(got[r]["dist"], got[0]["dist"])
        assert got[r]["dist"]["objective"] == got[0]["dist"]["objective"]


def uneven(N, world, empty_first):
    if empty_first:
        return [0] + [N // (world - 1)] * (world - 2) + [N - N // (world - 1) * (world - 2)]
    return [N // (2 * world)] * (world - 1) + [N - N // (2 * world) * (world - 1)]


@need_two
@pytest.mark.parametrize("world", MULTI)
@pytest.mark.parametrize("on_cuda", [False, True])
@pytest.mark.parametrize("empty_first", [False, True])
def test_multi_rank_fixed_thetas_match_the_plain_one_vs_rest(world, on_cuda, empty_first):
    got = run("fit_pair", world, data="global", kind="random", on_cuda=on_cuda, sizes=uneven(1500, world, empty_first),
              fixed=True)
    for r in range(world):
        o = got[r]
        d, p = o["dist"], o["plain"]
        # each class's modes are the plain fit's at the rows of the rank's experts
        np.testing.assert_allclose(d["latent"], p["latent"][:, o["rows"]], rtol=1e-12, atol=1e-13)
        for (G, b), (G0, b0) in zip(o["stats"], o["stats_plain"]):
            assert np.abs(G - G0).max() <= 1e-11 * np.abs(G0).max()
            assert np.abs(b - b0).max() <= 1e-11 * np.abs(b0).max()
        for k in ("raw", "prob"):
            assert np.abs(d[k] - p[k]).max() <= 1e-5 * max(1.0, np.abs(p[k]).max()), k
        same_model(d, got[0]["dist"])
