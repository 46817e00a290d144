"""The data-parallel fit on GPUs (`process_group=` of the estimators, `sgp_kmeans_sharded`).

Each case spawns `world` workers, worker r on cuda:r, joined in one NCCL process group; the case passes or fails on the
parent's comparison of what the workers send back, within a deadline, and every worker is joined (or killed) before the
next case.  At world 1:
  * the distributed fit equals the plain fit bit for bit -- theta, active set, magic pair, predictions -- for the
    regression with the random, explicit and GPU K-means providers, on host and CUDA inputs, and for the binary
    classifier on the mnist68 rows;
  * `sgp_kmeans_sharded` equals `sgp_kmeans` bit for bit;
  * the greedy and scikit-learn providers are refused.
With two or more GPUs: every rank returns the same model bits; at a fixed theta the model matches the plain fit on the
concatenation (G, b to 1e-11 relative, predictions to 1e-5); `sgp_kmeans_sharded` on integer blobs equals `sgp_kmeans`
on the concatenation bit for bit at every world size."""
import multiprocessing as mp
import os
import queue
import socket
import traceback

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

DEADLINE = 300.0
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
def regression_data(N=3001, d=4, f32=False):
    rng = np.random.default_rng(11)
    X = rng.standard_normal((N, d))
    y = np.sin(X.sum(1)) + 0.1 * rng.standard_normal(N)
    return (X.astype(np.float32) if f32 else X), y, rng.standard_normal((64, d))


def provider(kind, X):
    import spark_gp_b200 as sg
    from spark_gp_b200.regression import ExplicitActiveSetProvider
    return {"random": sg.RandomActiveSetProvider, "explicit": ExplicitActiveSetProvider(np.asarray(X[5:45], np.float64)),
            "kmeans": sg.KMeansActiveSetProvider(maxIter=10, on_gpu=True),
            "sklearn": sg.KMeansActiveSetProvider(), "greedy": sg.GreedilyOptimizingActiveSetProvider()}[kind]


def shard(a, rank, world, sizes=None):
    n = len(a)
    cuts = [0] + [int(c) for c in np.cumsum(sizes)] if sizes else [r * n // world for r in range(world + 1)]
    return a[cuts[rank]:cuts[rank + 1]]


def model_out(model, Xt, gp):
    mean, var = model.rawPredictor.predict(Xt)
    rp = model.rawPredictor
    return dict(theta=np.asarray(model.hyperparameters), Z=np.asarray(rp.activeSet), mv=rp.magicVector, mm=rp.magicMatrix,
                mean=host(mean), var=host(var), G=gp.last_stats[0], b=gp.last_stats[1])


def regression_gp(kind, X, group=None):
    import spark_gp_b200 as sg
    return (sg.GaussianProcessRegression(device=0 if group is None else __import__("torch").cuda.current_device(),
                                         process_group=group)
            .setDatasetSizeForExpert(100).setActiveSetSize(40).setMaxIter(5).setSeed(7)
            .setActiveSetProvider(provider(kind, X)))


def regression_world(rank, world, group, kind, on_cuda, f32=False, sizes=None, fixed=False):
    """The distributed fit of this rank's shard and, on every rank, the plain fit of the concatenation."""
    import torch
    X, y, Xt = regression_data(f32=f32)
    dev = torch.device("cuda", rank)
    put = (lambda a: torch.as_tensor(a, device=dev)) if on_cuda else (lambda a: a)
    theta = np.array([1.3]) if fixed else None
    gp_d = regression_gp(kind, X, group)
    md = gp_d.fit(put(shard(X, rank, world, sizes)), put(shard(y, rank, world, sizes)), theta)
    gp_p = regression_gp(kind, X)
    gp_p._device = rank
    mp_ = gp_p.fit(put(X), put(y), theta)
    return dict(dist=model_out(md, Xt, gp_d), plain=model_out(mp_, Xt, gp_p))


def mnist68():
    c = np.load(os.path.join(GOLD, "mnist68_case.npz"))
    n = int(c["n_rows"])
    X = (c["pixels"].astype(np.float64) - c["mean"]) / c["std"]
    return X[:n], c["y01"][:n], X[n:n + 100]


def classifier_world(rank, world, group, on_cuda, fixed=False):
    import torch
    import spark_gp_b200 as sg
    X, y, Xt = mnist68()
    dev = torch.device("cuda", rank)
    put = (lambda a: torch.as_tensor(a, device=dev)) if on_cuda else (lambda a: a)
    make = lambda g: (sg.GaussianProcessClassifier(device=rank, process_group=g).setDatasetSizeForExpert(100)
                      .setActiveSetSize(100).setKernel(lambda: sg.RBFKernel(10.0)).setTol(1e-3).setMaxIter(3))
    theta = np.array([9.0]) if fixed else None
    gp_d, gp_p = make(group), make(None)
    md = gp_d.fit(put(shard(X, rank, world)), put(shard(y, rank, world)), theta)
    mp_ = gp_p.fit(put(X), put(y), theta)
    from spark_gp_b200.distributed import ShardPlan
    sizes = [len(shard(X, r, world)) for r in range(world)]
    rows = ShardPlan(sizes, rank, 100).expert_rows()      # the global rows of this rank's experts
    return dict(dist=model_out(md, Xt, gp_d), plain=model_out(mp_, Xt, gp_p),
                latent=host(gp_d.last_latent), latent_plain=host(gp_p.last_latent)[rows])


def virtual_ranks(rank, world, group, R):
    """The per-rank halves of an R-rank classifier fit on one GPU, without a communicator: for each rank of an uneven
    split, its expert rows (`ShardPlan.expert_rows`, the rows the shuffle delivers) uploaded with the strided upload
    (E_r < E experts), the Laplace objective at a fixed theta, its modes ungrouped into row order, the statistics over
    its rows with the modes as labels, and the regression BCM objective of its experts.  The parent sums them and
    compares with the plain upload of all rows."""
    import torch
    import spark_gp_b200 as sg
    from spark_gp_b200 import _native as N
    from spark_gp_b200.distributed import ShardPlan
    X, y, _ = mnist68()
    dev = torch.device("cuda", rank)
    kernel = (sg.RBFKernel(10.0) + sg.const(1e-3) * sg.EyeKernel()).setHyperparameters(np.array([9.0]))
    Z = X[::37][:60]

    def halves(eng, Xd, yd, upload):
        upload()
        v, g = eng.laplace_nll_any_size(kernel, 1e-6)
        f = eng.experts_modes_rows(N.SGP_MODES_BINARY, 0, len(Xd))
        eng.set_precision(N.SGP_PREC_F64_STRICT)
        G, b = eng.statistics(kernel, Z, Xd, f)
        upload()
        vb, gb = eng.bcm_nll(kernel)
        return dict(v=v, g=g, f=f.cpu().numpy(), G=G, b=b, vb=vb, gb=gb)

    eng = sg.ProjectedProcessEngine(rank)
    try:
        Xd, yd = torch.as_tensor(X, device=dev), torch.as_tensor(y, device=dev)
        plain = halves(eng, Xd, yd, lambda: eng.experts_upload_grouped(Xd, yd, 100))
        rng = np.random.default_rng(R)
        cuts = np.sort(rng.integers(0, len(X) + 1, size=R - 1))
        sizes = np.diff(np.concatenate([[0], cuts, [len(X)]]))
        parts = []
        for r in range(R):
            plan = ShardPlan(sizes, r, 100)
            rows = plan.expert_rows()
            Xr, yr = Xd[torch.as_tensor(rows, device=dev)], yd[torch.as_tensor(rows, device=dev)]
            part = halves(eng, Xr, yr, lambda: eng.experts_upload_strided(Xr, yr, plan.local_experts))
            parts.append(dict(part, rows=rows, E=plan.local_experts))
        return dict(plain=plain, parts=parts, E=ShardPlan(sizes, 0, 100).E)
    finally:
        eng.close()


def refused_providers(rank, world, group):
    X, y, _ = regression_data()
    out = {}
    for kind in ("sklearn", "greedy"):
        try:
            regression_gp(kind, X, group).fit(shard(X, rank, world), shard(y, rank, world))
            out[kind] = None
        except ValueError as e:
            out[kind] = str(e)
    return out


def blobs(N=5000, d=5, seed=2):
    rng = np.random.default_rng(seed)
    centres = rng.integers(-50, 50, size=(12, d))
    return (centres[rng.integers(0, 12, size=N)] + rng.integers(-3, 4, size=(N, d))).astype(np.float64)


def kmeans_world(rank, world, group, integer, on_cuda, sizes=None, k=20):
    import torch
    import spark_gp_b200 as sg
    from spark_gp_b200.distributed import attach_communicator
    X = blobs() if integer else np.random.default_rng(4).standard_normal((5000, 5))
    eng = sg.ProjectedProcessEngine(rank)
    solo = sg.ProjectedProcessEngine(rank)
    try:
        attach_communicator(eng, group, torch.device("cuda", rank))
        cuts = [0] + [int(c) for c in np.cumsum(sizes)] if sizes else [r * len(X) // world for r in range(world + 1)]
        Xl = X[cuts[rank]:cuts[rank + 1]]
        Xl = torch.as_tensor(Xl, device="cuda:%d" % rank) if on_cuda else Xl
        c, lab, it, cost = eng.kmeans_sharded(Xl, cuts[rank], len(X), k, max_iter=20, seed=5, d=X.shape[1])
        c0, lab0, it0, cost0 = solo.kmeans(X, k, max_iter=20, seed=5)
        # sgp_kmeans on the communicator context still ignores the communicator
        c1, _, _, _ = eng.kmeans(X, k, max_iter=20, seed=5)
        return dict(c=c, lab=lab, it=it, cost=cost, c0=c0, lab0=lab0[cuts[rank]:cuts[rank + 1]], it0=it0, cost0=cost0,
                    c1=c1)
    finally:
        eng.close()
        solo.close()


def kmeans_model_world(rank, world, group, sizes):
    """sgp_kmeans_sharded on real-valued data, this rank's block of `sizes` rows (host fp64)."""
    import torch
    import spark_gp_b200 as sg
    from oracle import kmeans_cases as kc
    from spark_gp_b200.distributed import attach_communicator
    X = kc._lattice_mixture(5000, 5, 9)
    eng = sg.ProjectedProcessEngine(rank)
    try:
        attach_communicator(eng, group, torch.device("cuda", rank))
        cuts = [0] + [int(c) for c in np.cumsum(sizes)]
        c, lab, it, cost = eng.kmeans_sharded(X[cuts[rank]:cuts[rank + 1]], cuts[rank], len(X), 20, max_iter=20, seed=5,
                                              d=X.shape[1])
        return dict(c=c, lab=lab, it=it, cost=cost)
    finally:
        eng.close()


# ---------------- cases ------------------------------------------------------------------------------------------------
def same_model(a, b, keys=("theta", "Z", "mv", "mm", "mean", "var")):
    for k in keys:
        assert np.array_equal(bits(a[k]), bits(b[k])), k


@pytest.mark.parametrize("kind,on_cuda,f32", [("random", False, False), ("random", True, True),
                                              ("explicit", False, True), ("explicit", True, False),
                                              ("kmeans", False, False), ("kmeans", True, True)])
def test_world_one_regression_equals_the_plain_fit(kind, on_cuda, f32):
    out = run("regression_world", kind=kind, on_cuda=on_cuda, f32=f32)[0]
    same_model(out["dist"], out["plain"])
    assert np.array_equal(bits(out["dist"]["G"]), bits(out["plain"]["G"]))


@pytest.mark.parametrize("on_cuda", [False, True])
def test_world_one_classifier_equals_the_plain_fit(on_cuda):
    out = run("classifier_world", on_cuda=on_cuda)[0]
    same_model(out["dist"], out["plain"])
    assert np.array_equal(bits(out["latent"]), bits(out["latent_plain"]))


@pytest.mark.parametrize("integer,on_cuda", [(True, False), (False, False), (False, True)])
def test_world_one_sharded_kmeans_equals_kmeans(integer, on_cuda):
    o = run("kmeans_world", integer=integer, on_cuda=on_cuda)[0]
    assert np.array_equal(bits(o["c"]), bits(o["c0"])) and np.array_equal(bits(o["c1"]), bits(o["c0"]))
    assert np.array_equal(o["lab"], o["lab0"]) and o["it"] == o["it0"] and np.array_equal(bits(o["cost"]), bits(o["cost0"]))


def test_greedy_and_scikit_learn_providers_are_refused():
    out = run("refused_providers")[0]
    assert "on_gpu=True" in out["sklearn"] and "GreedilyOptimizingActiveSetProvider" in out["greedy"]


@pytest.mark.parametrize("R", [2, 3, 7])
def test_rank_halves_of_the_regrouped_experts_sum_to_the_plain_upload(R):
    o = run("virtual_ranks", R=R)[0]
    p, parts = o["plain"], o["parts"]
    assert sum(q["E"] for q in parts) == o["E"] and all(q["E"] < o["E"] for q in parts)
    # every expert is the plain upload's: its modes are the plain modes at its rows, and the objectives add up
    F = np.full(len(p["f"]), np.nan)
    for q in parts:
        F[q["rows"]] = q["f"]
    np.testing.assert_allclose(F, p["f"], rtol=1e-12, atol=1e-13)
    for v, g in (("v", "g"), ("vb", "gb")):
        assert abs(sum(q[v] for q in parts) - p[v]) <= 1e-12 * abs(p[v]), v
        np.testing.assert_allclose(sum(q[g] for q in parts), p[g], rtol=1e-10, atol=1e-10 * np.abs(p[g]).max())
    # the statistics over each rank's rows with its modes as labels add up to the plain statistics
    for k in ("G", "b"):
        assert np.abs(sum(q[k] for q in parts) - p[k]).max() <= 1e-11 * np.abs(p[k]).max(), k


@need_two
@pytest.mark.parametrize("world", MULTI)
@pytest.mark.parametrize("kind,on_cuda", [("random", False), ("kmeans", True), ("explicit", True)])
def test_every_rank_returns_the_same_regression_model(world, kind, on_cuda):
    got = run("regression_world", world, kind=kind, on_cuda=on_cuda)
    for r in range(world):
        same_model(got[r]["dist"], got[0]["dist"], ("theta", "Z", "mv", "mm"))
        # the optimisation ran on the regrouped experts: its theta is the plain fit's up to the objective's summation order
        np.testing.assert_allclose(got[r]["dist"]["theta"], got[r]["plain"]["theta"], rtol=1e-6)


@need_two
@pytest.mark.parametrize("world", MULTI)
def test_multi_rank_fixed_theta_matches_the_plain_fit(world):
    sizes = [0] + [3001 // (world - 1)] * (world - 2) + [3001 - 3001 // (world - 1) * (world - 2)]   # rank 0 empty
    got = run("regression_world", world, kind="random", on_cuda=False, sizes=sizes, fixed=True)
    for r in range(world):
        d, p = got[r]["dist"], got[r]["plain"]
        assert np.array_equal(bits(d["Z"]), bits(p["Z"]))
        for k in ("G", "b"):
            assert np.abs(d[k] - p[k]).max() <= 1e-11 * np.abs(p[k]).max(), k
        for k in ("mean", "var"):
            assert np.abs(d[k] - p[k]).max() <= 1e-5 * max(1.0, np.abs(p[k]).max()), k
        same_model(d, got[0]["dist"], ("theta", "Z", "mv", "mm"))


@need_two
@pytest.mark.parametrize("world", MULTI)
def test_multi_rank_classifier_every_rank_same_model(world):
    got = run("classifier_world", world, on_cuda=True)
    for r in range(1, world):
        same_model(got[r]["dist"], got[0]["dist"], ("theta", "Z", "mv", "mm"))


@need_two
@pytest.mark.parametrize("world", MULTI)
@pytest.mark.parametrize("on_cuda", [False, True])
def test_multi_rank_fixed_theta_classifier_matches_the_plain_fit(world, on_cuda):
    got = run("classifier_world", world, on_cuda=on_cuda, fixed=True)
    for r in range(world):
        d, p = got[r]["dist"], got[r]["plain"]
        # the rank's modes are the plain fit's modes at the rows of its experts
        np.testing.assert_allclose(got[r]["latent"], got[r]["latent_plain"], rtol=1e-12, atol=1e-13)
        for k in ("G", "b"):
            assert np.abs(d[k] - p[k]).max() <= 1e-11 * np.abs(p[k]).max(), k
        for k in ("mean", "var"):
            assert np.abs(d[k] - p[k]).max() <= 1e-5 * max(1.0, np.abs(p[k]).max()), k
        same_model(d, got[0]["dist"], ("theta", "Z", "mv", "mm"))


@need_two
@pytest.mark.parametrize("world", MULTI)
@pytest.mark.parametrize("uneven", [False, True])
def test_multi_rank_sharded_kmeans_on_integer_blobs_equals_kmeans(world, uneven):
    sizes = ([0] + [5000 // (world - 1)] * (world - 2) + [5000 - 5000 // (world - 1) * (world - 2)]) if uneven else None
    got = run("kmeans_world", world, integer=True, on_cuda=True, sizes=sizes)
    for r in range(world):
        o = got[r]
        assert np.array_equal(bits(o["c"]), bits(o["c0"])) and o["it"] == o["it0"] and np.array_equal(bits(o["cost"]), bits(o["cost0"]))
        assert np.array_equal(o["lab"], o["lab0"])


@need_two
@pytest.mark.parametrize("split", ["rank0_empty", "rank0_seven_rows", "even"])
def test_two_rank_sharded_kmeans_on_real_data_equals_the_two_rank_model(split):
    """Real-valued data at two ranks, where every all-reduced value is one addition: the outputs are the model's two-rank
    form bit for bit (each rank's fixed-order sums added), including a rank with no rows and one with fewer rows than
    candidates."""
    from oracle import kmeans_cases as kc
    from oracle import kmeans_model as km
    sizes = {"rank0_empty": [0, 5000], "rank0_seven_rows": [7, 4993], "even": [2500, 2500]}[split]
    X = kc._lattice_mixture(5000, 5, 9)
    (Cm, labm, itm, costm), info = km.run(X, 20, max_iter=20, seed=5, sizes=sizes)
    assert info["C"] > 20 and (split == "even" or info["C"] > sizes[0])
    got = run("kmeans_model_world", 2, sizes=sizes)
    cuts = [0] + [int(c) for c in np.cumsum(sizes)]
    for r in range(2):
        o = got[r]
        assert np.array_equal(bits(o["c"]), bits(Cm)) and o["it"] == itm and np.array_equal(bits(o["cost"]), bits(costm))
        assert np.array_equal(o["lab"], labm[cuts[r]:cuts[r + 1]])
