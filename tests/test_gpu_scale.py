"""Feature scaling on the GPU (`sgp_column_sums_device`, `sgp_scale_apply_device`, `scale` of CUDA tensors and over a
process group).
  * The apply pass: for fp32 and fp64 CUDA X, n from 0 past several row blocks and d in {1, 5, 16, 32, 100}, the host
    formula (x - mean) / sd on the device's own mean and sd gives every output element bit for bit.
  * The sums: S and the centred squares Q are within the blocked-sum bound of oracle/scaling_model.py of the exact
    (math.fsum) sums, on columns with a 1e6 offset, a constant column and a column of zeros; those two get sd = 1.
  * The same bits from two calls, and from two contexts on concurrent threads.
  * Refusals before any launch: host memory as device memory, a bad dtype flag, n > 0 with a null X.
  * Spawned NCCL workers: at world 1 `scale(X, process_group=g)` equals the plain device `scale` bit for bit for host and
    CUDA shards, and scaling then a regression group fit equals the plain scale and fit bit for bit.  With two or more
    GPUs every rank applies the same mean and sd bits, within the bound of the oracle on the concatenation."""
import ctypes as C
import multiprocessing as mp
import queue
import socket
import threading
import traceback

import numpy as np
import pytest

from oracle import scaling_model as SM

pytestmark = pytest.mark.gpu

DEADLINE = 300.0
NS = [0, 1, 2, 2047, 2048, 2049, 5 * 2048 + 3]
DS = [1, 5, 16, 32, 100]


def visible_gpus():
    import torch
    return torch.cuda.device_count() if torch.cuda.is_available() else 0


GPUS = visible_gpus()
need_two = pytest.mark.skipif(GPUS < 2, reason="needs two or more GPUs; this machine has %d" % GPUS)


def data(n, d, seed=0, dtype=np.float64):
    """Mixed columns: standard normal, a 1e6 offset with small noise, a constant, zeros, a wide spread."""
    rng = np.random.default_rng(seed)
    X = rng.standard_normal((n, d))
    kinds = np.arange(d) % 5
    X[:, kinds == 1] = 1e6 + 0.25 * X[:, kinds == 1]
    X[:, kinds == 2] = 3.5
    X[:, kinds == 3] = 0.0
    X[:, kinds == 4] *= 1e3
    return X.astype(dtype)


def cuda(X):
    import torch
    return torch.as_tensor(X, device="cuda:0")


def bits(a):
    return np.ascontiguousarray(np.asarray(a, dtype=np.float64)).tobytes()


@pytest.fixture(scope="module")
def eng():
    import spark_gp_b200 as sg
    e = sg.ProjectedProcessEngine(0)
    yield e
    e.close()


@pytest.mark.parametrize("dtype", [np.float32, np.float64])
@pytest.mark.parametrize("d", DS)
def test_apply_gives_the_host_formula_bit_for_bit(eng, dtype, d):
    from spark_gp_b200.utils import moments, scale
    for n in NS:
        X = data(n, d, seed=n + d, dtype=dtype)
        Y = scale(cuda(X))
        assert str(Y.dtype) == "torch.float64" and tuple(Y.shape) == (n, d) and Y.is_cuda
        if n == 0:
            continue
        mean, sd = moments(eng, cuda(X))
        ref = (X.astype(np.float64) - mean) / sd
        assert Y.cpu().numpy().tobytes() == ref.tobytes(), (n, d)


def test_empty_rows_launch_nothing(eng):
    import torch
    before = eng.launch_count()
    assert eng.column_sums(torch.empty((0, 7), device="cuda:0")).tobytes() == np.zeros(7).tobytes()
    assert tuple(eng.scale_apply(torch.empty((0, 7), device="cuda:0"), np.zeros(7), np.ones(7)).shape) == (0, 7)
    assert eng.launch_count() == before


@pytest.mark.parametrize("dtype", [np.float32, np.float64])
@pytest.mark.parametrize("n", [1, 2049, 3 * 2048 + 77, 300_000])
def test_mean_and_variance_are_within_the_blocked_sum_bound(eng, dtype, n):
    d = 10
    X = data(n, d, seed=7, dtype=dtype)
    X64 = X.astype(np.float64)
    Xt = cuda(X)
    S = eng.column_sums(Xt)
    S0 = SM.exact_sums(X64)
    A = np.abs(X64).sum(0)
    assert (np.abs(S - S0) <= SM.sum_bound(n, A) + SM.U * np.abs(S0)).all()
    mean = S / n
    Q = eng.column_sums(Xt, mean)
    T = SM.centred_squares(X64, mean)
    Q0 = SM.exact_sums(T)
    assert (np.abs(Q - Q0) <= SM.sum_bound(n, T.sum(0)) + SM.U * Q0).all()
    # against the rule's own mean: S / n rounds once more
    mean0, sd0 = SM.moments(X64)
    assert (np.abs(mean - mean0) <= (SM.sum_bound(n, A) + 2 * SM.U * A) / n + 2 * SM.U * np.abs(mean0)).all()
    from spark_gp_b200.utils import moments
    m, sd = moments(eng, Xt)
    assert m.tobytes() == mean.tobytes()
    kinds = np.arange(d) % 5
    assert (sd[(kinds == 2) | (kinds == 3)] == 1.0).all() and (Q[(kinds == 2) | (kinds == 3)] == 0.0).all()


def test_two_calls_and_two_concurrent_contexts_give_the_same_bits():
    import torch
    import spark_gp_b200 as sg
    X = cuda(data(200_003, 16, seed=3, dtype=np.float32))
    mean = np.linspace(-1, 1, 16)
    ref = {}

    def run(key):
        e = sg.ProjectedProcessEngine(0)
        try:
            out = []
            for _ in range(4):
                out.append((bits(e.column_sums(X)), bits(e.column_sums(X, mean)),
                            e.scale_apply(X, mean, np.full(16, 3.0)).cpu().numpy().tobytes()))
            ref[key] = out
        except BaseException:                                   # noqa: BLE001 -- reported below
            ref[key] = traceback.format_exc()
        finally:
            e.close()

    threads = [threading.Thread(target=run, args=(k,)) for k in range(2)]
    for t in threads:
        t.start()
    for t in threads:
        t.join()
    torch.cuda.synchronize()
    assert all(isinstance(v, list) for v in ref.values()), ref
    first = ref[0][0]
    for k in range(2):
        for out in ref[k]:
            assert out == first


def test_refusals_come_before_any_launch(eng):
    from spark_gp_b200 import _native as N
    lib = N.load()
    X = data(100, 4)
    dX = cuda(X)
    out = np.empty(4)
    mean, sd = np.zeros(4), np.ones(4)
    Y = cuda(np.empty((100, 4)))
    before = eng.launch_count()
    p = lambda t: C.c_void_p(t.data_ptr())
    cases = [lib.sgp_column_sums_device(eng._h, N.ptr(X), 0, 100, 4, None, N.ptr(out)),            # host as device
             lib.sgp_scale_apply_device(eng._h, N.ptr(X), 0, 100, 4, N.ptr(mean), N.ptr(sd), p(Y)),
             lib.sgp_scale_apply_device(eng._h, p(dX), 0, 100, 4, N.ptr(mean), N.ptr(sd), N.ptr(out)),  # host Y
             lib.sgp_column_sums_device(eng._h, p(dX), 2, 100, 4, None, N.ptr(out)),                # bad dtype
             lib.sgp_scale_apply_device(eng._h, p(dX), -1, 100, 4, N.ptr(mean), N.ptr(sd), p(Y)),
             lib.sgp_column_sums_device(eng._h, None, 0, 100, 4, None, N.ptr(out)),                 # null X
             lib.sgp_scale_apply_device(eng._h, None, 1, 100, 4, N.ptr(mean), N.ptr(sd), p(Y)),
             lib.sgp_column_sums_device(eng._h, p(dX), 0, 100, 0, None, N.ptr(out)),                # no features
             lib.sgp_column_sums_device(eng._h, p(dX), 0, 100, 4, None, None)]                      # null out
    assert cases == [N.SGP_E_BADARG] * len(cases)
    assert eng.launch_count() == before
    # the context stays usable
    assert eng.column_sums(dX).tobytes() == eng.column_sums(dX).tobytes()


# ---------------- spawned NCCL workers ----------------------------------------------------------------------------------
def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    port = s.getsockname()[1]
    s.close()
    return port


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


def _recording_engine():
    import spark_gp_b200 as sg

    class Recording(sg.ProjectedProcessEngine):
        applied = None

        def scale_apply(self, X, mean, sd):
            Recording.applied = (mean.copy(), sd.copy())
            return super().scale_apply(X, mean, sd)

    return Recording


def shard(a, rank, world):
    cuts = [r * len(a) // world for r in range(world + 1)]
    return a[cuts[rank]:cuts[rank + 1]]


def scale_world(rank, world, group, N=30_001, d=16):
    """Every kind of shard scaled over the group, the applied mean and sd, and (world 1) the plain device scale."""
    import torch
    from spark_gp_b200 import distributed as D
    from spark_gp_b200.utils import scale
    Rec = _recording_engine()
    X = data(N, d, seed=11)
    Xs = shard(X, rank, world)
    dev = torch.device("cuda", rank)
    out = {}
    for kind, Xl in (("host", Xs), ("cuda64", torch.as_tensor(Xs, device=dev)),
                     ("cuda32", torch.as_tensor(Xs.astype(np.float32), device=dev))):
        Y = D.scale(Xl, group, engine_factory=Rec)
        out[kind] = dict(Y=Y if isinstance(Y, np.ndarray) else Y.cpu().numpy(), is_host=isinstance(Y, np.ndarray),
                         applied=Rec.applied, public=scale(Xl, process_group=group))
        out[kind]["public"] = np.asarray(out[kind]["public"] if isinstance(out[kind]["public"], np.ndarray)
                                         else out[kind]["public"].cpu().numpy())
        plain = torch.as_tensor(Xl, device=dev) if isinstance(Xl, np.ndarray) else Xl
        out[kind]["plain"] = scale(plain).cpu().numpy()
    return out


def scale_fit_world(rank, world, group):
    """Scaling then a regression fit over the group against the plain device scale and plain fit (world 1)."""
    import torch
    import spark_gp_b200 as sg
    rng = np.random.default_rng(5)
    X = data(4001, 4, seed=5) + rng.standard_normal((4001, 4))
    y = np.sin(X[:, 0]) + 0.1 * rng.standard_normal(4001)
    dev = torch.device("cuda", rank)
    Xt, yt = torch.as_tensor(X, device=dev), torch.as_tensor(y, device=dev)
    Xtest = torch.as_tensor(rng.standard_normal((64, 4)), device=dev)

    def gp(g):
        return (sg.GaussianProcessRegression(device=rank, process_group=g).setDatasetSizeForExpert(100)
                .setActiveSetSize(40).setMaxIter(5).setSeed(7))

    def out(model, Ys):
        mean, var = model.rawPredictor.predict(Xtest)
        rp = model.rawPredictor
        return dict(Y=Ys.cpu().numpy(), theta=np.asarray(model.hyperparameters), Z=np.asarray(rp.activeSet),
                    mv=np.asarray(rp.magicVector), mm=np.asarray(rp.magicMatrix), mean=mean.cpu().numpy(),
                    var=var.cpu().numpy())

    Yg = sg.scale(Xt, process_group=group)
    Yp = sg.scale(Xt)
    return dict(group=out(gp(group).fit(Yg, yt), Yg), plain=out(gp(None).fit(Yp, yt), Yp))


def test_world_one_group_scale_equals_the_plain_device_scale():
    o = run("scale_world")[0]
    for kind in ("host", "cuda64", "cuda32"):
        assert o[kind]["is_host"] == (kind == "host")
        assert o[kind]["Y"].tobytes() == o[kind]["plain"].tobytes() == o[kind]["public"].tobytes(), kind
    assert bits(o["host"]["applied"][0]) == bits(o["cuda64"]["applied"][0])


def test_world_one_scale_then_group_fit_equals_the_plain_scale_and_fit():
    o = run("scale_fit_world")[0]
    for key in ("Y", "theta", "Z", "mv", "mm", "mean", "var"):
        assert bits(o["group"][key]) == bits(o["plain"][key]), key


@need_two
@pytest.mark.parametrize("world", sorted({2, min(GPUS, 8)}))
def test_every_rank_applies_the_same_mean_and_sd_within_the_oracle_bound(world):
    got = run("scale_world", world)
    N, d = 30_001, 16
    for kind in ("host", "cuda64", "cuda32"):
        X = data(N, d, seed=11)
        X = X.astype(np.float32).astype(np.float64) if kind == "cuda32" else X
        A = np.abs(X).sum(0)
        mean0, _ = SM.moments(X)
        mean, sd = got[0][kind]["applied"]
        for r in range(world):
            m_r, s_r = got[r][kind]["applied"]
            assert bits(m_r) == bits(mean) and bits(s_r) == bits(sd)
            Xs = shard(X, r, world)
            assert got[r][kind]["Y"].tobytes() == ((Xs - mean) / sd).tobytes()
        assert (np.abs(mean - mean0) <= (SM.sum_bound(N, A) + (world + 2) * SM.U * A) / N
                + 2 * SM.U * np.abs(mean0)).all()
        T = SM.centred_squares(X, mean)
        Q0 = SM.exact_sums(T)
        var = sd * sd
        live = Q0 > 0
        assert (np.abs(var[live] * N - Q0[live]) <= SM.sum_bound(N, T.sum(0))[live] + (world + 8) * SM.U * Q0[live]).all()
