"""Several contexts side by side on one GPU, each driven from its own thread (run on an H100: `pytest -m gpu`).

This is the deployment INTEGRATION.md ("Threading") describes: every Spark task creates its own context on device
partitionId % nGPUs, so with more task slots than GPUs several contexts run on one device at once.  sgp.h promises that
contexts are independent.  Here each of four contexts runs one scripted call sequence of every entry-point family on its
own seeded data, at deliberately different shapes, so that their launch plans (dynamic shared memory, grids, paths)
differ.  The scripts run once sequentially on one thread, then all at once, one thread per context (ctypes releases the
GIL for the length of each library call, so the threads really overlap inside the library).  Every output, every path
and every error text of the concurrent run must equal the sequential run's bit for bit; the single-thread results are
pinned on the oracle by the other GPU tests, and one output per family is also checked against the oracle here.

While the four run, a fifth context makes calls the library refuses (its errors must stay its own), and a sixth thread
creates a context, evaluates one objective and destroys it (sgp_ctx_destroy synchronises the device: that may delay the
others, not change them).  The last test fits three estimators from three threads, the Spark task pattern at the Python
level.  Nothing here repeats a call to provoke a race: each script is one normal call sequence."""
import os
import struct
import threading

import numpy as np
import pytest

import oracle
import oracle.regression
import spark_gp_b200 as sg
from oracle import kmeans as okm
from oracle.classification import classification_likelihood_and_gradient
from spark_gp_b200 import _native as N
from spark_gp_b200.hyperopt import group_for_experts
from spark_gp_b200.regression import ExplicitActiveSetProvider
from test_gpu_parity import _oracle_stats_chunked, rel

pytestmark = pytest.mark.gpu

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
TOL_STATS, TOL_PRED, TOL_NLL = 1e-6, 1e-5, 1e-9

# One workload per context.  Shapes differ between contexts so that their plans differ: d 16 / 33 sends the int8 Gram
# to the tensor-core and the direct-distance producer; BCM experts of 64 / 150 / 169 / 400 points run the register,
# shared-memory and LU variants; Laplace experts of 30 .. 117 points share the on-chip kernel at four shared-memory
# plans, and 130 .. 240 points the global-memory kernel.
SPECS = [
    dict(seed=101, d=16, m=256, bcm_n=64, bcm_d=16, bcm_path=0, lap_n=30, lap_glob=200, lap_d=3, prov_d=16, sweep_d=16),
    dict(seed=202, d=33, m=200, bcm_n=150, bcm_d=33, bcm_path=0, lap_n=64, lap_glob=130, lap_d=5, prov_d=33, sweep_d=32),
    dict(seed=303, d=16, m=384, bcm_n=169, bcm_d=8, bcm_path=1, lap_n=100, lap_glob=160, lap_d=4, prov_d=64, sweep_d=8),
    dict(seed=404, d=33, m=128, bcm_n=400, bcm_d=5, bcm_path=1, lap_n=117, lap_glob=240, lap_d=6, prov_d=33, sweep_d=24),
]
STATS_N, STATS_CALLS = 150_000, 3          # three accumulate calls of 50k points: AUTO picks int8 on each (>= 32768)
EXPERTS, TOL_LAP = 4, 1e-6


def canon(x):
    """A value as comparable bits: arrays by dtype, shape and bytes, floats by their IEEE pattern (NaN == NaN)."""
    if hasattr(x, "detach"):
        x = x.detach().cpu().numpy()
    if isinstance(x, np.ndarray):
        return ("nd", x.dtype.str, x.shape, np.ascontiguousarray(x).tobytes())
    if isinstance(x, (float, np.floating)):
        return ("f", struct.pack("<d", float(x)))
    if isinstance(x, dict):
        return ("d", tuple((k, canon(v)) for k, v in sorted(x.items(), key=lambda kv: str(kv[0]))))
    if isinstance(x, (list, tuple)):
        return ("l", tuple(canon(v) for v in x))
    if isinstance(x, np.integer):
        return int(x)
    return x


def assert_same(got, want, what):
    assert got.keys() == want.keys(), what
    diff = [k for k in want if canon(got[k]) != canon(want[k])]
    assert not diff, "%s: not bit-identical to the sequential run: %s" % (what, ", ".join(map(str, diff)))


def last_error(eng):
    return eng._lib.sgp_last_error(eng._h).decode()


def ard(d, beta, noise=1e-2, scale=1.0):
    return (scale * sg.ARDRBFKernel(beta) + sg.const(noise) * sg.EyeKernel(),
            lambda: scale * oracle.ARDRBFKernel(beta) + oracle.const(noise) * oracle.EyeKernel())


def labels01(X, rng):
    d = X.shape[1]
    return (np.sin(2 * X[:, 0]) + 0.5 * X.sum(1) / np.sqrt(d) + 0.3 * rng.standard_normal(len(X)) > 0).astype(np.float64)


# ---------------- the scripts ------------------------------------------------------------------------------------------
def stats_inputs(spec):
    rng = np.random.default_rng(spec["seed"])
    d, m = spec["d"], spec["m"]
    X = rng.random((STATS_N, d), dtype=np.float32)
    y = np.sin(X.astype(np.float64).sum(1)) + 0.1 * rng.standard_normal(STATS_N)
    Z = X[rng.permutation(STATS_N)[:m]].astype(np.float64)
    k, ok = ard(d, np.full(d, np.sqrt(18.0 / d)), noise=1e-2)
    Xt = rng.random((3000, d))
    return X, y, Z, k, ok, Xt


def run_stats_and_tail(eng, spec, dev, out):
    import torch
    X, y, Z, k, _, Xt = stats_inputs(spec)
    cuda = torch.device("cuda", dev)
    Xd, yd = torch.from_numpy(X).to(cuda), torch.from_numpy(y).to(cuda)
    torch.cuda.current_stream(cuda).synchronize()
    step = STATS_N // STATS_CALLS
    for name, prec in (("i8", N.SGP_PREC_I8), ("auto", N.SGP_PREC_AUTO), ("f64", N.SGP_PREC_F64)):
        for entry in ("host", "device"):
            eng.set_precision(prec)
            eng.begin(k, Z)
            for s in range(0, STATS_N, step):
                if entry == "host":
                    eng.accumulate(X[s:s + step], y[s:s + step])
                else:
                    eng.accumulate_ptr(Xd[s:s + step].data_ptr(), True, yd[s:s + step].data_ptr(), step, device=True)
            out["stats_%s_%s" % (name, entry)] = eng.finish()
            out["stats_%s_%s_path" % (name, entry)] = eng.last_path()
    # the tail on the last window (fp64, device entry), then every prediction entry
    out["magic"] = eng.magic()
    out["tail_path"] = eng.last_tail_path()
    out["predict_host"] = eng.predict(Xt)
    out["predict_device"] = eng.predict_tensor(torch.from_numpy(Xt).to(cuda))
    out["probability_host"] = eng.predict_probability(Xt, nodes=32, with_mean_var=True)
    out["probability_device"] = eng.predict_probability_tensor(torch.from_numpy(Xt).to(cuda), nodes=32,
                                                               with_mean_var=True)


def run_sweep(eng, spec, dev, out):
    import torch
    rng = np.random.default_rng(spec["seed"] + 1)
    d = spec["sweep_d"]
    X = rng.random((20_000, d), dtype=np.float32)
    k, _ = ard(d, np.full(d, np.sqrt(4.0 / d)))
    eng.begin(k, X[:spec["m"]].astype(np.float64))
    out["sweep_host"] = eng.kmn_sweep(X)
    cuda = torch.device("cuda", dev)
    Xd = torch.from_numpy(X).to(cuda)
    K = torch.empty((len(X), spec["m"]), dtype=torch.float32, device=cuda)
    torch.cuda.current_stream(cuda).synchronize()
    eng.kmn_sweep_device(Xd.data_ptr(), True, len(X), K.data_ptr())
    eng.sync()
    out["sweep_device"] = K


def bcm_inputs(spec):
    rng = np.random.default_rng(spec["seed"] + 2)
    n_e, d = spec["bcm_n"], spec["bcm_d"]
    X = rng.standard_normal((EXPERTS * n_e, d))
    y = np.sin(X.sum(1)) + 0.3 * rng.standard_normal(len(X))
    k, ok = ard(d, rng.uniform(0.3, 3.0, d) / np.sqrt(d), scale=1.3)
    return X, y, k, ok


def run_bcm(eng, spec, out):
    X, y, k, _ = bcm_inputs(spec)
    theta = k.getHyperparameters()
    k2 = ard(spec["bcm_d"], np.ones(spec["bcm_d"]), scale=1.3)[0].setHyperparameters(theta * 1.1)
    assert eng.experts_upload_grouped(X, y, spec["bcm_n"]) == EXPERTS
    out["bcm"] = eng.bcm_nll(k)
    out["bcm_path"] = eng.last_bcm_path()
    out["bcm_slots"] = eng.bcm_nll_slots([k, k2])
    eng.experts_upload_folds(X, y, np.arange(len(X)) % 3, 3, spec["bcm_n"])
    out["bcm_folds"] = eng.bcm_nll_folds([0, 1, 2], [k, k2, k])
    out["bcm_folds_path"] = eng.last_bcm_path()


def laplace_inputs(spec, n_e):
    rng = np.random.default_rng(spec["seed"] + n_e)
    d = spec["lap_d"]
    X = rng.standard_normal((EXPERTS * n_e, d))
    k, ok = ard(d, rng.uniform(0.5, 1.5, d), scale=1.2)
    return X, labels01(X, rng), k, ok


def run_laplace(eng, spec, out):
    for tag, n_e in (("chip", spec["lap_n"]), ("global", spec["lap_glob"])):
        X, y, k, _ = laplace_inputs(spec, n_e)
        eng.experts_upload_grouped(X, y, n_e)
        out["laplace_%s" % tag] = eng.laplace_nll_any_size(k, TOL_LAP)
        out["laplace_%s_path" % tag] = eng.last_laplace_path()
        out["laplace_%s_f" % tag] = eng.experts_f(len(X))
    # one-vs-rest classes and fold slots, on chip
    X, y, k, _ = laplace_inputs(spec, spec["lap_n"])
    y3 = np.digitize(X[:, 0], [-0.4, 0.4]).astype(np.float64)
    eng.experts_upload_grouped(X, y3, spec["lap_n"])
    out["laplace_classes"] = eng.laplace_nll_classes_any_size(3, [0, 1, 2], [k, k, k], TOL_LAP)
    out["laplace_classes_f"] = [eng.experts_f_class(c, len(X)) for c in range(3)]
    fold_of = np.arange(len(X)) % 3
    eng.experts_upload_folds(X, y, fold_of, 3, spec["lap_n"])
    out["laplace_fold_slots"] = eng.laplace_nll_fold_slots_any_size(3, [0, 1, 2], [0, 1, 2], [1, 1, 1], [k, k, k],
                                                                     TOL_LAP)
    out["laplace_fold_slots_f"] = [eng.experts_f_fold_slot(s, s, int(np.sum(fold_of != s))) for s in range(3)]


def provider_inputs(spec):
    rng = np.random.default_rng(spec["seed"] + 3)
    d = spec["prov_d"]
    centres = 10.0 * rng.standard_normal((8, d))
    blob = rng.integers(0, 8, 20_000)
    X = centres[blob] + 0.3 * rng.standard_normal((20_000, d))
    init = X[[int(np.argmax(blob == j)) for j in range(8)]]           # one point of each blob: wide assignment margins
    return X, init


def run_providers(eng, spec, out):
    X, init = provider_inputs(spec)
    out["kmeans"] = eng.kmeans(X, 8, max_iter=10, seed=spec["seed"])
    out["kmeans_init"] = eng.kmeans(X, 8, max_iter=10, init_centers=init)
    rng = np.random.default_rng(spec["seed"] + 4)
    d = spec["prov_d"]
    Xg = rng.random((3000, d))
    yg = np.sin(3 * Xg.sum(1) / np.sqrt(d)) + 0.1 * rng.standard_normal(3000)
    k, _ = ard(d, np.full(d, 2.0 / np.sqrt(d)))
    out["greedy"] = eng.greedy_active_set(k, Xg, yg, 30, 7, 24)


def workload(spec, dev=0):
    """One context's script: (outputs, the context's last error text)."""
    out = {}
    eng = sg.ProjectedProcessEngine(dev)
    try:
        run_stats_and_tail(eng, spec, dev, out)
        run_sweep(eng, spec, dev, out)
        run_bcm(eng, spec, out)
        run_laplace(eng, spec, out)
        run_providers(eng, spec, out)
        out["last_error"] = last_error(eng)
    finally:
        eng.close()
    return out


def refusals(dev=0):
    """A context whose calls the library refuses on the host or reports as a status: a bad argument, a predict with no
    magic pair (SGP_E_STATE), and an AUTO window whose first chunk is benign and whose later chunks exceed the int8
    magnitude budget (SGP_E_RANGE at finish, as test_auto_budget_checked_over_whole_window)."""
    out = {}
    eng = sg.ProjectedProcessEngine(dev)
    try:
        rng = np.random.default_rng(9)
        d, m = 32, 128
        Xa = rng.random((65_536, d), dtype=np.float32)                 # the first staged chunk: 65536 benign points
        Xb = rng.random((234_464, d), dtype=np.float32) * 12.0
        X = np.vstack([Xa, Xb]); y = rng.random(len(X))
        Z = Xa[:m].astype(np.float64)
        k = 1 * sg.ARDRBFKernel(np.full(d, 0.5)) + sg.const(1) * sg.EyeKernel()
        with pytest.raises(ValueError) as e:
            eng.kmeans(Xa[:1000], 1)                                   # k < 2: SGP_E_BADARG before any launch
        out["badarg"] = str(e.value)
        eng.begin(k, Z)
        eng.accumulate(Xa[:5000], y[:5000])
        eng.finish()
        with pytest.raises(sg.TrainingVectorsNotInitializedException) as e:
            eng.predict(Xa[:10].astype(np.float64))
        out["state"] = str(e.value)
        eng.set_precision(N.SGP_PREC_AUTO)
        eng.begin(k, Z)
        eng.accumulate(X, y)
        out["range_path"] = eng.last_path()
        with pytest.raises(sg.OperandRangeError) as e:
            eng.finish()
        out["range"] = str(e.value)
        out["last_error"] = last_error(eng)
    finally:
        eng.close()
    return out


def lifecycle(dev=0):
    """Create a context, evaluate one small BCM objective, destroy the context."""
    spec = dict(SPECS[0], seed=505, bcm_n=40, bcm_d=3)
    X, y, k, _ = bcm_inputs(spec)
    eng = sg.ProjectedProcessEngine(dev)
    try:
        eng.experts_upload_grouped(X, y, spec["bcm_n"])
        return {"bcm": eng.bcm_nll(k), "last_error": last_error(eng)}
    finally:
        eng.close()


def run_threads(jobs):
    """Runs every job in its own thread, all released together; returns their results in order (a job's exception is
    re-raised here)."""
    results, errors = [None] * len(jobs), [None] * len(jobs)
    start = threading.Barrier(len(jobs))

    def run(i, fn):
        try:
            start.wait()
            results[i] = fn()
        except BaseException as ex:                                     # surfaced in the main thread
            errors[i] = ex

    ts = [threading.Thread(target=run, args=(i, fn)) for i, fn in enumerate(jobs)]
    [t.start() for t in ts]
    [t.join() for t in ts]
    for ex in errors:
        if ex is not None:
            raise ex
    return results


@pytest.fixture(scope="module")
def sequential():
    """Every script once, one after another on this thread, on device 0."""
    return [workload(s) for s in SPECS], refusals(), lifecycle()


def check_concurrent(sequential, devices):
    want, want_err, want_life = sequential
    jobs = [lambda s=s, dev=dev: workload(s, dev) for s, dev in zip(SPECS, devices)]
    jobs += [refusals, lifecycle]
    got = run_threads(jobs)
    for i, (g, w) in enumerate(zip(got, want)):
        assert_same(g, w, "context %d (device %d)" % (i, devices[i]))
    assert_same(got[len(SPECS)], want_err, "refusing context")
    assert_same(got[len(SPECS) + 1], want_life, "short-lived context")


# ---------------- the tests --------------------------------------------------------------------------------------------
def test_sequential_scripts_take_the_planned_paths(sequential):
    """The scripts reach what they are meant to: int8 and direct int8 statistics, the register / shared-memory / LU
    objectives, both Laplace kernels, and the refusals with their own texts."""
    runs, err, life = sequential
    for spec, out in zip(SPECS, runs):
        i8 = N.SGP_PREC_I8 if spec["d"] <= 32 else N.SGP_PREC_I8_DIRECT
        for entry in ("host", "device"):
            assert out["stats_i8_%s_path" % entry] == i8 and out["stats_auto_%s_path" % entry] == i8
            assert out["stats_f64_%s_path" % entry] == N.SGP_PREC_F64
        assert out["bcm_path"] == spec["bcm_path"]
        assert out["laplace_chip_path"] == 0 and out["laplace_global_path"] == 1
        assert out["tail_path"] == 1
        for key in ("predict_device", "probability_device"):               # host and device entries: the same bits
            assert canon(list(out[key])) == canon(list(out[key.replace("device", "host")]))
        assert canon(out["sweep_device"]) == canon(out["sweep_host"])
    assert "k" in err["badarg"] and err["state"] and err["range_path"] == N.SGP_PREC_I8
    assert err["last_error"] == err["range"] and err["range"] != err["state"]
    assert np.isfinite(life["bcm"][0])


def test_sequential_scripts_match_oracle(sequential):
    """For diagnosis: one output per family of the first context against the oracle, at its own test's tolerance."""
    out, spec = sequential[0][0], SPECS[0]
    X, y, Z, _, ok, Xt = stats_inputs(spec)
    G0, b0 = _oracle_stats_chunked(ok, X, y, Z)
    G, b = out["stats_f64_host"]
    assert rel(G, G0) < TOL_STATS and rel(b, b0) < TOL_STATS
    k0 = ok().set_hyperparameters(ok().get_hyperparameters()).set_training_vectors(Z)
    mv0, mm0 = oracle.get_magic_vector(k0, G0, b0)
    m0, v0 = oracle.GaussianProjectedProcessRawPredictor(mv0, mm0, k0).predict_many(Xt)
    mean, var = out["predict_host"]
    assert rel(mean, m0) < TOL_PRED and np.abs(var / v0 - 1).max() < TOL_PRED
    X, y, k, ok = bcm_inputs(spec)
    nll0, _ = oracle.regression.bcm_objective(oracle.get_expert_labels_and_kernels(X, y, ok, spec["bcm_n"]),
                                              k.getHyperparameters())
    assert abs(out["bcm"][0] - nll0) <= TOL_NLL * abs(nll0)
    X, y, k, ok = laplace_inputs(spec, spec["lap_n"])
    theta, v0 = k.getHyperparameters(), 0.0
    for (ye, ke), g in zip(oracle.get_expert_labels_and_kernels(X, y, ok, spec["lap_n"]),
                           group_for_experts(len(X), spec["lap_n"])):
        v0 += classification_likelihood_and_gradient(ye, np.zeros(len(g)), ke, theta, TOL_LAP)[0]
    assert abs(out["laplace_chip"][0] - v0) <= TOL_NLL * abs(v0)
    X, init = provider_inputs(spec)
    C0 = okm.kmeans(X, 8, max_iter=10, init_centers=init)[0]
    assert np.abs(out["kmeans_init"][0] - C0).max() <= 1e-9 * np.abs(C0).max()


def test_four_contexts_on_one_gpu(sequential):
    """Four contexts on device 0, one thread each, next to a refusing context and a short-lived one: every output, path
    and error text equals the sequential run's bit for bit."""
    check_concurrent(sequential, [0, 0, 0, 0])


def test_two_contexts_per_gpu_on_two_gpus(sequential):
    import torch
    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    check_concurrent(sequential, [0, 0, 1, 1])


# ---------------- estimators -------------------------------------------------------------------------------------------
def mnist68():
    c = np.load(os.path.join(GOLD, "mnist68_case.npz"))
    n = int(c["n_rows"])
    X = (c["pixels"].astype(np.float64) - c["mean"]) / c["std"]
    return X[:n], c["y01"][:n], X[n:n + 100]


def fit_classifier(n_e):
    X, y, Xte = mnist68()
    gp = (sg.GaussianProcessClassifier().setDatasetSizeForExpert(n_e).setActiveSetSize(100)
          .setKernel(lambda: sg.RBFKernel(10.0)).setTol(1e-3).setMaxIter(3))
    model = gp.fit(X, y)
    return {"theta": model.hyperparameters, "objective": gp.last_objective, "latent": gp.last_latent,
            "raw": model.predictRaw(Xte)}


def fit_regression():
    c = np.load(os.path.join(GOLD, "airfoil_case.npz"))
    X, y = c["X"], c["y"]
    gp = (sg.GaussianProcessRegression().setKernel(lambda: 1 * sg.ARDRBFKernel(5) + sg.const(1) * sg.EyeKernel())
          .setSigma2(float(c["sigma2"])).setDatasetSizeForExpert(100).setActiveSetSize(150).setMaxIter(10)
          .setActiveSetProvider(ExplicitActiveSetProvider(X[::10][:150])))
    model = gp.fit(X, y)
    return {"theta": model.hyperparameters, "objective": gp.last_objective, "stats": gp.last_stats,
            "predict": model.rawPredictor.predict(X[:200])}


def test_estimators_fit_from_three_threads():
    """Two classifier fits (mnist68, experts of 100 and of 60 points) and one regression fit (airfoil), each in its own
    thread with the contexts the estimators take from the pool: theta, the objective record and the predictions equal
    the sequential fits bit for bit."""
    jobs = [lambda: fit_classifier(100), lambda: fit_classifier(60), fit_regression]
    want = [job() for job in jobs]
    got = run_threads(jobs)
    for i, (g, w) in enumerate(zip(got, want)):
        assert_same(g, w, "estimator %d" % i)
