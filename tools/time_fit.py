"""SURVEY 8(d)(iv): whole `fit` at a fixed maxIter, BASELINE configs[1] shape (GPU box).

    python tools/time_fit.py [N=1000000] [maxIter=20]

Times GaussianProcessRegression.fit (hyper-parameter optimisation on the per-expert BCM objective + projected-process
statistics + m x m tail) on one GPU, with the breakdown, and the same three stages of the CPU restatement on a bounded
sample scaled linearly (every stage is exactly linear in N at fixed m, n_e)."""
import sys, time
sys.path.insert(0, ".")
import numpy as np
import spark_gp_b200 as sg

N_ = int(sys.argv[1]) if len(sys.argv) > 1 else 1_000_000
max_iter = int(sys.argv[2]) if len(sys.argv) > 2 else 20
d, m, n_e = 16, 1000, 100
rng = np.random.default_rng(13)
X = rng.random((N_, d), dtype=np.float32)
y = np.sin(X.astype(np.float64).sum(1)) + 0.1 * rng.standard_normal(N_)

gp = (sg.GaussianProcessRegression().setKernel(lambda: 1 * sg.ARDRBFKernel(np.full(d, np.sqrt(18.0 / d))) + sg.const(1) * sg.EyeKernel())
      .setDatasetSizeForExpert(n_e).setActiveSetSize(m).setSigma2(1e-4).setMaxIter(max_iter).setTol(1e-6).setSeed(13))
# warm-up: CUDA context, cuSOLVER handles, kernels' first-launch costs
sg.GaussianProcessRegression().setKernel(lambda: 1 * sg.ARDRBFKernel(d) + sg.const(1) * sg.EyeKernel()).setActiveSetSize(64).setMaxIter(2).fit(X[:20000], y[:20000])

from spark_gp_b200.hyperopt import optimize_hypers
for rep in range(2):          # the first pass also pays one-off costs (cuSOLVER/cuBLAS kernels for m x m, allocations)
    t0 = time.perf_counter()
    eng = sg.ProjectedProcessEngine.acquire(0)
    theta = optimize_hypers(gp, eng, eng.experts_upload_grouped(X, y, n_e))
    eng.release()
    t1 = time.perf_counter()
    model = gp._produce_model(X, y, theta)
    t2 = time.perf_counter()
    print("pass %d: hyperopt %.3f s, stats+tail %.3f s" % (rep, t1 - t0, t2 - t1), flush=True)
info = gp.last_objective
print("fit N=%d d=%d m=%d n_e=%d maxIter=%d: total %.3f s = hyperopt %.3f s (%d objective evaluations, %d L-BFGS-B iterations, %.1f ms each incl. host) + stats+tail %.3f s"
      % (N_, d, m, n_e, max_iter, t2 - t0, t1 - t0, info["evaluations"], info["iterations"], 1e3 * (t1 - t0) / max(info["evaluations"], 1), t2 - t1), flush=True)
print("fit throughput: %.3e points/s  (objective passes: %.3e point-evaluations/s)" % (N_ / (t2 - t0), N_ * info["evaluations"] / (t1 - t0)), flush=True)
Xt = rng.random((2000, d), dtype=np.float32)
yt = np.sin(Xt.astype(np.float64).sum(1))
pred = model.predict(Xt)
print("held-out RMSE vs noiseless target: %.4f (noise sd 0.1)" % float(np.sqrt(np.mean((np.asarray(pred) - yt) ** 2))), flush=True)

# CPU restatement of the same stages on a sample (oracle; test infrastructure, used here as the timed baseline only)
import oracle
from oracle.regression import bcm_objective
from oracle import cpu_baseline
ns = 20000
fac = oracle.get_kernel(lambda: 1 * oracle.ARDRBFKernel(np.full(d, np.sqrt(18.0 / d))) + oracle.const(1) * oracle.EyeKernel(), 1e-4)
ex = oracle.get_expert_labels_and_kernels(X[:ns].astype(np.float64), y[:ns], fac, n_e)
th0 = fac().get_hyperparameters()
t0 = time.perf_counter(); bcm_objective(ex, th0); dt = time.perf_counter() - t0
cores = cpu_baseline.usable_cores()
per_eval_full = dt * N_ / ns / cores
print("CPU restatement: one objective evaluation %.2f s per %d points on 1 core -> %.1f s per evaluation at N=%d on %d cores (perfect scaling assumed)"
      % (dt, ns, per_eval_full, N_, cores), flush=True)
print("=> %d evaluations would take %.0f s on %d CPU cores" % (info["evaluations"], per_eval_full * info["evaluations"], cores), flush=True)
