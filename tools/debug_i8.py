"""GPU-side bring-up diagnostics for the int8 path (run on the GPU box).
Stage 1: T tile of the distance contraction vs an exact CPU model of the fp16 split operands.
Stage 2: fixed-point words vs round(2^T * C0).   Stage 3: G, b vs the fp64 oracle, several shapes."""
import sys, time
sys.path.insert(0, ".")
import numpy as np
import oracle
import spark_gp_b200 as sg
from spark_gp_b200 import _native as N

C0 = 8355000.0


def emulate_T(X, Z, beta):
    """-q*log2(e) of the fp16 hi/lo represented points (what the distance MMA should produce)."""
    s = np.sqrt(np.log2(np.e)) * beta
    ctr = Z.mean(0)
    def split(A):
        v = (A - ctr) * s
        h = v.astype(np.float16).astype(np.float64)
        l = (v - h).astype(np.float16).astype(np.float64)
        return h, l
    xh, xl = split(X); zh, zl = split(Z)
    xr, zr = xh + xl, zh + zl
    T = 2 * (zh @ xh.T + zl @ xh.T + zh @ xl.T) - (zr * zr).sum(1)[:, None] - (xr * xr).sum(1)[None, :]
    return T   # [active, point]


def case(n, d, m, seed=0, check_dbg=False, label=""):
    rng = np.random.default_rng(seed)
    X = rng.random((n, d), dtype=np.float32)
    y = np.sin(X.astype(np.float64).sum(1)) + 0.1 * rng.standard_normal(n)
    Z = rng.random((m, d))
    beta = np.full(d, np.sqrt(18.0 / d))
    C = 1.7
    k = C * sg.ARDRBFKernel(beta) + sg.const(1) * sg.EyeKernel() + sg.const(1e-4) * sg.EyeKernel()
    ok = lambda: C * oracle.ARDRBFKernel(beta) + oracle.const(1) * oracle.EyeKernel() + oracle.const(1e-4) * oracle.EyeKernel()
    t00 = time.perf_counter()
    e = sg.ProjectedProcessEngine(0)
    e.set_precision(N.SGP_PREC_I8)
    if check_dbg:
        e.debug_i8_tile()
    e.begin(k, Z)
    t0 = time.perf_counter()
    e.accumulate(X, y)
    G, b = e.finish()
    dt = time.perf_counter() - t0
    if check_dbg:
        T, w = e.debug_i8_tile()
        Te = emulate_T(X[:64].astype(np.float64), Z[:128], beta)
        rows = min(m, 128); cols = min(n, 64)
        dT = np.abs(T[:rows, :cols] - Te[:rows, :cols]).max()
        dd = (T[:rows, :cols] - Te[:rows, :cols])
        print("  [dbg] max|T - T_emul| = %.3e  mean(T - T_emul) = %.3e  rms = %.3e (T range %.2f..%.2f)" % (dT, dd.mean(), np.sqrt((dd ** 2).mean()), Te[:rows, :cols].min(), Te[:rows, :cols].max()))
        u = (w & 0x7FFFFF).astype(np.int64) - 0x4040
        ue = np.rint(np.exp2(T.astype(np.float64)) * C0)
        print("  [dbg] max|u - rint(2^T*C0)| = %d ; top byte ok: %s" % (np.abs(u[:rows, :cols] - ue[:rows, :cols]).max(), bool(np.all((w[:rows, :cols] >> 24) == 0x4B))))
    ex = oracle.get_expert_labels_and_kernels(X.astype(np.float64), y, ok, 100)
    for _, kk in ex:
        kk.set_hyperparameters(ok().get_hyperparameters())
    G0, b0 = oracle.get_matrix_kmn_knm_and_vector_kmny(ex, Z)
    eg = np.abs(G - G0).max() / np.abs(G0).max()
    eb = np.abs(b - b0).max() / np.abs(b0).max()
    sym = np.array_equal(G, G.T)
    print("%-28s n=%-7d d=%-3d m=%-5d dG=%.2e db=%.2e sym=%s  (%.1f ms; case wall %.1f s)" % (label, n, d, m, eg, eb, sym, dt * 1e3, time.perf_counter() - t00), flush=True)
    e.close()
    return eg, eb


if __name__ == "__main__":
    case(64, 16, 128, check_dbg=True, label="one unit, diag tile")
    case(200, 16, 128, check_dbg=True, label="ragged units, diag")
    case(1000, 16, 256, label="off-diagonal tile")
    case(5000, 5, 300, label="d=5, m ragged")
    case(5000, 32, 384, label="d=32 (2 K chunks)")
    case(20000, 16, 1000, label="36 tiles x 4 slices")
    case(300000, 16, 256, label="fold boundary (>25600/slice)")
    # throughput at BASELINE configs[1]
    import ctypes as C
    rng = np.random.default_rng(1)
    n, d, m = 1_000_000, 16, 1000
    X = rng.random((n, d), dtype=np.float32); y = rng.random(n)
    Z = X[:m].astype(np.float64)
    k = 1 * sg.ARDRBFKernel(np.full(d, np.sqrt(18.0 / d))) + sg.const(1) * sg.EyeKernel() + sg.const(1e-4) * sg.EyeKernel()
    e = sg.ProjectedProcessEngine(0)
    for mode, name in ((N.SGP_PREC_I8, "I8"), (N.SGP_PREC_F64, "F64")):
        e.set_precision(mode)
        for rep in range(3):
            e.begin(k, Z)
            t0 = time.perf_counter(); e.accumulate(X, y); G, b = e.finish(); dt = time.perf_counter() - t0
            ms, nl = e.gram_kernel_time()
            print("%s rep %d: host->G %.1f ms, gram kernels %.2f ms (%d launches) -> %.1f Mpts/s kernel-only" % (name, rep, dt * 1e3, ms, nl, n / ms / 1e3), flush=True)
        if mode == N.SGP_PREC_I8: G8, b8 = G, b
    print("I8 vs F64 at 1M: dG=%.2e db=%.2e" % (np.abs(G8 - G).max() / np.abs(G).max(), np.abs(b8 - b).max() / np.abs(b).max()))
