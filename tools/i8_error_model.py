"""CPU emulation of the int8 path's arithmetic (design study, not product code): which error term moves the
posterior mean?  (a) fixed-point quantisation + dropped low-digit products (exact integer model);
(b) fp32 accumulation of T = -q log2 e in the tensor core, modelled as round-toward-zero at each k-step."""
import sys, time
import numpy as np
sys.path.insert(0, ".")
import oracle
from oracle import ARDRBFKernel, EyeKernel, const

C0 = 8355000.0

def rz32(x):                       # round a float64 array toward zero to fp32 precision
    y = x.astype(np.float32).astype(np.float64)
    over = np.abs(y) > np.abs(x)
    y[over] = np.nextafter(y[over].astype(np.float32), np.float32(0)).astype(np.float64)
    return y

def split16(v):
    h = v.astype(np.float16).astype(np.float64)
    l = (v - h).astype(np.float16).astype(np.float64)
    return h, l

def T_model(X, Z, beta, mode):
    s = np.sqrt(np.log2(np.e)) * beta
    ctr = Z.mean(0)
    xh, xl = split16((X - ctr) * s); zh, zl = split16((Z - ctr) * s)
    xr, zr = xh + xl, zh + zl
    parts = [2 * xh @ zh.T, 2 * xh @ zl.T, 2 * xl @ zh.T, (-(xr * xr).sum(1))[:, None] + (-(zr * zr).sum(1))[None, :]]
    if mode == "exact":
        return sum(parts)
    acc = np.zeros_like(parts[0])
    for p_ in parts:               # one rounding per k-step
        acc = rz32(acc + p_) if mode == "rz" else (acc + p_).astype(np.float32).astype(np.float64)
    return acc

def gram_from_T(T, y, full_products=False):
    """The kernel's digit layout: u = s2*2^15 + s1*2^7 + s0, s2 in [0,255] (unsigned operand), s1 in [-128,127],
    s0 in [-64,63]; stored planes P2 = s2, P1 = s1, P0 = 2 s0 are the base-256 digits of W = 2u."""
    kap = np.exp2(T)
    u = np.rint(kap * C0).astype(np.int64)
    t = u + 0x4040
    f = lambda a: a.astype(np.float64)      # exact: |sums| < 2^53
    P0, P1, P2 = f(2 * ((t & 127) - 64)), f(((t >> 7) & 255) - 128), f(t >> 15)
    g = 2.0 ** 32 * (P2.T @ P2) + 2.0 ** 24 * (P2.T @ P1 + P1.T @ P2) + 2.0 ** 16 * (P2.T @ P0 + P0.T @ P2 + P1.T @ P1)
    if full_products:
        g = g + 2.0 ** 8 * (P1.T @ P0 + P0.T @ P1) + P0.T @ P0
    return g / (4.0 * C0 ** 2), (kap.T @ y)


def gram_from_T_byte_aligned(T, y):
    """The first layout (byte-aligned digits of u: s2 only 7 bits), kept for comparison."""
    kap = np.exp2(T)
    u = np.rint(kap * C0).astype(np.int64)
    t = u + 0x8080
    f = lambda a: a.astype(np.float64)
    S0, S1, S2 = f((t & 255) - 128), f(((t >> 8) & 255) - 128), f(t >> 16)
    g = 2.0 ** 32 * (S2.T @ S2) + 2.0 ** 24 * (S2.T @ S1 + S1.T @ S2) + 2.0 ** 16 * (S2.T @ S0 + S0.T @ S2 + S1.T @ S1)
    return g / C0 ** 2, (kap.T @ y)


def main(N=200000, d=16, m=1000, chunk=20000):
    rng = np.random.default_rng(13)
    X = rng.random((N + 1000, d), dtype=np.float32).astype(np.float64)
    y = np.sin(X.sum(1)) + 0.1 * rng.standard_normal(N + 1000)
    Xt, X, y = X[N:], X[:N], y[:N]
    beta = np.full(d, np.sqrt(18.0 / d))
    Z = X[np.random.default_rng(7).permutation(N)[:m]]
    variants = {"fp64": None, "fixedpoint_fullprod+exactT": ("exact", True), "digits_dropped+exactT": ("exact", False),
                "digits+T_rn32": ("rn", False), "digits+T_rz32": ("rz", False), "byte_aligned_digits+T_rz32": ("rz", None)}
    G = {k: np.zeros((m, m)) for k in variants}; b = {k: np.zeros(m) for k in variants}
    for s in range(0, N, chunk):
        Xc, yc = X[s:s + chunk], y[s:s + chunk]
        Xb, Zb = Xc * beta, Z * beta
        q = np.maximum((Xb * Xb).sum(1)[:, None] + (Zb * Zb).sum(1)[None, :] - 2 * Xb @ Zb.T, 0)
        K = np.exp(-q); G["fp64"] += K.T @ K; b["fp64"] += K.T @ yc
        for name, cfg in variants.items():
            if cfg is None: continue
            g, bb = (gram_from_T_byte_aligned(T_model(Xc, Z, beta, cfg[0]), yc) if cfg[1] is None
                     else gram_from_T(T_model(Xc, Z, beta, cfg[0]), yc, cfg[1]))
            G[name] += g; b[name] += bb
    fac = oracle.get_kernel(lambda: 1 * ARDRBFKernel(d) + const(1) * EyeKernel(), 1e-4)
    kern = fac().set_hyperparameters(np.concatenate([[1.0], beta])).set_training_vectors(Z)
    ref = None
    print("N=%d" % N)
    for name in variants:
        mv, mm = oracle.get_magic_vector(kern, G[name], b[name])
        mean, var = oracle.GaussianProjectedProcessRawPredictor(mv, mm, kern).predict_many(Xt)
        if ref is None: ref = (mean, var)
        print("%-30s dG=%.2e dmean=%.2e dvar=%.2e" % (name, np.abs(G[name] - G["fp64"]).max() / np.abs(G["fp64"]).max(),
              np.abs(mean - ref[0]).max() / np.abs(ref[0]).max(), np.abs(var / ref[1] - 1).max()), flush=True)

if __name__ == "__main__":
    main(*[int(a) for a in sys.argv[1:]])
