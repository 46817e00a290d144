"""Extended-precision model of the fp64 DMMA statistics kernel (`kmn_gram_f64_kernel`, csrc/gram_f64.cu): the exact
G = K^T K and b = K^T y of an oracle kernel in `np.longdouble` (a 64-bit mantissa on x86-64), K = k(X, Z) in the direct
form sum_t C_t exp(-sum_k ((x_k - z_k) beta_tk)^2), and a bound on each element's distance from the GPU's result.

The kernel flattening (terms, C_t with its rounding count r_t, beta including the RBF beta = fl(1 / fl(fl(sqrt 2) sigma)))
is KernelEvalModel's.  The bound follows the arithmetic of gram_f64.cu, first-order sums with u32 = 2^-24 and
u64 = 2^-53; u is u32 in the fp32-element loops (SGP_PREC_F64) and u64 in strict mode (SGP_PREC_F64_STRICT):
  * centre c: stats_scales in api.cu, the active-set mean rounded to a whole multiple of its standard deviation.  The
    distances do not depend on it; it sets the size of the staged coordinates x^ = (x - c) beta, z^ = (z - c) beta.
  * staging: x~ = fl32(fl(fl(x - c) fl(beta s))) (or fl32(fl(fl(fl(x - c) beta) s)) in the pipelined loop), z~ =
    fl32(fl(-s fl(fl(z - c) beta))), s = fl(sqrt(log2 e)); strict: s = 1 and no fp32 rounding.  Error per coordinate
    (u32 + 3 u64) |x^| (3 u64 strict) plus the smallest subnormal of the element type.
  * d_k = x~ - z~: one more rounding, u (|d_k| + staging errors).
  * q: fp32 loops, two float2 lanes (even and odd dims) of dpad / 2 fma steps each and one add: gamma_u(dpad / 2 + 1);
    strict, one fma chain: gamma_u(dpad).  Plus sum_k (2 |d_k| dd_k + dd_k^2) from the operands, 3 u64 q where
    fl(sqrt(log2 e))^2 ln 2 != 1 (fp32 loops), 6 u64 q from the three roundings of an RBF beta.
  * exponential: fp32 loops, ex2.approx.ftz.f32 within 2 ulp (EX2_REL = 2^-22 relative, the figure the source and the
    PTX ISA give), results below 2^-126 flushed to 0 (absolute FLT_MIN); strict, CUDA's exp within 1 ulp (2 u64, TINY).
    The relative error is expm1(|dq|) + that, so it grows with q and far pairs are judged fairly.
  * C_t ex in fp64 (r_t + 1 roundings of C_t, HALF_TINY), T - 1 fp64 adds across terms.
Each element of K then has an absolute bound a_in.  With R roundings along the longest accumulation path (the points of
the fullest slice -- one DMMA rounding per point --, the slices gram_reduce_kernel adds in order, one G += per launch):
  |G^_ij - G_ij| <= sum_n (k_in a_jn + a_in k_jn + a_in a_jn) + gamma64(R) sum_n (k_in + a_in)(k_jn + a_jn)
  |b^_i - b_i|   <= sum_n a_in |y_n| + gamma64(R_b) sum_n (k_in + a_in) |y_n|
plus n TINY (products in fp64's subnormal range), times SAFETY.  The reference's own error -- the longdouble K and sums
-- is bounded separately (`ref`), added to the gate, and kept below 1/8 of the device bound.
"""
from __future__ import annotations

import numpy as np

from .kernel_eval_model import HALF_TINY, LD, SAFETY, TINY, KernelEvalModel, bound_fraction  # noqa: F401

U32 = LD(2) ** -24
U64 = LD(2) ** -53
ULD = LD(2) ** -64                         # longdouble unit roundoff
FLT_MIN = LD(2) ** -126                    # ex2.approx.ftz flushes results below this to 0
FLT_TRUE_MIN = LD(2) ** -149               # one ulp in fp32's subnormal range
EX2_REL = LD(2) ** -22                     # ex2.approx.f32: 2 ulp
SQRT_LOG2E = float.fromhex("0x1.337cc2183b050p+0")   # kSqrtLog2e, sgp_internal.h
FULL_GRAM_WORK = 4e8                       # n m^2 above which only sampled rows of G are formed in longdouble


def gamma(n, u):
    return n * u / (1 - n * u)


def centre(Z):
    """The fp64 kernel's centre (stats_scales in api.cu): the active-set mean rounded to a whole multiple of its standard
    deviation, the mean itself where the deviation is 0."""
    Z = np.asarray(Z, dtype=np.float64)
    mean = Z.sum(0) / len(Z)
    sd = np.sqrt(((Z - mean) ** 2).sum(0) / len(Z))
    return np.where(sd > 0, np.rint(mean / np.where(sd > 0, sd, 1.0)) * sd, mean)


def sample_rows(m, rng):
    """Rows of G formed in longdouble when the full G is too costly: the first and last row of every 64-row block (the
    128-row tiles and the 64-column staircase edges) and 8 random rows per 128-row tile.  G is exactly symmetric (asserted
    on its own), so these rows cover the columns too."""
    rows = set()
    for r0 in range(0, m, 64):
        rows.update((r0, min(r0 + 63, m - 1)))
    for r0 in range(0, m, 128):
        rows.update(rng.integers(r0, min(r0 + 128, m), 8).tolist())
    return np.array(sorted(rows))


class GramF64Model:
    """G and b of one begin..finish window in longdouble, and per-element bounds of the GPU's fp64 result."""

    def __init__(self, kernel, Z, strict):
        self.kev = KernelEvalModel(kernel)
        self.Z = np.asarray(Z, dtype=np.float64)
        self.strict = strict
        self.c = centre(self.Z)

    def elements(self, X):
        """(K, a, e): K = k(X, Z) in longdouble (n x m), a the bound on each element the kernel computes, e the bound on
        the longdouble K's own error.  X is read as float64 (an fp32 X by its upcast, the bits the GPU converts)."""
        X = np.asarray(X, dtype=np.float64)
        (n, d), m = X.shape, len(self.Z)
        dpad = (d + 3) // 4 * 4
        if self.strict:
            u, srel, floor, L = U64, 3 * U64, TINY, dpad
        else:
            u, srel, floor, L = U32, U32 + 3 * U64, FLT_TRUE_MIN, dpad // 2 + 1
        Xl, Zl, cl = X.astype(LD), self.Z.astype(LD), self.c.astype(LD)
        K, a, e = np.zeros((n, m), LD), np.zeros((n, m), LD), np.zeros((n, m), LD)
        T = len(self.kev.terms)
        for t, term in enumerate(self.kev.terms):
            beta = self.kev.beta(t, d)
            q, dq = np.zeros((n, m), LD), np.zeros((n, m), LD)
            for k in range(d):
                xh, zh = (Xl[:, k] - cl[k]) * beta[k], (Zl[:, k] - cl[k]) * beta[k]
                dk = xh[:, None] - zh[None, :]
                q += dk * dk
                ds = (srel * np.abs(xh) + floor)[:, None] + (srel * np.abs(zh) + floor)[None, :]
                dd = ds + u * (np.abs(dk) + ds) + floor
                dq += 2 * np.abs(dk) * dd + dd * dd
            dq += gamma(L, u) * q + L * floor
            if not self.strict:
                dq += 3 * U64 * q
            if term["kind"] == "rbf":
                dq += 6 * U64 * q
            ex = np.exp(-q)
            rho, eta = (np.expm1(dq) + 2 * U64, TINY) if self.strict else (np.expm1(dq) + EX2_REL, FLT_MIN)
            C = term["C"]
            K += C * ex
            a += C * (ex * (rho + (term["r"] + 1) * U64) + eta)
            e += C * ex * ULD * (3 * d + 8) * (1 + q)
        a += (T - 1) * U64 * K + T * HALF_TINY
        return K, a, e

    def statistics(self, X, y, R, R_b, rows=None, rng=None):
        """dict(rows, G [rows x m], bG, refG, b, bb, refb): the exact statistics, the device bounds (SAFETY included) and
        the reference's own error bounds.  rows None: every row if n m^2 <= FULL_GRAM_WORK, else sample_rows."""
        y = np.asarray(y, dtype=np.float64)
        K, a, e = self.elements(X)
        n, m = K.shape
        if rows is None:
            rows = np.arange(m) if n * m * m <= FULL_GRAM_WORK else sample_rows(m, rng or np.random.default_rng(0))
        G = K[:, rows].T @ K
        b = K.T @ y.astype(LD)
        kf, af, ef = K.astype(np.float64), a.astype(np.float64), e.astype(np.float64)
        ka = kf + af
        cross = kf[:, rows].T @ af + af[:, rows].T @ kf + af[:, rows].T @ af
        kmax = float(kf.max()) if kf.size else 0.0
        bG = (cross.astype(LD) + gamma(R, U64) * (ka[:, rows].T @ ka).astype(LD) + n * (1 + kmax) * TINY) * SAFETY
        refG = (kf[:, rows].T @ ef + ef[:, rows].T @ kf).astype(LD) + gamma(n + 2, ULD) * (kf[:, rows].T @ kf).astype(LD)
        ay = np.abs(y)
        bb = ((af.T @ ay).astype(LD) + gamma(R_b, U64) * (ka.T @ ay).astype(LD) + n * TINY) * SAFETY
        refb = (ef.T @ ay).astype(LD) + gamma(n + 2, ULD) * (kf.T @ ay).astype(LD)
        return dict(rows=rows, K=K, a=a, G=G, bG=bG, refG=refG, b=b, bb=bb, refb=refb)


def reference_share(st):
    """The largest ratio of the reference's own error bound to the device bound, over G and b."""
    return max(float(np.max(st["refG"] / st["bG"])) if st["G"].size else 0.0,
               float(np.max(st["refb"] / st["bb"])) if st["b"].size else 0.0)


def fractions(G, b, st):
    """(G fraction, b fraction): bound_fraction of the GPU's G rows and b against the exact values, the gate being the
    device bound plus the reference's own error."""
    return (bound_fraction(np.asarray(G)[st["rows"]], st["G"], st["bG"] + st["refG"]),
            bound_fraction(b, st["b"], st["bb"] + st["refb"]))
