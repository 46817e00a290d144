"""Extended-precision model of prediction (`sgp_predict`, `sgp_predict_probability` and their device entries,
csrc/predict.cu): the exact mean k v, variance selfKernel + k M k^T and averaged probability of each point in
`np.longdouble` (a 64-bit mantissa on x86-64), and a bound on each output's distance from the GPU's fp64 result.

The bound follows the arithmetic of predict.cu, first-order sums with u = 2^-53:
  * elements k(x, z_j) (`predict_elements_kernel`): x~ = fl(fl(x - c) beta) with the fp64 kernel's centre c (the
    `stats_scales` value that `sgp_stats_begin` writes after the betas in dBeta), z~ = fl(fl(z - c) beta) from Zc
    (`scale_rows_kernel`), d_k = fl(x~ - z~), q one fp64 fma chain over dpad, each term folded by fma(C_t, exp(-q), acc)
    with CUDA's exp within 1 ulp; no Eye terms in a cross kernel.  That is the strict loop of the fp64 Gram
    (`GramF64Model.elements(strict=True)`): the same two staging roundings (its 3u per coordinate covers them), the same
    chain length L = dpad, and its per-term product plus T - 1 adds bound the fma fold (T roundings of partial sums, the
    first of C_t e_t itself).  So the element bound a_j is that model's, unchanged.
  * mean (`predict_elements_kernel`): per thread an fma chain over the m_pad / kElemCols column tiles, a butterfly over
    the 32 lanes of a warp, then the kElemCols / 32 warps added in order:
      R_mean = m_pad / kElemCols + log2(32) + kElemCols / 32 - 1
      |mean^ - mean| <= sum_j a_j |v_j| + gamma(R_mean) sum_j (k_j + a_j) |v_j|
  * variance (`pack_magic_kernel`, `predict_var_kernel`, `predict_var_reduce_kernel`): B = triu(M + M^T, 1) + diag(M),
    one rounding per off-diagonal entry; W_rc = sum_i K_ri B_ic by DMMA over kVarCols (C + 1) products, counted as one
    rounding each (conservative, the fp64 Gram model's premise); the epilogue's kVarCols / 8 fmas, two quad shuffle adds
    and one add of the two column warps; the n_ct = ceil(m / kVarCols) column-tile partials added in order from 0.0;
    selfKernel added once:
      R_var = kVarCols n_ct + (kVarCols / 8 + 3) + n_ct + 1
      |var^ - var| <= sum_ij |M_ij| (a_i k_j + k_i a_j + a_i a_j) + u sum_{i<j} (k + a)_i |M_ij + M_ji| (k + a)_j
                      + gamma(R_var) (selfKernel + (k + a) |B| (k + a)^T) + the rounding of selfKernel itself
    selfKernel is flatten_kernel's sum of the leaf scales from 0.0 (api.cu), each scale the Python layer's product along
    the leaf's path.
  * probability (`predict_var_reduce_kernel<true>`), judged on the device's own fp64 (mean, var) and the library's rule
    (`sgp_gauss_hermite_rule`, the bits `predict_prepare` uploads), so that only the kernel's arithmetic is measured:
    sd2 = fl(sqrt(2 max(v, 0))), z_i = fl(mu + fl(sd2 x_i)) (not contracted), e = exp(-z) within 1 ulp, fl(1 + e), the
    division, an fma chain over the nodes and the product with kRsqrtPi (with its own representation error).  Relative
    to sigma_i:  (1 - sigma_i)(|dz_i| + 2u) + 2u,  |dz_i| <= 2u |sd2 x_i| + u |z_i|;  then gamma(n + 1) for the chain and
    the last product.  Absolute floors where sigma_i leaves fp64's normal range: exp(-z) overflows for z < -709.78 and
    the device's sigma is 0; just above that sigma is subnormal and its division and fma are rounded absolutely.
Every bound carries small absolute floors for results in fp64's subnormal range, and SAFETY for the products of rounding
errors that first-order sums leave out.  The reference's own error (longdouble K, longdouble sums) is bounded
separately, added to the gate, and kept below 1/8 of the device bound.

Forming k M k^T in longdouble costs n m^2; above SAMPLE_WORK only sampled points are modelled (`sample_points`).
"""
from __future__ import annotations

import numpy as np

from .gram_f64_model import GramF64Model, gamma
from .kernel_eval_model import HALF_TINY, LD, SAFETY, TINY, bound_fraction  # noqa: F401

U = LD(2) ** -53
ULD = LD(2) ** -64                        # longdouble unit roundoff
DBL_MIN = LD(2) ** -1022
RSQRT_PI = 0.56418958354775628695         # kRsqrtPi, predict.cu (as the compiler rounds it)
SAMPLE_WORK = 3e8                         # n m^2 above which only sampled points are modelled

# tile constants of predict.cu (tests/test_host_predict_model.py reads them from the source)
ELEM_COLS = 128                           # kElemCols: active-set columns per element tile, one per thread
ELEM_PTS = 16                             # kElemPts: points per point group, two groups per element CTA
VAR_ROWS = 128                            # kVarRows: points per variance row tile
VAR_COLS = 64                             # kVarCols: columns per variance column tile
WARP = 32


def m_padded(m):
    """m_pad: m rounded up to whole element tiles (kTile = kElemCols = 128)."""
    return (m + ELEM_COLS - 1) // ELEM_COLS * ELEM_COLS


def rounding_counts(m):
    """(R_mean, R_var) of an active set of m points, from the tile constants."""
    n_ct = (m + VAR_COLS - 1) // VAR_COLS
    r_mean = m_padded(m) // ELEM_COLS + int(np.log2(WARP)) + ELEM_COLS // WARP - 1
    epilogue = VAR_COLS // 8 + 2 + 1           # 8 columns per lane of a quad, the quad's two shuffles, two column warps
    r_var = VAR_COLS * n_ct + epilogue + n_ct + 1
    return r_mean, r_var


def sample_points(n, rng, windows=(), count=64):
    """Points modelled when the whole set is too costly.  Every point's arithmetic is the same wherever it lands, so the
    sample is the edges where the indexing changes -- the first and last point of the first two and the last 16-point
    group, 32-point element CTA and 128-row variance tile, and of each window (a list of (start, length)) -- and `count`
    points drawn at random."""
    pts = {0, n - 1}
    for unit in (ELEM_PTS, 2 * ELEM_PTS, VAR_ROWS):
        last = (n - 1) // unit
        for u in {0, 1, last}:
            pts.update((u * unit, min(u * unit + unit - 1, n - 1)))
    for w0, wn in windows:
        pts.update((w0, w0 + wn - 1))
    pts.update(rng.integers(0, n, count).tolist())
    return np.array(sorted(p for p in pts if 0 <= p < n))


class PredictModel:
    """Mean, variance and probability of the installed magic pair (v, M) in longdouble, with per-output bounds of the
    GPU's fp64 results.  kernel: the oracle kernel (its hyper-parameters set); Z: the active set (m x d)."""

    def __init__(self, kernel, Z, v, M):
        self.gram = GramF64Model(kernel, Z, strict=True)
        self.kev = self.gram.kev
        self.m = len(Z)
        self.v = np.asarray(v, dtype=np.float64)
        self.M = np.asarray(M, dtype=np.float64)
        self.R_mean, self.R_var = rounding_counts(self.m)
        Ml = self.M.astype(LD)
        self.B = np.triu(Ml + Ml.T, 1) + np.diag(np.diag(Ml))       # exact; the device rounds the off-diagonal
        self.self_k = sum((t["C"] for t in self.kev.terms), LD(0)) + self.kev.eye
        # each leaf scale within r_t roundings of its exact product, then one add per leaf; eye_r already counts the
        # roundings and adds of the Eye leaves
        r_max = max([t["r"] for t in self.kev.terms], default=0)
        self.self_k_err = gamma(r_max + len(self.kev.terms) + self.kev.eye_r + 1, U) * self.self_k

    def elements(self, X):
        """(K, a, e): K = k(X, Z) in longdouble, a the bound on each element the kernel computes, e the bound on the
        longdouble K's own error.  X is read as float64 (an fp32 X by its upcast, the bits the GPU converts)."""
        return self.gram.elements(X)

    def predict(self, X, with_var=True):
        """dict(K, a, e, mean, bmean, rmean[, var, bvar, rvar]) for the rows of X: exact values, device bounds (SAFETY
        included) and the reference's own error bounds."""
        K, a, e = self.elements(X)
        kf, af, ef = K.astype(np.float64), a.astype(np.float64), e.astype(np.float64)
        ka = kf + af
        av = np.abs(self.v)
        m = self.m
        out = dict(K=K, a=a, e=e, mean=K @ self.v.astype(LD))
        out["bmean"] = ((af @ av).astype(LD) + gamma(self.R_mean, U) * (ka @ av).astype(LD)
                        + (self.R_mean + 1) * TINY) * SAFETY
        out["rmean"] = (ef @ av).astype(LD) + gamma(m + 2, ULD) * (kf @ av).astype(LD)
        if not with_var:
            return out
        out["var"] = self.self_k + np.einsum("ti,ti->t", K @ self.M.astype(LD), K)
        aM = np.abs(self.M)
        aB = np.abs(self.B).astype(np.float64)
        kerr = (np.einsum("ti,ti->t", af @ aM, kf) + np.einsum("ti,ti->t", kf @ aM, af)
                + np.einsum("ti,ti->t", af @ aM, af))
        pack = float(U) * np.einsum("ti,ti->t", ka @ np.triu(aB, 1), ka)
        quad = float(self.self_k) + np.einsum("ti,ti->t", ka @ aB, ka)
        floor = (self.R_var + m) * (1 + float(aB.max(initial=0.0))) * (1 + float(kf.max(initial=0.0))) * TINY
        out["bvar"] = ((kerr + pack).astype(LD) + gamma(self.R_var, U) * quad.astype(LD) + self.self_k_err
                       + floor) * SAFETY
        out["rvar"] = ((np.einsum("ti,ti->t", ef @ aM, kf) + np.einsum("ti,ti->t", kf @ aM, ef)).astype(LD)
                       + gamma(m + 3, ULD) * (float(self.self_k) + np.einsum("ti,ti->t", kf @ aM, kf)).astype(LD))
        return out


def probability(mean, var, nodes, weights):
    """(p, bound, ref) for the device's fp64 (mean, var) under the rule (nodes, weights) the library uploads: p the exact
    averaged probability in longdouble, bound the device bound (SAFETY included), ref the reference's own error bound.
    NaN inputs give NaN p."""
    mu = np.asarray(mean, dtype=np.float64).astype(LD)[:, None]
    vv = np.asarray(var, dtype=np.float64)
    x = np.asarray(nodes, dtype=np.float64)
    w = np.asarray(weights, dtype=np.float64).astype(LD)
    sd2 = np.sqrt(2 * np.where(vv < 0.0, 0.0, vv).astype(LD))[:, None]
    sx = sd2 * x.astype(LD)
    z = mu + sx
    with np.errstate(over="ignore"):                         # z below longdouble's range: sigma is 0 there
        sig = 1 / (1 + np.exp(-z))
    rsqrt_pi = 1 / np.sqrt(np.arccos(LD(-1)))
    p = (sig @ w) * rsqrt_pi
    dz = (2 * U * (1 + 2 * U)) * np.abs(sx) + U * (1 + U) * np.abs(z) + 2 * TINY
    one_minus = 1 - sig
    rho = (one_minus + dz) * np.expm1(dz) + one_minus * 2 * U + 2 * U
    # sigma at or below fp64's normal range (z < -706.6): the device's 0 where exp(-z) overflows, or a subnormal off by
    # its absolute roundings; twice the exact sigma, so that a fraction near 1 always means a relative error
    low = sig < 4 * DBL_MIN
    floor_node = np.where(low, 2 * sig * (1 + rho) + 2 * TINY, LD(0))
    n = len(x)
    rep = abs(LD(RSQRT_PI) - rsqrt_pi) / rsqrt_pi
    bound = (((sig * rho + floor_node) @ w) * rsqrt_pi + (gamma(n + 1, U) + rep) * p + (n + 2) * TINY) * SAFETY
    # the longdouble z, exp, sum and division: the device's error terms with ULD in place of u
    ref = ((sig * ((one_minus + 4 * ULD) * 4 * ULD * (np.abs(sx) + np.abs(z) + 1) + 4 * ULD)) @ w) * rsqrt_pi \
        + (n + 4) * ULD * p
    return p, bound, ref


def reference_share(st, prob=None):
    """The largest ratio of the reference's own error bound to the device bound over the mean, the variance (where
    modelled) and the probability (prob = (p, bound, ref))."""
    shares = [float(np.max(st["rmean"] / st["bmean"])) if len(st["mean"]) else 0.0]
    if "var" in st and len(st["var"]):
        shares.append(float(np.max(st["rvar"] / st["bvar"])))
    if prob is not None and len(prob[0]):
        ok = np.isfinite(prob[0])
        if ok.any():
            shares.append(float(np.max(prob[2][ok] / prob[1][ok])))
    return max(shares)


def fractions(st, mean, var=None):
    """(mean fraction, var fraction): bound_fraction of the GPU's outputs, the gate being the device bound plus the
    reference's own error."""
    fm = bound_fraction(mean, st["mean"], st["bmean"] + st["rmean"])
    fv = bound_fraction(var, st["var"], st["bvar"] + st["rvar"]) if var is not None else 0.0
    return fm, fv


def probability_fraction(got, prob):
    p, bound, ref = prob
    return bound_fraction(got, p, bound + ref)
