"""Extended-precision model of kernel evaluation (`sgp_kernel_eval`, `sgp_kernel_eval_device`, csrc/kernel_eval.cu): K and
every dK of an oracle kernel tree in `np.longdouble` (a 64-bit mantissa on x86-64), with a bound on each element's
distance from the GPU's fp64 result.

The bound follows the arithmetic that kernel_eval.cu's header documents, with u = 2^-53 and first-order error sums:
  * CROSS    df_k = fma(a_k, beta_k, -fl(b_k beta_k)):        |d df_k| <= u (|df_k| + |b_k beta_k|)
    TRAINING df_k = fl(a_k beta_k) - fl(b_k beta_k):          |d df_k| <= u (|a_k beta_k| + |b_k beta_k| + |df_k|)
    (each plus two roundings in fp64's subnormal range, HALF_TINY each)
  * q_t = sum_k df_k^2 by an fma chain of d roundings:        |d q_t| <= gamma_d q_t + sum_k (2 |df_k| |d df_k| + d df_k^2)
    RBF terms also read beta = fl(1 / fl(fl(sqrt 2) sigma)), three roundings of the exact 1/(sqrt 2 sigma): + 6u q_t
  * e_t = exp(-q_t), CUDA's exp within 1 ulp:                 relative rho_t = expm1(|d q_t|) + 2u, plus TINY absolute
  * K = fma fold of C_t e_t over the T terms:                 sum_t C_t e_t (rho_t + r_t u) + T (u K + HALF_TINY)
    + sum_t C_t TINY, then on the TRAINING diagonal one more rounding for the Eye sum
  * ARD (t, k):  fl(fl(-2 beta_k fl(fl(a_k - b_k)^2)) fl(C_t e_t)): relative 4u + (rho_t + (r_t + 1) u) + u, and the
    absolute errors of each factor times the other
  * RBF t:       fl(fl(fl(s2 e_t) / fl(fl(sigma sigma) sigma)) C_t), s2 = sum_k fl(fl(a_k - b_k)^2) added in order:
    relative (d + 2) u + rho_t + u + 3u + (r_t + 1) u, absolute errors carried through the division and the product
  * SCALE:       the fma fold of coef_t e_t, plus the Eye coefficient on the TRAINING diagonal: as K
r_t counts the roundings in the double C_t (or coefficient) the library gets: the Python layer multiplies the scalars
on a term's path one by one from 1.0, and adds the Eye coefficients one by one from 0.0.

The absolute terms make subnormal and zero results fair: e_t may be off by TINY = 2^-1074 where it is subnormal, and
each later rounding in that range by HALF_TINY.  They are carried through the products, so a derivative plane whose
factor -2 beta_k d_k^2 is large gets a correspondingly larger floor.  SAFETY covers the products of two rounding errors
that the first-order sums leave out (far below 2^-20 of the bound in every case the tests build).  Where fl(sigma^3)
overflows fp64 (sigma above about 5.6e102) the RBF plane is 0, which the bound accepts only while the exact value is
below its floor; no case here comes near that.
"""
from __future__ import annotations

import numpy as np

from . import kernels as ok

LD = np.longdouble
U = LD(2) ** -53
TINY = LD(2) ** -1074          # one ulp in fp64's subnormal range
HALF_TINY = LD(2) ** -1075     # the largest rounding error of a result in that range
SAFETY = LD(1) + LD(2) ** -20


def gamma(n):
    return n * U / (1 - n * U)


def kernel_shapes(rng, d):
    """(name, factory) pairs: factory(m) builds the kernel with the DSL of module m (the library or the oracle).  The five
    shapes of tests/test_gpu_kernel_eval.py -- ARD, RBF, Eye only, nested trainable scalars with white noise, four
    non-Eye terms with Eye terms -- and a trainable scalar around a sum with Eye terms."""
    b1 = rng.uniform(0.2, 1.5, d) / np.sqrt(d)
    b1[::3] = 0.0
    b2 = rng.uniform(0.1, 1.0, d) / np.sqrt(d)
    s = float(np.sqrt(d))
    return [
        ("ard", lambda m: 1 * m.ARDRBFKernel(b1)),
        ("rbf", lambda m: m.RBFKernel(0.8 * s)),
        ("eye", lambda m: m.const(0.5) * m.EyeKernel()),
        ("nested", lambda m: m.Scalar(0.7) * (2.0 * m.ARDRBFKernel(b1) + m.Scalar(0.3) * m.RBFKernel(0.6 * s))
         + m.const(0.25) * m.EyeKernel() + m.WhiteNoiseKernel(0.1, 0.0, 1.0)),
        ("four", lambda m: 0.5 * m.ARDRBFKernel(b1) + m.const(0.3) * m.ARDRBFKernel(b2) + 0.2 * m.RBFKernel(s)
         + m.Scalar(0.1) * m.RBFKernel(0.5 * s) + m.WhiteNoiseKernel(0.05, 0.0, 1.0) + m.const(1e-3) * m.EyeKernel()),
        ("scaled_sum", lambda m: m.Scalar(0.6) * (m.Scalar(0.5) * m.ARDRBFKernel(b1) + m.RBFKernel(0.7 * s)
                                                  + m.const(0.2) * m.EyeKernel() + m.WhiteNoiseKernel(0.1, 0.0, 1.0))),
    ]


def _walk(k, path, leaves, hypers):
    """Leaves (kind, path, beta or sigma) in flatten order and hyper-parameters in getHyperparameters order; a path is
    the list of (scalar id or None for a constant, C) above the leaf."""
    if isinstance(k, ok.SumOfKernels):
        _walk(k.kernel1, path, leaves, hypers)
        _walk(k.kernel2, path, leaves, hypers)
    elif isinstance(k, ok.TrainableScalarTimesKernel):
        sid = len(hypers)
        hypers.append(("scale", sid))
        _walk(k.kernel, path + [(sid, k.C)], leaves, hypers)
    elif isinstance(k, ok.ConstantTimesKernel):
        _walk(k.kernel, path + [(None, k.C)], leaves, hypers)
    elif isinstance(k, ok.EyeKernel):
        leaves.append(("eye", path, None))
    elif isinstance(k, ok.ARDRBFKernel):
        hypers.extend(("ard", len(leaves), j) for j in range(len(k.beta)))
        leaves.append(("ard", path, np.asarray(k.beta, dtype=np.float64)))
    elif isinstance(k, ok.RBFKernel):
        hypers.append(("rbf", len(leaves)))
        leaves.append(("rbf", path, k.sigma))
    else:
        raise TypeError("no model for %r" % type(k).__name__)


def _product(factors):
    """The exact product (longdouble) and the roundings of the library's double product taken from 1.0."""
    p = LD(1)
    for c in factors:
        p *= LD(c)
    return p, max(len(factors) - 1, 0)


class KernelEvalModel:
    """K and dK of an oracle kernel in longdouble, and a bound on each element of the GPU's result."""

    def __init__(self, kernel):
        leaves, hypers = [], []
        _walk(kernel, [], leaves, hypers)
        self.terms = []                 # non-Eye terms in flattened order: dict(kind, C, r, beta, sigma)
        flat_of = {}
        eye, eye_r = [], []
        for li, (kind, path, v) in enumerate(leaves):
            C, r = _product([c for _, c in path])
            if kind == "eye":
                eye.append(C)
                eye_r.append(r)
                continue
            flat_of[li] = len(self.terms)
            self.terms.append(dict(kind=kind, C=C, r=r, beta=v.astype(LD) if kind == "ard" else None,
                                   sigma=None if kind == "ard" else LD(v)))
        self.eye, self.eye_r = self._sum(eye, eye_r)
        self.hypers = []                # ("ard", t, k) | ("rbf", t) | ("scale", coef[T], r[T], eye coef, eye r)
        for h in hypers:
            if h[0] == "ard":
                self.hypers.append(("ard", flat_of[h[1]], h[2]))
            elif h[0] == "rbf":
                self.hypers.append(("rbf", flat_of[h[1]]))
            else:
                coef, r = [LD(0)] * len(self.terms), [0] * len(self.terms)
                ec, er = [], []
                for li, (kind, path, _) in enumerate(leaves):
                    if all(s != h[1] for s, _ in path):
                        continue
                    c, rc = _product([c for s, c in path if s != h[1]])
                    if kind == "eye":
                        ec.append(c)
                        er.append(rc)
                    else:
                        coef[flat_of[li]], r[flat_of[li]] = c, rc
                self.hypers.append(("scale", coef, r) + self._sum(ec, er))

    @staticmethod
    def _sum(values, rounds):
        """A sum of nonnegative doubles the library adds one by one from 0.0: exact value, roundings bound."""
        if not values:
            return LD(0), 0
        return sum(values, LD(0)), max(rounds) + len(values) - 1

    def beta(self, t, d):
        """The feature scales of term t: the ARD betas, or 1 / (sqrt 2 sigma) for an RBF term."""
        term = self.terms[t]
        if term["kind"] == "ard":
            return term["beta"]
        return np.full(d, LD(1) / (np.sqrt(LD(2)) * term["sigma"]))

    def evaluate(self, A, B=None, derivatives=True):
        """(K, bound of K, dK, bound of dK) for crossKernel rows A against B, or the training kernel of A (B None), as
        longdouble arrays; dK is [n_hypers, n, m] in getHyperparameters order.  A and B are read as float64 (an fp32 A
        by its upcast, the bits the GPU converts it to)."""
        training = B is None
        A = np.asarray(A, dtype=np.float64)
        B = A if training else np.asarray(B, dtype=np.float64)
        (n, d), m = A.shape, B.shape[0]
        Al, Bl = A.astype(LD), B.astype(LD)
        e, rho = [], []
        for t, term in enumerate(self.terms):
            beta = self.beta(t, d)
            q, dq = np.zeros((n, m), LD), np.zeros((n, m), LD)
            for k in range(d):
                ab, bb = Al[:, k, None] * beta[k], Bl[None, :, k] * beta[k]
                df = ab - bb
                ddf = U * (np.abs(df) + np.abs(bb) + (np.abs(ab) if training else 0)) + 2 * HALF_TINY
                q += df * df
                dq += 2 * np.abs(df) * ddf + ddf * ddf
            dq += gamma(d) * q + d * HALF_TINY + (6 * U * q if term["kind"] == "rbf" else 0)
            e.append(np.exp(-q))
            rho.append(np.expm1(dq) + 2 * U)
        diag = np.eye(n, m, dtype=bool) if training else None
        K, bK = self._fold((n, m), [t["C"] for t in self.terms], [t["r"] for t in self.terms], e, rho, diag,
                           self.eye, self.eye_r)
        if not derivatives:
            return K, bK, None, None
        dK = np.empty((len(self.hypers), n, m), LD)
        bdK = np.empty_like(dK)
        s2 = np.zeros((n, m), LD)
        for k in range(d):
            dk = Al[:, k, None] - Bl[None, :, k]
            s2 += dk * dk
        for h, hp in enumerate(self.hypers):
            if hp[0] == "scale":
                dK[h], bdK[h] = self._fold((n, m), hp[1], hp[2], e, rho, diag, hp[3], hp[4])
                continue
            t = hp[1]
            C, r = self.terms[t]["C"], self.terms[t]["r"]
            E, rE, aE = C * e[t], rho[t] + (r + 1) * U, C * TINY + HALF_TINY
            if hp[0] == "ard":
                k = hp[2]
                dk = Al[:, k, None] - Bl[None, :, k]
                bk = self.terms[t]["beta"][k]
                P, rP, aP = -2 * bk * dk * dk, 4 * U, (2 * abs(bk) + 1) * HALF_TINY
                dK[h] = P * E
                bdK[h] = np.abs(dK[h]) * (rP + rE + U) + np.abs(P) * aE + np.abs(E) * aP + HALF_TINY
            else:
                sig3 = self.terms[t]["sigma"] ** 3
                x1 = s2 * e[t]
                r1 = (d + 2) * U + rho[t] + U
                a1 = s2 * TINY + e[t] * 2 * d * HALF_TINY + HALF_TINY
                x2, r2, a2 = x1 / sig3, r1 + 3 * U, a1 / sig3 + HALF_TINY
                dK[h] = x2 * C
                bdK[h] = np.abs(dK[h]) * (r2 + (r + 1) * U) + a2 * C + HALF_TINY
        return K, bK * SAFETY, dK, bdK * SAFETY

    @staticmethod
    def _fold(shape, w, rw, e, rho, diag, w_eye, r_eye):
        """sum_t w_t e_t by the kernel's fma fold over every term, plus w_eye on the diagonal (TRAINING): value, bound."""
        T = len(e)
        S, b = np.zeros(shape, LD), np.zeros(shape, LD)
        for t in range(T):
            S += w[t] * e[t]
            b += w[t] * e[t] * (rho[t] + rw[t] * U) + w[t] * TINY
        b += T * (U * S + HALF_TINY)
        if diag is not None:
            b += np.where(diag, w_eye * r_eye * U + U * (S + w_eye) + HALF_TINY, 0)
            S = S + np.where(diag, w_eye, LD(0))
        return S, b


def bound_fraction(got, exact, bound):
    """The largest |got - exact| / bound over the elements (got: the GPU's fp64 values); inf where got is not finite.  A
    bound of 0 (an element no rounding reaches: K of a kernel without non-Eye terms) asks for the exact value."""
    got = np.asarray(got, dtype=np.float64)
    if not np.all(np.isfinite(got)):
        return float("inf")
    if got.size == 0:
        return 0.0
    err = np.abs(got.astype(LD) - exact)
    safe = np.where(bound > 0, bound, LD(1))
    return float(np.max(np.where(bound > 0, err / safe, np.where(err == 0, LD(0), LD(np.inf)))))
