// Shared device code of the two per-expert objective kernels (bcm_nll.cu, laplace.cu): one CTA of 256 threads per expert,
// everything in shared memory.
//
// The gradient of both objectives has the form  g_i = sum_ab dK_i[a,b] W_ab  with a symmetric pair weight W
//   regression     (GPR:63-66):    W = alpha alpha^T - K^-1                                   (out = -1/2 g)
//   classification (GPCls:121-126): W = 1/2 (a a^T - R) + 1/2 (u glp^T + glp u^T),  u = s2 - R K s2   (out = -g)
// and every derivative matrix the kernel DSL can produce is a combination of a few sums over the pairs, per non-Eye
// term t:
//   S_t = sum k_t W           Q_t = sum |x_a - x_b|^2 k_t W          D_tk = sum (x_ak - x_bk)^2 k_t W        trW
//   SCALE     (ScalarTimesKernel.scala:50-54,93-97): sum_t coef_t S_t + coef_eye trW
//   ARD_BETA  (ARDRBFKernel.scala:61-79)           : -2 beta_k scale_t D_tk
//   RBF_SIGMA (RBFKernel.scala:56-64)              : scale_t Q_t / sigma^3
// so ONE sweep over the lower triangle (off-diagonal pairs weighted 2) yields all hyper-parameters; ARD dimensions go
// through register accumulators DCH at a time (more sweeps only when d > DCH or several terms carry ARD betas).
#pragma once
#include "sgp_internal.h"

namespace sgp {

constexpr int EX_THREADS = 256;
constexpr int EX_WARPS = EX_THREADS / 32;
constexpr int DCH = 16;                                   // ARD dimensions per sweep
constexpr int EX_SUMS = 2 * kMaxTerms + 1 + DCH;          // doubles of shared memory the sweep needs

// host side (bcm_nll.cu): total[s][c] = sum_e per_expert[s][e][c] for each of n_slots slots, deterministic; a slot's sums
// do not depend on the other slots.  E: the slots' row stride and expert count; with sets (device, [n_slots]) and first
// (device, fold sets' first experts), slot s sums only the first[sets[s] + 1] - first[sets[s]] rows of its stride E.
cudaError_t launch_rows_reduce(double* dTotal, const double* dPerExpert, long long E, int width, cudaStream_t s,
                               int n_slots = 1, const int* sets = nullptr, const long long* first = nullptr);

template <int NW = EX_WARPS>
__device__ __forceinline__ double ex_block_sum(double v, double* red) {
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  const int w = threadIdx.x >> 5, l = threadIdx.x & 31;
  __syncthreads();
  if (l == 0) red[w] = v;
  __syncthreads();
  double s = 0.0;
  for (int i = 0; i < NW; ++i) s += red[i];
  return s;
}

// Stage the expert's rows in shared memory (odd row stride: rows a, a+1, ... fall into different banks).
__device__ __forceinline__ const double* ex_stage_rows(const double* Xg, int n, int d, int in_smem, double* Xs, int& xld) {
  if (!in_smem) { xld = d; return Xg; }
  xld = d | 1;
  for (int idx = threadIdx.x; idx < n * d; idx += EX_THREADS) Xs[(idx / d) * xld + idx % d] = Xg[idx];
  return Xs;
}

// K (lower triangle incl. diagonal, optionally mirrored): warp w owns rows a = w, w+8, ...; lanes own columns b <= a.
template <bool MIRROR>
__device__ __forceinline__ void ex_build_kernel(const HyperView& hv, const double* Xe, int xld, int n, double* K, int ld) {
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  for (int a = warp; a < n; a += EX_WARPS) {
    for (int b = lane; b <= a; b += 32) {
      double v = 0.0;
      for (int t = 0; t < hv.kf.n_terms; ++t) {
        const double* bt = hv.beta + t * hv.d;
        double q = 0.0;
        for (int k = 0; k < hv.d; ++k) {
          const double df = (Xe[a * xld + k] - Xe[b * xld + k]) * bt[k];
          q = fma(df, df, q);
        }
        v = hv.kf.fold_term(v, t, q);
      }
      if (a == b) v += hv.kf.eye_sum;
      K[a * ld + b] = v;
      if (MIRROR) K[b * ld + a] = v;
    }
  }
}

// In-place lower Cholesky (right-looking; the scaled column goes through `col`, the trailing update is row-per-warp).
// Returns sum(log diag L) (computed in parallel after the factorisation: the per-column critical path is one rsqrt);
// `bad` is set when a pivot is not positive.  `red`: 8 doubles.
__device__ __forceinline__ double ex_cholesky(double* M, int n, int ld, double* col, double* red, bool& bad) {
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  for (int j = 0; j < n; ++j) {
    const double djj = M[j * ld + j];
    if (!(djj > 0.0)) bad = true;
    const double inv = rsqrt(djj > 0.0 ? djj : 1.0);
    __syncthreads();
    if (tid == 0) M[j * ld + j] = (djj > 0.0 ? djj : 1.0) * inv;
    for (int i = j + 1 + tid; i < n; i += EX_THREADS) col[i] = M[i * ld + j] * inv;
    __syncthreads();
    for (int i = j + 1 + warp; i < n; i += EX_WARPS) {
      const double lij = col[i];
      for (int k = j + 1 + lane; k <= i; k += 32) M[i * ld + k] = fma(-lij, col[k], M[i * ld + k]);
      if (lane == 0) M[i * ld + j] = lij;
    }
    __syncthreads();
  }
  double part = 0.0;
  for (int j = tid; j < n; j += EX_THREADS) part += log(M[j * ld + j]);
  return ex_block_sum(part, red);
}

// L -> L^-1 in place, right-looking (Gauss-Jordan on the triangle): step k finalises row k and applies its rank-1
// update to the rows below -- (n-k-1) x (k+1) independent FMAs per step instead of one serial dot product per element.
__device__ __forceinline__ void ex_invert_lower(double* M, int n, int ld, double* rowbuf) {
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  for (int k = 0; k < n; ++k) {
    const double pinv = 1.0 / M[k * ld + k];
    __syncthreads();
    for (int j = tid; j <= k; j += EX_THREADS) {            // row k of the inverse: scale; keep a copy for the update
      const double v = (j == k) ? pinv : M[k * ld + j] * pinv;
      M[k * ld + j] = v;
      rowbuf[j] = v;
    }
    __syncthreads();
    for (int i = k + 1 + warp; i < n; i += EX_WARPS) {
      const double f = M[i * ld + k];
      for (int j = lane; j < k; j += 32) M[i * ld + j] = fma(-f, rowbuf[j], M[i * ld + j]);
      __syncwarp();                                           // every lane has read M[i][k] before lane 0 overwrites it
      if (lane == 0) M[i * ld + k] = -f * rowbuf[k];
    }
  }
  __syncthreads();
}

// L^-1 -> (L L^T)^-1 = L^-T L^-1 in place, lower triangle.  out[i][j] = sum_{k>=i} X[k][i] X[k][j] needs rows >= i of X
// only, so bands of EX_WARPS rows are processed top-down: every thread first accumulates its entries of the band in
// registers (independent chains), then the band is overwritten.  Two barriers per band instead of two per row.
constexpr int EX_LTL_MAXC = 6;      // columns per lane: n <= 192
__device__ __forceinline__ void ex_ltl_inplace(double* M, int n, int ld, double* /*rowbuf*/) {
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  for (int i0 = 0; i0 < n; i0 += EX_WARPS) {
    const int i = i0 + warp;
    double acc[EX_LTL_MAXC];
#pragma unroll
    for (int c = 0; c < EX_LTL_MAXC; ++c) acc[c] = 0.0;
    if (i < n) {
      for (int k = i; k < n; ++k) {
        const double xki = M[k * ld + i];
#pragma unroll
        for (int c = 0; c < EX_LTL_MAXC; ++c) {
          const int j = lane + 32 * c;
          if (j <= i) acc[c] = fma(xki, M[k * ld + j], acc[c]);
        }
      }
    }
    __syncthreads();
    if (i < n) {
#pragma unroll
      for (int c = 0; c < EX_LTL_MAXC; ++c) {
        const int j = lane + 32 * c;
        if (j <= i) M[i * ld + j] = acc[c];
      }
    }
    __syncthreads();
  }
}

// Tail of a gradient sweep: block-reduce the per-thread sums (fixed order: deterministic) and turn them into the
// hyper-parameters this sweep owns.  S, Q: per term (sweep 0 only); D: the DCH dimensions k0 .. k0+kn-1 of term ts.
template <int NW = EX_WARPS>
__device__ __forceinline__ void ex_gradient_emit(const HyperView& hv, int sw, int ts, int k0, int kn,
                                                 const double (&S)[kMaxTerms], const double (&Q)[kMaxTerms],
                                                 const double (&D)[DCH], double trW, double factor, double* out,
                                                 double* sums, double* red) {
  const int tid = threadIdx.x;
  double* sS = sums;                          // [kMaxTerms]
  double* sQ = sums + kMaxTerms;              // [kMaxTerms]
  double* sTr = sums + 2 * kMaxTerms;         // [1]
  double* sD = sTr + 1;                       // [DCH]  per-dimension sums of this sweep's (term, dimension chunk)
    if (sw == 0) {
#pragma unroll
    for (int t = 0; t < kMaxTerms; ++t) {
      if (t < hv.kf.n_terms) {
        const double s_ = ex_block_sum<NW>(S[t], red), q_ = ex_block_sum<NW>(Q[t], red);
        if (tid == 0) { sS[t] = s_; sQ[t] = q_; }
      }
    }
    const double v = ex_block_sum<NW>(trW, red);
    if (tid == 0) sTr[0] = v;
  }
#pragma unroll
  for (int k = 0; k < DCH; ++k) {
    if (k < kn) {
      const double v = ex_block_sum<NW>(D[k], red);
      if (tid == 0) sD[k] = v;
    }
  }
  __syncthreads();
  for (int i = tid; i < hv.n_hypers; i += EX_THREADS) {
    const int kind = hv.h_kind[i];
    double g = 0.0;
    bool mine = (sw == 0);
    if (kind == 0) {                                                 // trainable scalar above a sub-tree
      const double* cf = hv.h_coef + static_cast<size_t>(i) * (kMaxTerms + 1);
      g = cf[kMaxTerms] * sTr[0];
      for (int t = 0; t < hv.kf.n_terms; ++t) g = fma(cf[t], sS[t], g);
    } else if (kind == 1) {                                          // ARD beta_k
      const int t = hv.h_term[i], k = hv.h_dim[i];
      mine = (t == ts && k >= k0 && k < k0 + kn);
      if (mine) g = hv.kf.term_scale(t) * (-2.0 * hv.h_value[i]) * sD[k - k0];
    } else {                                                         // RBF sigma
      const int t = hv.h_term[i];
      const double sg = hv.h_value[i];
      g = hv.kf.term_scale(t) * sQ[t] / (sg * sg * sg);
    }
    if (mine) out[i] = factor * g;
  }
  __syncthreads();
}

// out[i] = factor * sum_ab dK_i[a,b] W_ab for every hyper-parameter;  wf(a, b), b <= a, returns the symmetric W_ab.
// sums: EX_SUMS doubles of shared memory; red: 8 doubles.  All threads of the CTA must call it.
template <class WF>
__device__ __forceinline__ void ex_descriptor_gradient(const HyperView& hv, const double* Xe, int xld, int n, WF wf,
                                                       double factor, double* out, double* sums, double* red) {
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int chunks = (hv.d + DCH - 1) / DCH;
  const int n_sweeps = hv.any_ard ? hv.kf.n_terms * chunks : 1;
  for (int sw = 0; sw < n_sweeps; ++sw) {
    const int ts = hv.any_ard ? sw / chunks : -1;
    const int k0 = hv.any_ard ? (sw % chunks) * DCH : 0;
    const int kn = hv.any_ard ? ((hv.d - k0 < DCH) ? (hv.d - k0) : DCH) : 0;
    double S[kMaxTerms], Q[kMaxTerms], D[DCH], trW = 0.0;
#pragma unroll
    for (int t = 0; t < kMaxTerms; ++t) { S[t] = 0.0; Q[t] = 0.0; }
#pragma unroll
    for (int k = 0; k < DCH; ++k) D[k] = 0.0;
    for (int a = warp; a < n; a += EX_WARPS) {
      for (int b = lane; b <= a; b += 32) {
        const double W = ((a == b) ? 1.0 : 2.0) * wf(a, b);
        if (a == b) trW += W;
        double kws = 0.0;
#pragma unroll
        for (int t = 0; t < kMaxTerms; ++t) {
          if (t < hv.kf.n_terms && (sw == 0 || t == ts)) {
            const double* bt = hv.beta + t * hv.d;
            double q = 0.0, s2 = 0.0;
            for (int k = 0; k < hv.d; ++k) {
              const double dx = Xe[a * xld + k] - Xe[b * xld + k];
              const double df = dx * bt[k];
              q = fma(df, df, q);
              s2 = fma(dx, dx, s2);
            }
            const double kw = exp(-q) * W;
            if (sw == 0) { S[t] += kw; Q[t] = fma(s2, kw, Q[t]); }
            if (t == ts) kws = kw;
          }
        }
#pragma unroll
        for (int k = 0; k < DCH; ++k) {
          if (k < kn) {
            const double dx = Xe[a * xld + k0 + k] - Xe[b * xld + k0 + k];
            D[k] = fma(dx * dx, kws, D[k]);
          }
        }
      }
    }
    ex_gradient_emit(hv, sw, ts, k0, kn, S, Q, D, trW, factor, out, sums, red);
  }
}

}  // namespace sgp