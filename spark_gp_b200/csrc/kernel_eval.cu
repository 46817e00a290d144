// Kernel evaluation (sgp_kernel_eval, sgp_kernel_eval_device): K[i][j] = k(a_i, b_j) of the flattened kernel and,
// optionally, every dK / d theta_h -- the crossKernel / trainingKernel / trainingKernelAndDerivative methods of
// kernel/Kernel.scala:12-98.  The output is (1 + h) n m doubles, so the kernel is built around coalesced fp64 stores.
//
// A CTA of kEvalTy x 32 threads owns a tile of kEvalRows rows of A by kEvalCols columns (rows of B); a thread holds
// kEvalRows / kEvalTy rows by kEvalCols / 32 columns, its columns 32 apart so that a warp's stores cover 32 consecutive
// doubles of a row.  Per term, the rows of A and B are staged in shared memory in chunks of kEvalChunk dimensions (any d).
//
// Element arithmetic (the same in every tile and launch window):
//   CROSS:    df_k = fma(a_k, beta_k, -(b_k * beta_k)), the form of sgp_cross_kernel's cross_kernel_kernel (which the
//             compiler contracts to exactly this fma over the beta-scaled active set), so both give the same bits.
//   TRAINING: df_k = (a_k * beta_k) - (b_k * beta_k): the (j, i) element negates every df_k, so K and each dK are exactly
//             symmetric.  It runs the same fma with a weight of 1 on pre-scaled rows of A.
//   q_t = sum_k df_k^2 by fma in dimension order; K = fold of C_t exp(-q_t) over the terms (KernelFlat::fold_term), plus
//   the Eye sum on the training diagonal.
// Derivatives (kDeriv), from the raw difference d_k = a_k - b_k (beta_k = 0 happens, so not from df_k / beta_k):
//   ARD beta_k of term t:  (-2 beta_k d_k^2) (C_t e_t)      ARDRBFKernel.scala:61-79
//   RBF sigma of term t:   (|a - b|^2 e_t / sigma^3) C_t     RBFKernel.scala:56-64
//   trainable scalar:      sum_t coef_t e_t, plus the Eye coefficient on the training diagonal  ScalarTimesKernel.scala:93-97
// where e_t = exp(-q_t) stays in registers and d_k is recomputed in a second pass over the dimensions.
#include "sgp_internal.h"

namespace sgp {
namespace {

constexpr int kEvalRows = 32, kEvalCols = 64, kEvalChunk = 32, kEvalTy = 8;
constexpr int kEvalRi = kEvalRows / kEvalTy, kEvalCj = kEvalCols / 32;

__device__ __forceinline__ double load_row_value(const void* p, int is_f32, size_t i) {
  return is_f32 ? static_cast<double>(static_cast<const float*>(p)[i]) : static_cast<const double*>(p)[i];
}

struct EvalSmem {
  double a[kEvalRows][kEvalChunk];
  double b[kEvalChunk][kEvalCols + 1];   // padded: the staging writes run down a column
  double w[kEvalChunk];
  double beta[kMaxTerms][kEvalChunk];     // derivative pass: beta_tk
  int h[kMaxTerms][kEvalChunk];           // derivative pass: hyper-parameter index of ARD (t, k), -1 for none
};

// Stages dims [k0, k0 + kc) of the tile's rows of A and B: raw values, or each scaled by `scale` (nullptr: raw) where
// scale_a / scale_b says so.  Rows and dims outside the matrices read 0.
__device__ __forceinline__ void stage_chunk(EvalSmem& s, const KernelEvalArgs& a, long long r0, int col0, int k0, int kc,
                                            const double* scale, bool scale_a, bool scale_b) {
  const int tid = threadIdx.y * 32 + threadIdx.x;
  for (int idx = tid; idx < kEvalRows * kEvalChunk; idx += kEvalTy * 32) {
    const int r = idx / kEvalChunk, k = idx % kEvalChunk;
    const long long gr = r0 + r;
    double v = 0.0;
    if (k < kc && gr < a.n) {
      v = load_row_value(a.A, a.a_is_f32, static_cast<size_t>(gr) * a.d + k0 + k);
      if (scale_a) v = __dmul_rn(v, scale[k0 + k]);
    }
    s.a[r][k] = v;
  }
  for (int idx = tid; idx < kEvalCols * kEvalChunk; idx += kEvalTy * 32) {
    const int c = idx / kEvalChunk, k = idx % kEvalChunk;
    const int gc = col0 + c;
    double v = 0.0;
    if (k < kc && gc < a.m) {
      v = load_row_value(a.B, a.b_is_f32, static_cast<size_t>(gc) * a.d + k0 + k);
      if (scale_b) v = __dmul_rn(v, scale[k0 + k]);
    }
    s.b[k][c] = v;
  }
}

template <bool kDeriv>
__global__ void __launch_bounds__(kEvalTy * 32) kernel_eval_kernel(const KernelEvalArgs a) {
  __shared__ EvalSmem s;
  const int tx = threadIdx.x, ty = threadIdx.y, tid = ty * 32 + tx;
  const int col0 = blockIdx.x * kEvalCols;
  const long long row_tiles = (a.n + kEvalRows - 1) / kEvalRows;
  const KernelFlat& kf = a.kf;
  for (long long rt = blockIdx.y; rt < row_tiles; rt += gridDim.y) {
    const long long r0 = rt * kEvalRows;
    double K[kEvalRi][kEvalCj];
    double e[kDeriv ? kMaxTerms : 1][kEvalRi][kEvalCj];
#pragma unroll
    for (int i = 0; i < kEvalRi; ++i)
#pragma unroll
      for (int j = 0; j < kEvalCj; ++j) K[i][j] = 0.0;
#pragma unroll
    for (int t = 0; t < kMaxTerms; ++t) {
      if (t >= kf.n_terms) break;
      const double* bt = a.beta + static_cast<size_t>(t) * a.d;
      double q[kEvalRi][kEvalCj];
#pragma unroll
      for (int i = 0; i < kEvalRi; ++i)
#pragma unroll
        for (int j = 0; j < kEvalCj; ++j) q[i][j] = 0.0;
      for (int k0 = 0; k0 < a.d; k0 += kEvalChunk) {
        const int kc = min(kEvalChunk, a.d - k0);
        __syncthreads();
        stage_chunk(s, a, r0, col0, k0, kc, bt, a.training != 0, true);
        if (tid < kEvalChunk) s.w[tid] = a.training ? 1.0 : (tid < kc ? bt[k0 + tid] : 0.0);
        __syncthreads();
        for (int kk = 0; kk < kc; ++kk) {
          const double w = s.w[kk];
          double bv[kEvalCj];
#pragma unroll
          for (int j = 0; j < kEvalCj; ++j) bv[j] = s.b[kk][tx + 32 * j];
#pragma unroll
          for (int i = 0; i < kEvalRi; ++i) {
            const double av = s.a[ty + kEvalTy * i][kk];
#pragma unroll
            for (int j = 0; j < kEvalCj; ++j) {
              const double df = fma(av, w, -bv[j]);
              q[i][j] = fma(df, df, q[i][j]);
            }
          }
        }
      }
#pragma unroll
      for (int i = 0; i < kEvalRi; ++i)
#pragma unroll
        for (int j = 0; j < kEvalCj; ++j) {
          if constexpr (kDeriv) e[t][i][j] = exp(-q[i][j]);
          K[i][j] = kf.fold_term(K[i][j], t, q[i][j]);
        }
    }
    // element (i, j) of this thread: row r0 + ty + kEvalTy i, column col0 + tx + 32 j
    auto store = [&](double* out, int i, int j, double v) {
      const long long gr = r0 + ty + kEvalTy * i;
      const int gc = col0 + tx + 32 * j;
      if (gr < a.n && gc < a.m) out[static_cast<size_t>(gr) * a.m + gc] = v;
    };
    auto on_diag = [&](int i, int j) { return a.training && a.row0 + r0 + ty + kEvalTy * i == col0 + tx + 32 * j; };
#pragma unroll
    for (int i = 0; i < kEvalRi; ++i)
#pragma unroll
      for (int j = 0; j < kEvalCj; ++j) store(a.K, i, j, on_diag(i, j) ? K[i][j] + kf.eye_sum : K[i][j]);
    if constexpr (kDeriv) {
      double s2[kEvalRi][kEvalCj];   // |a - b|^2, in dimension order
#pragma unroll
      for (int i = 0; i < kEvalRi; ++i)
#pragma unroll
        for (int j = 0; j < kEvalCj; ++j) s2[i][j] = 0.0;
      for (int k0 = 0; k0 < a.d && kf.n_terms > 0; k0 += kEvalChunk) {
        const int kc = min(kEvalChunk, a.d - k0);
        __syncthreads();
        stage_chunk(s, a, r0, col0, k0, kc, nullptr, false, false);
        for (int idx = tid; idx < kMaxTerms * kEvalChunk; idx += kEvalTy * 32) {
          const int t = idx / kEvalChunk, k = idx % kEvalChunk;
          const bool in = t < kf.n_terms && k < kc;
          s.h[t][k] = in ? a.ard_h[static_cast<size_t>(t) * a.d + k0 + k] : -1;
          s.beta[t][k] = in ? a.beta[static_cast<size_t>(t) * a.d + k0 + k] : 0.0;
        }
        __syncthreads();
        for (int kk = 0; kk < kc; ++kk) {
          double dsq[kEvalRi][kEvalCj];
#pragma unroll
          for (int i = 0; i < kEvalRi; ++i)
#pragma unroll
            for (int j = 0; j < kEvalCj; ++j) {
              const double df = s.a[ty + kEvalTy * i][kk] - s.b[kk][tx + 32 * j];
              dsq[i][j] = __dmul_rn(df, df);
              s2[i][j] = __dadd_rn(s2[i][j], dsq[i][j]);
            }
#pragma unroll
          for (int t = 0; t < kMaxTerms; ++t) {
            if (t >= kf.n_terms) break;
            const int h = s.h[t][kk];
            if (h < 0) continue;
            const double c2 = -2.0 * s.beta[t][kk], ct = kf.term_scale(t);
            double* out = a.dK + static_cast<size_t>(h) * a.dk_stride;
#pragma unroll
            for (int i = 0; i < kEvalRi; ++i)
#pragma unroll
              for (int j = 0; j < kEvalCj; ++j) store(out, i, j, (c2 * dsq[i][j]) * (ct * e[t][i][j]));
          }
        }
      }
#pragma unroll
      for (int t = 0; t < kMaxTerms; ++t) {
        if (t >= kf.n_terms) break;
        const int h = a.rbf_h[t];
        if (h < 0) continue;
        double* out = a.dK + static_cast<size_t>(h) * a.dk_stride;
#pragma unroll
        for (int i = 0; i < kEvalRi; ++i)
#pragma unroll
          for (int j = 0; j < kEvalCj; ++j) store(out, i, j, (s2[i][j] * e[t][i][j] / a.sigma3[t]) * kf.term_scale(t));
      }
      for (int sh = 0; sh < a.n_scale; ++sh) {
        const double* cf = a.scale_coef + static_cast<size_t>(sh) * (kMaxTerms + 1);
        double* out = a.dK + static_cast<size_t>(a.scale_h[sh]) * a.dk_stride;
#pragma unroll
        for (int i = 0; i < kEvalRi; ++i)
#pragma unroll
          for (int j = 0; j < kEvalCj; ++j) {
            double v = 0.0;
#pragma unroll
            for (int t = 0; t < kMaxTerms; ++t)
              if (t < kf.n_terms) v = fma(cf[t], e[t][i][j], v);
            store(out, i, j, on_diag(i, j) ? v + cf[kMaxTerms] : v);
          }
      }
    }
  }
}

}  // namespace

cudaError_t launch_kernel_eval(const KernelEvalArgs& a, cudaStream_t s) {
  const long long row_tiles = (a.n + kEvalRows - 1) / kEvalRows;
  const dim3 block(32, kEvalTy);
  const dim3 grid(static_cast<unsigned>((a.m + kEvalCols - 1) / kEvalCols),
                  static_cast<unsigned>(row_tiles < 65535 ? row_tiles : 65535));
  if (a.dK)
    kernel_eval_kernel<true><<<grid, block, 0, s>>>(a);
  else
    kernel_eval_kernel<false><<<grid, block, 0, s>>>(a);
  return cudaGetLastError();
}

}  // namespace sgp
