// Block prediction (commons/GaussianProcessCommons.scala:121-125), all fp64:
//   mean_t = k_t . v      var_t = selfKernel + k_t M k_t^T      k_t = k(x_t, Z)  (1 x m),  (v, M) the installed magic pair.
//
// Two kernels per window of points:
//   predict_elements_kernel  every kernel element k_tj in fp64 (direct form on centred, beta-scaled coordinates, CUDA
//                            cores), folded into the mean in a fixed order.  A mean-only call stops here: K never reaches
//                            memory.  A variance call also stores the window's K (rows x m_pad, fp64) -- once.
//   predict_var_kernel       the quadratic form on fp64 tensor cores over the packed upper triangle
//                            B = triu(M + M^T, 1) + diag(M):  k M k^T = sum_{i <= j} k_i B_ij k_j  for ANY M (the
//                            antisymmetric part of M adds nothing to a quadratic form).  A CTA owns point tile R and
//                            column tile C and accumulates W_RC = sum_{I <= C} K_RI B_IC (mma.sync m8n8k4 f64): n m^2
//                            flops instead of the 2 n m^2 of a full K M product.  The epilogue folds sum_c W_rc K_rc into
//                            one partial per (C, point); W never reaches memory.  predict_var_reduce_kernel adds the
//                            partials in column-tile order.  Its probability instantiation (sgp_predict_probability)
//                            goes on to the averaged probability of GPML eq. 3.25 on the point's (mean, var):
//                              p = (1/sqrt(pi)) sum_i w_i sigmoid(mean + sqrt(2 max(var, 0)) x_i)
//                            with the n-node Gauss-Hermite rule (x_i, w_i) of commons/util/Integrator.scala.
// No atomics, and every point's arithmetic is the same whatever window or CTA row it lands in: a point gets the same bits
// from the host and the device entry, from fp32 input and its fp64 upcast, in one call or split over several, and (the
// mean) with or without the variance.
#include "sgp_internal.h"

#include <cmath>

namespace sgp {
namespace {

// ---- element kernel -------------------------------------------------------------------------------------------------
constexpr int kElemCols = 128;        // active-set columns per tile (one per thread of a point group)
constexpr int kElemPts = 16;          // points per point group; two groups per CTA
constexpr int kElemCtaPts = 2 * kElemPts;
constexpr int kElemDC = 32;           // feature dims staged per chunk
constexpr int kElemZS = kElemDC + 1;  // staged z row stride (doubles): conflict-free column reads
constexpr int kElemThreads = 256;

struct ElemParams {
  const void* X;          // n x d row-major, fp32 or fp64
  int x_is_f32;
  long long n;            // points of the window
  long long rows_out;     // rows of K to write (>= n, padded rows get zeros)
  int d, dpad, m, m_pad;
  KernelFlat kf;
  const double* Zc;       // [n_terms][m_pad][dpad] (Z - c) * beta (zero padded)
  const double* beta;     // [kMaxTerms][dpad] beta, then [dpad] the centre c
  const double* v;        // m: magic vector
  double* K;              // rows_out x m_pad, or nullptr (mean only)
  double* mean;           // n
};

__global__ void __launch_bounds__(kElemThreads, 1) predict_elements_kernel(const ElemParams p) {
  __shared__ double zs[kElemCols * kElemZS];
  __shared__ __align__(16) double xs[kElemCtaPts * kElemDC];
  __shared__ double red[2][4][kElemPts];
  const int tid = threadIdx.x, col = tid & (kElemCols - 1), grp = tid >> 7;
  const int lane = tid & 31, wig = (tid >> 5) & 3;                // warp inside the point group
  const long long pt_cta = static_cast<long long>(blockIdx.x) * kElemCtaPts;
  const long long pt0 = pt_cta + grp * kElemPts;
  const double* centre = p.beta + kMaxTerms * p.dpad;

  double macc[kElemPts];
#pragma unroll
  for (int i = 0; i < kElemPts; ++i) macc[i] = 0.0;

  for (int ct = 0; ct < p.m_pad / kElemCols; ++ct) {
    double e[kElemPts];
#pragma unroll
    for (int i = 0; i < kElemPts; ++i) e[i] = 0.0;
    for (int t = 0; t < p.kf.n_terms; ++t) {
      double q[kElemPts];
#pragma unroll
      for (int i = 0; i < kElemPts; ++i) q[i] = 0.0;
      const double* bt = p.beta + t * p.dpad;
      for (int c0 = 0; c0 < p.dpad; c0 += kElemDC) {
        const int clen = (p.dpad - c0 < kElemDC) ? (p.dpad - c0) : kElemDC;   // a multiple of 4
        __syncthreads();                                                     // previous users of zs / xs are done
        const double* zsrc = p.Zc + (static_cast<size_t>(t) * p.m_pad + ct * kElemCols) * p.dpad + c0;
        for (int idx = tid; idx < kElemCols * clen; idx += kElemThreads) {
          const int cc = idx / clen, k = idx - cc * clen;
          zs[cc * kElemZS + k] = zsrc[static_cast<size_t>(cc) * p.dpad + k];
        }
        for (int idx = tid; idx < kElemCtaPts * clen; idx += kElemThreads) {
          const int pp = idx / clen, k = idx - pp * clen, dim = c0 + k;
          const long long pt = pt_cta + pp;
          double xv = 0.0;
          if (pt < p.n && dim < p.d) {
            const size_t off = static_cast<size_t>(pt) * p.d + dim;
            const double x = p.x_is_f32 ? static_cast<double>(static_cast<const float*>(p.X)[off])
                                        : static_cast<const double*>(p.X)[off];
            xv = (x - centre[dim]) * bt[dim];
          }
          xs[pp * kElemDC + k] = xv;
        }
        __syncthreads();
        const double* zc = zs + col * kElemZS;
        const double* xg = xs + grp * kElemPts * kElemDC;
        for (int k = 0; k < clen; k += 2) {
          const double z0 = zc[k], z1 = zc[k + 1];
#pragma unroll
          for (int pp = 0; pp < kElemPts; ++pp) {
            const double2 x = *reinterpret_cast<const double2*>(xg + pp * kElemDC + k);   // warp-wide broadcast
            const double d0 = x.x - z0, d1 = x.y - z1;
            q[pp] = fma(d0, d0, q[pp]);
            q[pp] = fma(d1, d1, q[pp]);
          }
        }
      }
#pragma unroll
      for (int pp = 0; pp < kElemPts; ++pp) e[pp] = p.kf.fold_term(e[pp], t, q[pp]);
    }
    const int j = ct * kElemCols + col;
    const bool zvalid = j < p.m;
    const double vj = zvalid ? p.v[j] : 0.0;
#pragma unroll
    for (int pp = 0; pp < kElemPts; ++pp) {
      const long long pt = pt0 + pp;
      const double ev = (zvalid && pt < p.n) ? e[pp] : 0.0;
      macc[pp] = fma(ev, vj, macc[pp]);
      if (p.K && pt < p.rows_out) p.K[static_cast<size_t>(pt) * p.m_pad + j] = ev;
    }
  }
  // sum over the 128 columns of the point group: a butterfly inside each warp (every lane ends with the same bits), then
  // the four warps in order
#pragma unroll
  for (int pp = 0; pp < kElemPts; ++pp) {
    double s = macc[pp];
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
    if (lane == 0) red[grp][wig][pp] = s;
  }
  __syncthreads();
  if (col < kElemPts && pt0 + col < p.n) {
    const double s = ((red[grp][0][col] + red[grp][1][col]) + red[grp][2][col]) + red[grp][3][col];
    p.mean[pt0 + col] = s;
  }
}

// ---- variance kernel ------------------------------------------------------------------------------------------------
constexpr int kVarRows = 128;         // points per CTA tile (R)
constexpr int kVarCols = 64;          // columns per CTA tile (C); also the edge of the triangular block schedule
constexpr int kVarK = 32;             // k extent of one staged chunk (two chunks per 64-wide block I)
constexpr int kVarKS = kVarK + 4;     // staged K row stride (doubles): conflict-free A fragments
constexpr int kVarBS = kVarCols + 4;  // staged B row stride (doubles): conflict-free B fragments
constexpr int kVarThreads = 256;      // 8 warps: 4 (rows) x 2 (columns), warp tile 32 x 32
constexpr int kVarGroup = 8;          // rasterisation: row tiles per group, column tiles innermost within a group
constexpr size_t kVarStageDoubles = static_cast<size_t>(kVarRows) * kVarKS + static_cast<size_t>(kVarK) * kVarBS;
constexpr size_t kVarSmem = 2 * kVarStageDoubles * sizeof(double);

__device__ __forceinline__ void dmma_m8n8k4(double (&c)[2], double a, double b) {
  asm volatile("mma.sync.aligned.m8n8k4.row.col.f64.f64.f64.f64 {%0,%1}, {%2}, {%3}, {%0,%1};\n"
               : "+d"(c[0]), "+d"(c[1])
               : "d"(a), "d"(b));
}
__device__ __forceinline__ void cp_async16(void* dst, const void* src) {
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(static_cast<uint32_t>(__cvta_generic_to_shared(dst))),
               "l"(src) : "memory");
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void cp_async_wait() { asm volatile("cp.async.wait_group %0;" ::"n"(N) : "memory"); }

// Tile of a linear block index: groups of kVarGroup row tiles; inside a group the column tiles run from the widest
// (C = n_ct - 1, the most work) down, the group's row tiles innermost, so that CTAs running together share B column
// strips and K row tiles in L2.
__device__ __forceinline__ void var_tile(int b, int n_rt, int n_ct, int* rt, int* ct) {
  const int g = b / (kVarGroup * n_ct);
  const int rows = min(kVarGroup, n_rt - g * kVarGroup);
  const int local = b - g * kVarGroup * n_ct;
  *ct = n_ct - 1 - local / rows;
  *rt = g * kVarGroup + local % rows;
}

// vpart[ct][r] = sum_{c in C} K[r][c] * sum_{i < 64 (ct + 1)} K[r][i] B[i][c]     (rows r of tile R)
__global__ void __launch_bounds__(kVarThreads, 2)
    predict_var_kernel(const double* __restrict__ K, const double* __restrict__ B, long long rows, int m_pad, int n_rt,
                       int n_ct, double* __restrict__ vpart) {
  extern __shared__ __align__(16) double vsm[];
  __shared__ double red[2][kVarRows];
  int rt, ct;
  var_tile(blockIdx.x, n_rt, n_ct, &rt, &ct);
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5, wr = warp >> 1, wc = warp & 1;
  const long long r0 = static_cast<long long>(rt) * kVarRows;
  const int c0 = ct * kVarCols;
  const int nk = (ct + 1) * (kVarCols / kVarK);                     // k chunks of blocks I = 0 .. C

  auto load = [&](int kc, int stage) {
    double* ks = vsm + stage * kVarStageDoubles;
    double* bs = ks + kVarRows * kVarKS;
    const int k0 = kc * kVarK;
#pragma unroll 1                                                   // rolled: 128 registers, two CTAs per SM
    for (int idx = tid; idx < kVarRows * kVarK / 2; idx += kVarThreads) {   // 16-byte pieces
      const int r = idx / (kVarK / 2), k2 = (idx % (kVarK / 2)) * 2;
      cp_async16(ks + r * kVarKS + k2, K + static_cast<size_t>(r0 + r) * m_pad + k0 + k2);
    }
#pragma unroll 1
    for (int idx = tid; idx < kVarK * kVarCols / 2; idx += kVarThreads) {
      const int k = idx / (kVarCols / 2), c2 = (idx % (kVarCols / 2)) * 2;
      cp_async16(bs + k * kVarBS + c2, B + static_cast<size_t>(k0 + k) * m_pad + c0 + c2);
    }
    cp_async_commit();
  };

  double acc[4][4][2];
#pragma unroll
  for (int i = 0; i < 4; ++i)
#pragma unroll
    for (int j = 0; j < 4; ++j) acc[i][j][0] = acc[i][j][1] = 0.0;

  load(0, 0);
  for (int kc = 0; kc < nk; ++kc) {
    if (kc + 1 < nk) {
      load(kc + 1, (kc + 1) & 1);
      cp_async_wait<1>();
    } else {
      cp_async_wait<0>();
    }
    __syncthreads();
    const double* ks = vsm + (kc & 1) * kVarStageDoubles;
    const double* bs = ks + kVarRows * kVarKS;
#pragma unroll
    for (int k4 = 0; k4 < kVarK; k4 += 4) {
      double a[4], b[4];
#pragma unroll
      for (int i = 0; i < 4; ++i) a[i] = ks[(wr * 32 + i * 8 + (lane >> 2)) * kVarKS + k4 + (lane & 3)];
#pragma unroll
      for (int j = 0; j < 4; ++j) b[j] = bs[(k4 + (lane & 3)) * kVarBS + wc * 32 + j * 8 + (lane >> 2)];
#pragma unroll
      for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j) dmma_m8n8k4(acc[i][j], a[i], b[j]);
    }
    __syncthreads();                                                 // the stage is refilled by the next iteration
  }
  // epilogue: sum_c W[r][c] K[r][c] for each row; the quad of lanes sharing a row, then the two column warps in order
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const int r = wr * 32 + i * 8 + (lane >> 2);
    const double* kr = K + static_cast<size_t>(r0 + r) * m_pad + c0 + wc * 32 + 2 * (lane & 3);
    double s = 0.0;
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const double2 kv = *reinterpret_cast<const double2*>(kr + j * 8);
      s = fma(acc[i][j][0], kv.x, s);
      s = fma(acc[i][j][1], kv.y, s);
    }
    s += __shfl_xor_sync(0xffffffffu, s, 1);
    s += __shfl_xor_sync(0xffffffffu, s, 2);
    if ((lane & 3) == 0) red[wc][r] = s;
  }
  __syncthreads();
  if (tid < kVarRows && r0 + tid < rows) vpart[static_cast<size_t>(ct) * rows + r0 + tid] = red[0][tid] + red[1][tid];
}

constexpr double kRsqrtPi = 0.56418958354775628695;   // 1 / sqrt(pi)

// var[r] = selfKernel + sum_ct vpart[ct][r], column tiles in order.
// kProb: then p[r] = (1/sqrt(pi)) sum_i w_i sigmoid(mean[r] + sqrt(2 v) x_i), nodes in rule order, with v = var[r]
// clamped at 0 from below (a negative variance is rounding, or a caller's magic pair; NaN stays NaN), sigmoid(z) =
// 1 / (1 + exp(-z)) as breeze defines it; var[r] is written only where var is given.
template <bool kProb>
__global__ void predict_var_reduce_kernel(const double* __restrict__ vpart, long long rows, int n_ct, double self_k,
                                          double* __restrict__ var, const double* __restrict__ mean,
                                          const double* __restrict__ rule, int n_nodes, double* __restrict__ prob) {
  const long long r = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x;
  if (r >= rows) return;
  double s = 0.0;
  for (int ct = 0; ct < n_ct; ++ct) s += vpart[static_cast<size_t>(ct) * rows + r];
  const double v = self_k + s;
  if (!kProb) {
    var[r] = v;
    return;
  }
  if (var) var[r] = v;
  const double mu = mean[r];
  const double sd2 = sqrt(2.0 * (v < 0.0 ? 0.0 : v));          // not fmax: fmax(NaN, 0) is 0
  const double* w = rule + n_nodes;
  double acc = 0.0;
  for (int i = 0; i < n_nodes; ++i) {
    // z = mu + sd2 x_i rounded twice, as written (not contracted to an fma): near z = 0 with a large |mu| one rounding
    // less would move sigmoid(z) by ~ulp(mu) / 4 against the same formula evaluated on the host
    const double z = __dadd_rn(mu, __dmul_rn(sd2, rule[i]));
    acc = fma(w[i], 1.0 / (1.0 + exp(-z)), acc);
  }
  prob[r] = acc * kRsqrtPi;
}

// B = triu(M + M^T, 1) + diag(M), zero padded to m_pad x m_pad
__global__ void pack_magic_kernel(double* __restrict__ B, const double* __restrict__ M, int m, int m_pad) {
  const int j = blockIdx.x * blockDim.x + threadIdx.x;
  const int i = blockIdx.y * blockDim.y + threadIdx.y;
  if (i >= m_pad || j >= m_pad) return;
  double v = 0.0;
  if (i < m && j < m) {
    if (i < j) v = M[static_cast<size_t>(i) * m + j] + M[static_cast<size_t>(j) * m + i];
    else if (i == j) v = M[static_cast<size_t>(i) * m + i];
  }
  B[static_cast<size_t>(i) * m_pad + j] = v;
}

}  // namespace

long long predict_window_points(int m_pad) {
  // K of one window: at most kPredictKBytes of fp64, whole CTA row tiles
  long long w = static_cast<long long>(kPredictKBytes / (static_cast<size_t>(m_pad) * sizeof(double)));
  w = w / kVarRows * kVarRows;
  return w < kVarRows ? kVarRows : w;
}

// K (rows x m_pad), the column-tile partials (n_ct x window), then the mean of a probability call that returns none
size_t predict_ws_bytes(long long window, int m_pad) {
  const long long rows = (window + kVarRows - 1) / kVarRows * kVarRows;
  const int n_ct = m_pad / kVarCols;
  return (static_cast<size_t>(rows) * m_pad + static_cast<size_t>(n_ct + 1) * window) * sizeof(double);
}

// Newton's method on the orthonormal Hermite recurrence
//   p_0 = pi^(-1/4),  p_j = x sqrt(2/j) p_{j-1} - sqrt((j-1)/j) p_{j-2},  p_n' = sqrt(2n) p_{n-1},
// whose roots are the nodes and whose weights are w = 2 / p_n'(x)^2.  The roots are found from the largest down.  Starting
// guesses: the first four from the Airy asymptotics of the largest zeros, x_k ~ sqrt(2n+1) - a_k 2^(-1/3) (2n+1)^(-1/6)
// (a_k the k-th zero of Ai, negated), the others one WKB half-wavelength pi / sqrt(2n+1 - x^2) below the last root.  The
// roots already found are divided out of the Newton step (Maehly), so that no guess falls back onto a larger root.  Only
// the non-negative half is computed and mirrored: the rule is exactly symmetric, the middle root of an odd rule exactly 0.
// Against numpy's hermgauss for n = 1 .. 256: nodes within 4e-15, weights within 4e-13 relative.
constexpr double kAiryZeros[4] = {2.338107410459767, 4.087949444130971, 5.520559828095551, 6.786708090071759};

bool gauss_hermite_rule(int n, double* nodes, double* weights) {
  if (n < 1 || n > kMaxHermiteNodes || !nodes || !weights) return false;
  const double p0 = 1.0 / std::sqrt(std::sqrt(std::acos(-1.0)));
  // (p_n(x), p_n'(x)) by the recurrence
  auto eval = [&](double x, double* pn) {
    double p = p0, q = 0.0;                                   // p_j, p_{j-1}
    for (int j = 1; j <= n; ++j) {
      const double r = x * std::sqrt(2.0 / j) * p - std::sqrt((j - 1.0) / j) * q;
      q = p;
      p = r;
    }
    *pn = p;
    return std::sqrt(2.0 * n) * q;
  };
  const int half = (n + 1) / 2;
  std::vector<double> z(half);
  for (int i = 0; i < half; ++i) {
    double x;
    if (n % 2 == 1 && i == half - 1) {
      x = 0.0;
    } else {
      if (i < 4) {
        x = std::sqrt(2.0 * n + 1.0) - kAiryZeros[i] * std::cbrt(0.5) * std::pow(2.0 * n + 1.0, -1.0 / 6.0);
      } else {                                                // one local half-wavelength below the last root
        const double h = std::acos(-1.0) / std::sqrt(2.0 * n + 1.0 - z[i - 1] * z[i - 1]);
        const double xm = z[i - 1] - 0.5 * h;
        x = z[i - 1] - std::acos(-1.0) / std::sqrt(2.0 * n + 1.0 - xm * xm);
      }
      for (int it = 0; it < 100; ++it) {
        double pn;
        const double dp = eval(x, &pn);
        double s = 0.0;                                       // Maehly: Newton on p_n / prod_{k < i} (x - z_k)
        for (int k = 0; k < i; ++k) s += 1.0 / (x - z[k]);
        const double dx = pn / (dp - pn * s);
        x -= dx;
        if (std::fabs(dx) <= 1e-15 * std::fabs(x)) break;
      }
    }
    z[i] = x;
    double pn;
    const double dp = eval(x, &pn);
    const double w = 2.0 / (dp * dp);
    nodes[i] = -x;
    nodes[n - 1 - i] = x;                                     // the middle root of an odd rule stays +0
    weights[i] = weights[n - 1 - i] = w;
  }
  return true;
}

cudaError_t launch_pack_magic(double* B, const double* M, int m, int m_pad, cudaStream_t s) {
  dim3 block(32, 8), grid((m_pad + 31) / 32, (m_pad + 7) / 8);
  pack_magic_kernel<<<grid, block, 0, s>>>(B, M, m, m_pad);
  return cudaGetLastError();
}

cudaError_t launch_predict(const PredictArgs& a, cudaStream_t s) {
  if (a.n <= 0) return cudaSuccess;
  const bool with_var = a.var || a.prob;
  const long long rows = (a.n + kVarRows - 1) / kVarRows * kVarRows;   // K rows: whole variance row tiles
  const int n_ct = (a.m + kVarCols - 1) / kVarCols;                  // trailing all-padding column tiles are skipped
  double* K = with_var ? a.ws : nullptr;                              // a mean-only call has no workspace
  double* vpart = with_var ? a.ws + static_cast<size_t>(rows) * a.m_pad : nullptr;
  double* mean = a.mean ? a.mean : vpart + static_cast<size_t>(n_ct) * a.n;   // a probability call without a mean
  ElemParams p{};
  p.X = a.X; p.x_is_f32 = a.x_is_f32; p.n = a.n; p.rows_out = rows;
  p.d = a.d; p.dpad = a.dpad; p.m = a.m; p.m_pad = a.m_pad; p.kf = a.kf;
  p.Zc = a.Zc; p.beta = a.beta; p.v = a.v; p.K = K; p.mean = mean;
  const long long cta_rows = with_var ? rows : a.n;
  predict_elements_kernel<<<static_cast<unsigned>((cta_rows + kElemCtaPts - 1) / kElemCtaPts), kElemThreads, 0, s>>>(p);
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess || !with_var) return e;
  const int n_rt = static_cast<int>(rows / kVarRows);
  // the cap is per device and shared by every context on it: set on every launch (allow_dynamic_smem), it is cheap
  e = allow_dynamic_smem(reinterpret_cast<const void*>(predict_var_kernel));
  if (e != cudaSuccess) return e;
  predict_var_kernel<<<static_cast<unsigned>(n_rt) * n_ct, kVarThreads, kVarSmem, s>>>(K, a.B, a.n, a.m_pad, n_rt, n_ct,
                                                                                     vpart);
  if ((e = cudaGetLastError()) != cudaSuccess) return e;
  const unsigned reduce_grid = static_cast<unsigned>((a.n + 255) / 256);
  if (a.prob)
    predict_var_reduce_kernel<true><<<reduce_grid, 256, 0, s>>>(vpart, a.n, n_ct, a.kf.self_kernel, a.var, mean, a.rule,
                                                               a.n_nodes, a.prob);
  else
    predict_var_reduce_kernel<false><<<reduce_grid, 256, 0, s>>>(vpart, a.n, n_ct, a.kf.self_kernel, a.var, nullptr,
                                                                nullptr, 0, nullptr);
  return cudaGetLastError();
}

}  // namespace sgp
