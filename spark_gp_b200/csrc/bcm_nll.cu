// Batched per-expert BCM objective: negative log marginal likelihood + gradient (fp64), one CTA per expert.
//
// Replaces, for all experts of a rank at once, the body of the hyper-parameter objective
//   regression/GaussianProcessRegression.scala:55-68   likelihoodAndGradient
//   commons/util/logDetAndInv.scala:36-63              (LU-based log|det| and inverse)
//   kernel/*.scala  trainingKernelAndDerivative        (ARDRBFKernel.scala:61-79, RBFKernel.scala:56-64,
//                                                       ScalarTimesKernel.scala:50-54,93-97, SumOfKernels.scala:50-55)
// summed over experts like the treeAggregate of commons/GaussianProcessCommons.scala:73-78.
//
//   K   = sum_t scale_t k_t(X_e, X_e) + eye_sum I                      (n_e x n_e, n_e ~ 100)
//   nll = 1/2 y^T K^-1 y + 1/2 log|det K|      (no n/2 log 2pi term -- GPR:61)
//   g_i = -1/2 sum_ab dK_i[a,b] (alpha_a alpha_b - K^-1[a,b]),   alpha = K^-1 y          (GPR:63-66)
//
// The reference factors K with LU; K is symmetric positive definite here (the sigma2 Eye term is always present,
// GPC:18), so Cholesky gives the same log-determinant and inverse (up to rounding) at a third of the work.  A
// non-positive pivot is reported (the reference would return a negative-determinant "logdet" of |det| instead).
//
// Slots (ObjectiveSlots): a second grid dimension runs several expert sets of the upload in one launch (sgp_bcm_nll is
// one slot on the whole upload).  Block (x, s) evaluates expert x of the set listed in slot s with slot s's flattened
// kernel and hyper-parameter block, output row [s][x]; the arithmetic does not depend on the slot.
#include <cstdlib>
#include <string>

#include "expert_common.cuh"

namespace sgp {
namespace {

struct NllParams {
  const double* X;          // packed expert-major: expert e owns rows off[e] .. off[e+1]-1 (row-major, d columns)
  const double* y;
  const long long* off;     // [E+1]
  int n_max;                // largest expert
  int x_in_smem;            // the expert's rows are staged in shared memory
  HyperView hv;             // slot 0's view; fold slot s reads kf[s] and the descriptor values s * slot_stride doubles on
  const int* sets;          // [n_slots] fold set of each slot, or nullptr: one slot over every expert
  const long long* first;   // [n_sets + 1] first expert of each fold set (with sets)
  const KernelFlat* kf;     // [n_slots] (with sets)
  long long slot_stride;    // (with sets)
  double* out;              // [n_slots][gridDim.x][1 + n_hypers]   per-expert (nll, gradient)
  int* flags;               // [n_slots]  bit 0: a pivot was not positive
};

// Block (x, s): expert x of slot s's fold set, at slot s's kernel and hyper-parameters (one slot: expert x at p.hv).
// False when the set has no expert x; the block then returns before its first barrier.
__device__ __forceinline__ bool nll_block(const NllParams& p, HyperView& hv, long long& e, double*& out) {
  const int slot = blockIdx.y;
  e = blockIdx.x;
  if (p.sets) {
    const int k = p.sets[slot];
    const long long first = p.first[k];
    if (e >= p.first[k + 1] - first) return false;
    e += first;
    hv.kf = p.kf[slot];
    hv.beta += slot * p.slot_stride; hv.h_coef += slot * p.slot_stride; hv.h_value += slot * p.slot_stride;
  }
  out = p.out + (static_cast<size_t>(slot) * gridDim.x + blockIdx.x) * (1 + hv.n_hypers);
  return true;
}

__global__ void __launch_bounds__(EX_THREADS, 2) bcm_nll_kernel(const NllParams p) {
  extern __shared__ double sm[];
  HyperView hv = p.hv;
  long long e;
  double* out;
  if (!nll_block(p, hv, e, out)) return;
  const long long r0 = p.off[e];
  const int n = static_cast<int>(p.off[e + 1] - r0);
  const int ld = p.n_max + 1;                 // padded leading dimension
  double* K = sm;                             // [n_max][ld]   K -> L -> L^-1 -> K^-1 (lower triangle)
  double* yv = K + static_cast<size_t>(p.n_max) * ld;      // [n_max]
  double* alpha = yv + p.n_max;               // [n_max]
  double* rowbuf = alpha + p.n_max;           // [n_max]
  double* red = rowbuf + p.n_max;             // [8]
  double* sums = red + 8;                     // [EX_SUMS]
  double* Xs = sums + EX_SUMS;                // [n_max][d|1] staged copy of the expert's rows (if it fits)
  const int tid = threadIdx.x;
  int xld;
  const double* Xe = ex_stage_rows(p.X + static_cast<size_t>(r0) * hv.d, n, hv.d, p.x_in_smem, Xs, xld);
  for (int i = tid; i < n; i += EX_THREADS) yv[i] = p.y[r0 + i];
  __syncthreads();
  ex_build_kernel<false>(hv, Xe, xld, n, K, ld);
  __syncthreads();
  bool bad = false;
  const double logdet = 2.0 * ex_cholesky(K, n, ld, rowbuf, red, bad);
  if (bad && tid == 0) atomicOr(p.flags + blockIdx.y, 1);
  ex_invert_lower(K, n, ld, rowbuf);
  ex_ltl_inplace(K, n, ld, rowbuf);           // K now holds K^-1 (lower)
  // ---- alpha = K^-1 y ;  nll ----------------------------------------------------------------------------------------
  for (int a = tid; a < n; a += EX_THREADS) {
    double s = 0.0;
    for (int b = 0; b < n; ++b) s = fma((b <= a) ? K[a * ld + b] : K[b * ld + a], yv[b], s);
    alpha[a] = s;
  }
  __syncthreads();
  double part = 0.0;
  for (int a = tid; a < n; a += EX_THREADS) part += yv[a] * alpha[a];
  const double yay = ex_block_sum(part, red);
  if (tid == 0) out[0] = 0.5 * yay + 0.5 * logdet;
  // ---- gradient: -1/2 sum_ab dK_i[a,b] (alpha_a alpha_b - K^-1[a,b])   (GPR:63-66) -----------------------------------
  ex_descriptor_gradient(hv, Xe, xld, n, [&](int a, int b) { return alpha[a] * alpha[b] - K[a * ld + b]; }, -0.5,
                         out + 1, sums, red);
}

// ---------------------------------------------------------------------------------------------------------------------
// Register-resident variant (one non-Eye term, experts of <= 128 points: every default configuration).
// The shared-memory kernel above spends its time in ~600 block barriers and latency-bound shared-memory updates
// (Cholesky, triangular inverse, L^-T L^-1: 10.3 ms per evaluation of 10^4 experts of 100 points, ~5 % of the fp64 rate).
// Here the matrix lives in REGISTERS: 512 threads form a 32 x 16 grid, thread (ty, tx) owns the entries
// (ty + 32 r, tx + 16 c) (cyclic: the work stays balanced while pivots move through the matrix; 16 warps hide the fp64
// and barrier latencies -- a 16 x 16 grid of 256 threads ran at 36 % issue utilisation, 5.1 ms), and K^-1 and
// log|det K| come from n SWEEPS (Goodnight's sweep operator = Gauss-Jordan on the symmetric matrix, no pivoting needed
// for an SPD matrix): sweep k broadcasts column k through shared memory (ONE barrier) and every thread applies the
// rank-1 update to its RB x RB block from registers; the pivots are the Schur complements (> 0 iff K is positive
// definite, their logs sum to log|det K|), and after n sweeps the registers hold -K^-1.
// The gradient needs no second exp(): the unscaled kernel values k_ab are parked in shared memory by the build, and with
// M = k o W (W = alpha alpha^T - K^-1) the per-dimension sums D_k = sum_ab (x_ak - x_bk)^2 M_ab are evaluated from
// registers, term by term from the pair differences like the shared-memory sweep does.  (The expanded form
// 2 (sum_a x_ak^2 m_a - x_k^T M x_k) is cheaper but cancels: its rounding error grows with |x_k|^2 / (x_ak - x_bk)^2, and
// on data spread over ~3 length scales it already exceeds the rounding bound of the pair sums.)
// ---------------------------------------------------------------------------------------------------------------------
constexpr int REG_GY = 32, REG_THREADS = REG_GY * 16, REG_WARPS = REG_THREADS / 32;   // 32 x 16 thread grid
template <int RBR, int RBC>      // rows / columns per thread: thread (ty, tx) owns entries (ty + 32 r, tx + 16 c)
__global__ void __launch_bounds__(REG_THREADS, 1) bcm_nll_reg_kernel(const NllParams p) {
  static_assert(RBC == 2 * RBR || RBC == 2 * RBR - 1, "the column extent covers the row extent");
  constexpr int NP = 16 * RBC;                // padded order of the matrix (rows beyond NP are never touched)
  constexpr int NR = 32 * RBR;                // >= NP
  extern __shared__ double sm[];
  HyperView hv = p.hv;
  long long e;
  double* out;
  if (!nll_block(p, hv, e, out)) return;
  const long long r0 = p.off[e];
  const int n = static_cast<int>(p.off[e + 1] - r0);
  const int d = hv.d, xld = d | 1;
  double* ys = sm;                            // [NR]
  double* alpha = ys + NR;                    // [NR]
  double* colbuf = alpha + NR;                // [2][NR]  column of the current sweep (double buffered by sweep parity)
  double* piv = colbuf + 2 * NR;              // [NR]     pivots
  double* red = piv + NR;                     // [16]
  double* sums = red + 16;                    // [EX_SUMS]
  double* Xs = sums + EX_SUMS;                // [NR][xld]  rows of the expert, minus its first row; zero padded
  double* Ks = Xs + static_cast<size_t>(NR) * xld;   // [NR][NP]  exponents, then unscaled kernel values (0 on padding)
  const int tid = threadIdx.x, tx = tid & 15, ty = tid >> 4;
  {
    const double* Xg = p.X + static_cast<size_t>(r0) * d;
    for (int idx = tid; idx < NR * d; idx += REG_THREADS) {
      const int i = idx / d, k = idx % d;
      Xs[i * xld + k] = (i < n) ? Xg[idx] - Xg[k] : 0.0;
    }
    for (int i = tid; i < NR; i += REG_THREADS) ys[i] = (i < n) ? p.y[r0 + i] : 0.0;
  }
  __syncthreads();
  // ---- build: A = scale exp(-sum_k ((x_ak - x_bk) beta_k)^2) + eye_sum I; identity on the padding -----------------------
  double A[RBR][RBC];
#pragma unroll
  for (int r = 0; r < RBR; ++r)
#pragma unroll
    for (int c = 0; c < RBC; ++c) A[r][c] = 0.0;
  for (int k = 0; k < d; ++k) {
    const double bk = hv.beta[k];
    double xa[RBR], xb[RBC];
#pragma unroll
    for (int r = 0; r < RBR; ++r) xa[r] = Xs[(ty + 32 * r) * xld + k] * bk;
#pragma unroll
    for (int c = 0; c < RBC; ++c) xb[c] = Xs[(tx + 16 * c) * xld + k] * bk;
#pragma unroll
    for (int r = 0; r < RBR; ++r)
#pragma unroll
      for (int c = 0; c < RBC; ++c) {
        const double df = xa[r] - xb[c];
        A[r][c] = fma(df, df, A[r][c]);
      }
  }
  // exp() through shared memory in a rolled loop: 28-56 inlined fp64 exp() are ~30 KB of straight-line code per thread
#pragma unroll
  for (int r = 0; r < RBR; ++r)
#pragma unroll
    for (int c = 0; c < RBC; ++c) Ks[(ty + 32 * r) * NP + tx + 16 * c] = A[r][c];
  __syncwarp();                               // a thread reads back only its own entries
#pragma unroll 1
  for (int rc = 0; rc < RBR * RBC; ++rc) {
    const int r = rc / RBC, c = rc % RBC;
    const int a = ty + 32 * r, b = tx + 16 * c;
    double* kp = Ks + a * NP + b;
    *kp = (a < n && b < n) ? exp(-*kp) : 0.0;
  }
  const double scale0 = hv.kf.term_scale(0);
#pragma unroll
  for (int r = 0; r < RBR; ++r)
#pragma unroll
    for (int c = 0; c < RBC; ++c) {
      const int a = ty + 32 * r, b = tx + 16 * c;
      const bool real = a < n && b < n;
      A[r][c] = real ? fma(scale0, Ks[a * NP + b], (a == b) ? hv.kf.eye_sum : 0.0) : ((a == b) ? 1.0 : 0.0);
    }
  // ---- n sweeps: A -> -K^-1.  Pivot k = 16 ck + kx sits in row block rk = ck / 2 (ty == 16 (ck % 2) + kx) ------------------
  bool bad = false;
#pragma unroll
  for (int ck = 0; ck < RBC; ++ck) {
    constexpr int dummy = 0; (void)dummy;
    const int rk = ck >> 1;                   // static after unrolling
    for (int kx = 0; kx < 16; ++kx) {
      const int k = kx + 16 * ck;
      if (k >= n) break;
      const int ky = 16 * (ck & 1) + kx;
      double* cb = colbuf + (k & 1) * NR;
      if (tx == kx) {
#pragma unroll
        for (int r = 0; r < RBR; ++r) cb[ty + 32 * r] = A[r][ck];
      }
      __syncthreads();
      const double pv = cb[k];
      if (!(pv > 0.0)) bad = true;
      const double pinv = __drcp_rn((pv > 0.0) ? pv : 1.0);
      if (tid == 0) piv[k] = (pv > 0.0) ? pv : 1.0;
      double ci[RBR], cj[RBC];
#pragma unroll
      for (int r = 0; r < RBR; ++r) ci[r] = cb[ty + 32 * r];
#pragma unroll
      for (int c = 0; c < RBC; ++c) cj[c] = cb[tx + 16 * c] * pinv;
      const bool rowk = (ty == ky), colk = (tx == kx);
      // the generic rank-1 update everywhere, then the pivot row / column are overwritten by their owners (selecting per
      // element cost 70 of the 140 instructions of a sweep)
#pragma unroll
      for (int r = 0; r < RBR; ++r)
#pragma unroll
        for (int c = 0; c < RBC; ++c) A[r][c] = fma(-ci[r], cj[c], A[r][c]);
      if (colk) {                             // column k: A_ik / p
#pragma unroll
        for (int r = 0; r < RBR; ++r) A[r][ck] = ci[r] * pinv;
      }
      if (rowk) {                             // row k: A_kj / p, and -1/p on the diagonal
#pragma unroll
        for (int c = 0; c < RBC; ++c) A[rk][c] = cj[c];
        if (colk) A[rk][ck] = -pinv;
      }
    }
  }
  if (bad && tid == 0) atomicOr(p.flags + blockIdx.y, 1);
  __syncthreads();
  // ---- log|det K| = sum log pivot;  alpha = K^-1 y ------------------------------------------------------------------------
  double part = 0.0;
  for (int k = tid; k < n; k += REG_THREADS) part += log(piv[k]);
  const double logdet = ex_block_sum<REG_WARPS>(part, red);
  {
    double yb[RBC];
#pragma unroll
    for (int c = 0; c < RBC; ++c) yb[c] = ys[tx + 16 * c];
#pragma unroll
    for (int r = 0; r < RBR; ++r) {
      double s = 0.0;
#pragma unroll
      for (int c = 0; c < RBC; ++c) s = fma(-A[r][c], yb[c], s);
      for (int o = 8; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);      // over the 16 threads of this row group
      if (tx == 0) alpha[ty + 32 * r] = (ty + 32 * r < n) ? s : 0.0;
    }
  }
  __syncthreads();
  part = 0.0;
  for (int a = tid; a < n; a += REG_THREADS) part += ys[a] * alpha[a];
  const double yay = ex_block_sum<REG_WARPS>(part, red);
  if (tid == 0) out[0] = 0.5 * yay + 0.5 * logdet;
  // ---- gradient: M = k o (alpha alpha^T - K^-1) in place of A --------------------------------------------------------------
  double S[kMaxTerms], Q[kMaxTerms], D[DCH], trW = 0.0;
#pragma unroll
  for (int t = 0; t < kMaxTerms; ++t) { S[t] = 0.0; Q[t] = 0.0; }
  {
    double aa[RBR], ab[RBC];
#pragma unroll
    for (int r = 0; r < RBR; ++r) aa[r] = alpha[ty + 32 * r];
#pragma unroll
    for (int c = 0; c < RBC; ++c) ab[c] = alpha[tx + 16 * c];
#pragma unroll
    for (int r = 0; r < RBR; ++r) {
#pragma unroll
      for (int c = 0; c < RBC; ++c) {
        const int a = ty + 32 * r, b = tx + 16 * c;
        const double W = fma(aa[r], ab[c], A[r][c]);             // A = -K^-1
        if (a == b && a < n) trW += W;
        const double Mv = Ks[a * NP + b] * W;                     // 0 on the padding
        A[r][c] = Mv;
        S[0] += Mv;
      }
    }
  }
  // this thread's share of D_k = sum_ab (x_ak - x_bk)^2 M_ab
  auto dim_sum = [&](int k) -> double {
    double xa[RBR], xb[RBC];
#pragma unroll
    for (int r = 0; r < RBR; ++r) xa[r] = Xs[(ty + 32 * r) * xld + k];
#pragma unroll
    for (int c = 0; c < RBC; ++c) xb[c] = Xs[(tx + 16 * c) * xld + k];
    double acc = 0.0;
#pragma unroll
    for (int r = 0; r < RBR; ++r)
#pragma unroll
      for (int c = 0; c < RBC; ++c) {
        const double df = xa[r] - xb[c];
        acc = fma(df * df, A[r][c], acc);
      }
    return acc;
  };
  const int chunks = (d + DCH - 1) / DCH;
  const int n_sweeps = hv.any_ard ? chunks : 1;
  if (!(hv.any_ard && chunks == 1)) {         // Q = sum_ab |x_a - x_b|^2 M_ab = sum_k D_k (RBF sigma); one ARD chunk: below
    double qsum = 0.0;
    for (int k = 0; k < d; ++k) qsum += dim_sum(k);
    Q[0] = qsum;
  }
  for (int sw = 0; sw < n_sweeps; ++sw) {
    const int ts = hv.any_ard ? 0 : -1;
    const int k0 = hv.any_ard ? sw * DCH : 0;
    const int kn = hv.any_ard ? ((d - k0 < DCH) ? (d - k0) : DCH) : 0;
#pragma unroll
    for (int k = 0; k < DCH; ++k) D[k] = (k < kn) ? dim_sum(k0 + k) : 0.0;
    if (hv.any_ard && chunks == 1) {
      double qsum = 0.0;
#pragma unroll
      for (int k = 0; k < DCH; ++k) qsum += D[k];
      Q[0] = qsum;
    }
    ex_gradient_emit<REG_WARPS>(hv, sw, ts, k0, kn, S, Q, D, trW, -0.5, out + 1, sums, red);
  }
}

// Sum the per-expert rows: one CTA per column, thread t adds experts t, t+256, ... and the 256 partials are combined by
// a fixed tree -- the order never depends on timing, so the result is deterministic.  blockIdx.y: the slot (one-vs-rest
// class, fold slot) whose rows [E][width] are summed; a fold slot sums only its set's experts.
__global__ void __launch_bounds__(EX_THREADS) rows_reduce_kernel(double* __restrict__ total,
                                                                   const double* __restrict__ per_expert, long long E,
                                                                   int width, const int* __restrict__ sets,
                                                                   const long long* __restrict__ first) {
  __shared__ double part[EX_THREADS];
  const int c = blockIdx.x;
  total += static_cast<size_t>(blockIdx.y) * width;
  per_expert += static_cast<size_t>(blockIdx.y) * E * width;
  const long long n_rows = sets ? first[sets[blockIdx.y] + 1] - first[sets[blockIdx.y]] : E;
  double s = 0.0;
  for (long long e = threadIdx.x; e < n_rows; e += EX_THREADS) s += per_expert[e * width + c];
  part[threadIdx.x] = s;
  __syncthreads();
  for (int o = EX_THREADS / 2; o > 0; o >>= 1) {
    if (threadIdx.x < o) part[threadIdx.x] += part[threadIdx.x + o];
    __syncthreads();
  }
  if (threadIdx.x == 0) total[c] = part[0];
}

// ---------------------------------------------------------------------------------------------------------------------
// General path: experts of ANY size (GaussianProcessParams.scala:36 puts no bound on datasetSizeForExpert) and kernel
// matrices that are not positive definite.  Exactly the reference's arithmetic: LU with partial pivoting
// (commons/util/logDetAndInv.scala:58-63 -> LAPACK dgetrf), log|det| = sum log|u_ii| with the SIGN IGNORED (GPR:59 drops
// it), inverse from the same factors (dgetri).  The kernel matrices live in global memory ([E][n_max][n_max], experts
// smaller than n_max padded with an identity block); the factorizations are cuBLAS' batched LU / inverse (plain library
// calls on small dense matrices), the build / objective / gradient kernels are ours.  Every index into an n_max x n_max
// matrix that the build shares with the on-chip kernels is an int: n_max <= kBcmLuMaxPoints.
// ---------------------------------------------------------------------------------------------------------------------
struct GenParams {
  const double* X; const double* y; const long long* off;
  int n_max, x_in_smem;
  HyperView hv;
  double* A;                // [E][n_max][n_max]  K, then its LU factors
  const double* Ainv;       // [E][n_max][n_max]  inverse
  double* ya;               // [E][2][n_max]  y and alpha of each expert when 2 n_max doubles do not fit in shared memory
                            // (plan.ya_in_ws), else nullptr: they live in shared memory
  const int* info;          // [E] dgetrf info (> 0: exactly singular)
  double* out;              // [E][1 + n_hypers]
  int* flags;               // bit 1: some expert's matrix is singular (MatrixSingularException)
};

__global__ void __launch_bounds__(EX_THREADS) gen_build_kernel(const GenParams p, double** Aptr, double** Cptr, double* Ainv) {
  const long long e = blockIdx.x;
  const long long r0 = p.off[e];
  const int n = static_cast<int>(p.off[e + 1] - r0), ld = p.n_max;
  double* K = p.A + static_cast<size_t>(e) * ld * ld;
  if (threadIdx.x == 0) { Aptr[e] = K; Cptr[e] = Ainv + static_cast<size_t>(e) * ld * ld; }
  const double* Xe = p.X + static_cast<size_t>(r0) * p.hv.d;
  ex_build_kernel<true>(p.hv, Xe, p.hv.d, n, K, ld);
  for (int idx = threadIdx.x; idx < ld * ld; idx += EX_THREADS) {      // identity padding (does not change det or alpha)
    const int a = idx / ld, b = idx % ld;
    if (a >= n || b >= n) K[idx] = (a == b) ? 1.0 : 0.0;
  }
}

__global__ void __launch_bounds__(EX_THREADS) gen_objective_kernel(const GenParams p) {
  extern __shared__ double sm[];
  const long long e = blockIdx.x;
  const long long r0 = p.off[e];
  const int n = static_cast<int>(p.off[e + 1] - r0), ld = p.n_max;
  double* yv = p.ya ? p.ya + static_cast<size_t>(e) * 2 * ld : sm;   // [n_max]
  double* alpha = yv + p.n_max;          // [n_max]
  double* red = p.ya ? sm : alpha + p.n_max;                         // [8]
  double* sums = red + 8;                // [EX_SUMS]
  double* Xs = sums + EX_SUMS;
  const int tid = threadIdx.x;
  const double* LU = p.A + static_cast<size_t>(e) * ld * ld;
  const double* Ki = p.Ainv + static_cast<size_t>(e) * ld * ld;
  int xld;
  const double* Xe = ex_stage_rows(p.X + static_cast<size_t>(r0) * p.hv.d, n, p.hv.d, p.x_in_smem, Xs, xld);
  for (int i = tid; i < n; i += EX_THREADS) yv[i] = p.y[r0 + i];
  __syncthreads();
  // log|det| = sum log|u_ii| (LU2logdet, logDetAndInv.scala:36-51; cuBLAS stores the factors column-major in place:
  // the diagonal is the same either way)
  double part = 0.0;
  for (int i = tid; i < n; i += EX_THREADS) part += log(fabs(LU[static_cast<size_t>(i) * ld + i]));
  const double logdet = ex_block_sum(part, red);
  if (tid == 0 && p.info[e] > 0) atomicOr(p.flags, 2);
  // alpha = K^-1 y  (the inverse of a symmetric matrix: row-/column-major reads agree up to rounding; use the average)
  for (int a = tid; a < n; a += EX_THREADS) {
    double s = 0.0;
    for (int b = 0; b < n; ++b)
      s = fma(0.5 * (Ki[static_cast<size_t>(a) * ld + b] + Ki[static_cast<size_t>(b) * ld + a]), yv[b], s);
    alpha[a] = s;
  }
  __syncthreads();
  part = 0.0;
  for (int a = tid; a < n; a += EX_THREADS) part += yv[a] * alpha[a];
  const double yay = ex_block_sum(part, red);
  double* out = p.out + static_cast<size_t>(e) * (1 + p.hv.n_hypers);
  if (tid == 0) out[0] = 0.5 * yay + 0.5 * logdet;                                            // GPR:61
  ex_descriptor_gradient(p.hv, Xe, xld, n,
                         [&](int a, int b) {
                           return alpha[a] * alpha[b] - 0.5 * (Ki[static_cast<size_t>(a) * ld + b] + Ki[static_cast<size_t>(b) * ld + a]);
                         },
                         -0.5, out + 1, sums, red);                                           // GPR:63-66
}

// ---------------------------------------------------------------------------------------------------------------------
// Dispatch: the shared memory of the BCM kernels and the one rule that picks the kernel of either objective.
// ---------------------------------------------------------------------------------------------------------------------
// bcm_nll_reg_kernel shapes for one non-Eye term, by 16-row blocks of the largest expert (up to 128 points)
struct RegShape { int blocks, rbr, rbc; void (*kernel)(NllParams); };
const RegShape kRegShapes[] = {{4, 2, 4, bcm_nll_reg_kernel<2, 4>}, {6, 3, 6, bcm_nll_reg_kernel<3, 6>},
                               {7, 4, 7, bcm_nll_reg_kernel<4, 7>}, {8, 4, 8, bcm_nll_reg_kernel<4, 8>}};
constexpr size_t kStageTwoCtas = 113 * 1024;   // bcm_nll_kernel stages the expert's rows while two CTAs fit per SM
constexpr size_t kStageGeneral = 200 * 1024;   // gen_objective_kernel (general path) stages them up to this size

size_t bcm_nll_reg_smem_bytes(int rbr, int rbc, int d) {
  const size_t nr = 32 * static_cast<size_t>(rbr), np = 16 * static_cast<size_t>(rbc);
  return sizeof(double) * (5 * nr + 16 + EX_SUMS + nr * (d | 1) + nr * np);
}
size_t gen_objective_smem_bytes(int n_max) { return sizeof(double) * (2 * static_cast<size_t>(n_max) + 8 + EX_SUMS); }

}  // namespace

// [E][n_max][n_max] K / LU, [E][n_max][n_max] K^-1, [E][2][n_max] y and alpha, 2 E pointers, E info, E n_max pivots
size_t bcm_general_workspace_bytes(long long E, int n_max) {
  const size_t mat = static_cast<size_t>(E) * n_max * n_max * sizeof(double);
  const size_t ya = static_cast<size_t>(E) * 2 * n_max * sizeof(double);
  return 2 * mat + ya + static_cast<size_t>(E) * (2 * sizeof(double*) + sizeof(int) * (1 + static_cast<size_t>(n_max))) +
         256;
}
size_t bcm_nll_smem_bytes(int n_max) {
  return sizeof(double) * (static_cast<size_t>(n_max) * (n_max + 1) + 3 * static_cast<size_t>(n_max) + 8 + EX_SUMS);
}

ObjectivePlan plan_objective(Objective kind, const ExpertSet& ex, int n_terms) {
  ObjectivePlan plan;
  auto stage_rows = [&](ObjectiveVariant v, size_t smem, size_t limit) {
    const size_t with_x = smem + sizeof(double) * static_cast<size_t>(ex.n_max) * (ex.d | 1);
    plan.variant = v;
    plan.x_in_smem = (with_x <= limit) ? 1 : 0;
    plan.smem = plan.x_in_smem ? with_x : smem;
    return plan;
  };
  if (kind == Objective::kLaplace || kind == Objective::kLaplaceAnySize) {
    if (laplace_smem_bytes(ex.n_max) > kSmemOptInMax) {
      if (kind == Objective::kLaplace) return plan;                      // kRefused
      plan.variant = ObjectiveVariant::kLaplaceGlobal;
      plan.cta_ws = laplace_global_cta_bytes(ex.n_max);
      return plan;
    }
    return stage_rows(ObjectiveVariant::kLaplace, laplace_smem_bytes(ex.n_max), kSmemOptInMax);
  }
  // experts whose shared-memory Cholesky does not fit, or a kernel matrix on which it broke down: the LU path
  if (kind == Objective::kBcmLu || bcm_nll_smem_bytes(ex.n_max) > kSmemOptInMax) {
    plan.lu_ws = bcm_general_workspace_bytes(ex.E, ex.n_max);
    stage_rows(ObjectiveVariant::kLu, gen_objective_smem_bytes(ex.n_max), kStageGeneral);
    if (plan.smem > kSmemOptInMax) {     // n_max > 14511: y and alpha go to the workspace (the rows are not staged here)
      plan.ya_in_ws = 1;
      plan.smem = gen_objective_smem_bytes(0);
    }
    return plan;
  }
  // one non-Eye term, experts of <= 128 points: the register-resident kernel (SGP_BCM_IMPL=smem selects the other one)
  static const bool force_smem = [] { const char* e = getenv("SGP_BCM_IMPL"); return e && std::string(e) == "smem"; }();
  if (n_terms == 1 && !force_smem) {
    const int rb = (ex.n_max + 15) / 16;
    for (const RegShape& r : kRegShapes) {
      if (rb > r.blocks) continue;
      const size_t smem = bcm_nll_reg_smem_bytes(r.rbr, r.rbc, ex.d);
      if (smem > kSmemOptInMax) break;                 // too wide: the shared-memory kernel
      plan.variant = static_cast<ObjectiveVariant>(&r - kRegShapes);   // kReg24 .. kReg48 in kRegShapes' order
      plan.smem = smem;
      return plan;
    }
  }
  return stage_rows(ObjectiveVariant::kSmem, bcm_nll_smem_bytes(ex.n_max), kStageTwoCtas);
}

cudaError_t launch_rows_reduce(double* dTotal, const double* dPerExpert, long long E, int width, cudaStream_t s,
                               int n_slots, const int* sets, const long long* first) {
  rows_reduce_kernel<<<dim3(width, n_slots), EX_THREADS, 0, s>>>(dTotal, dPerExpert, E, width, sets, first);
  return cudaGetLastError();
}

cudaError_t launch_bcm_nll(const ObjectivePlan& plan, const ExpertSet& ex, const HyperView& hv, const ObjectiveSlots& sl,
                           double* rows, double* total, int* flags, cudaStream_t s) {
  NllParams p{};
  p.X = ex.X; p.y = ex.y; p.off = ex.off; p.n_max = ex.n_max; p.x_in_smem = plan.x_in_smem;
  p.hv = hv; p.sets = sl.sets; p.first = sl.first; p.kf = sl.kf; p.slot_stride = sl.slot_stride;
  p.out = rows; p.flags = flags;
  const long long E = sl.E_max;
  const int n_slots = sl.n_slots;
  const bool reg = plan.variant < ObjectiveVariant::kSmem;
  void (*kernel)(NllParams) = reg ? kRegShapes[static_cast<int>(plan.variant)].kernel : bcm_nll_kernel;
  cudaError_t e = allow_dynamic_smem(reinterpret_cast<const void*>(kernel));
  if (e != cudaSuccess) return e;
  kernel<<<dim3(static_cast<unsigned>(E), static_cast<unsigned>(n_slots)), reg ? REG_THREADS : EX_THREADS, plan.smem, s>>>(p);
  e = cudaGetLastError();
  if (e != cudaSuccess) return e;
  return launch_rows_reduce(total, rows, E, 1 + hv.n_hypers, s, n_slots, p.sets, p.first);
}

cudaError_t launch_bcm_nll_general(const ObjectivePlan& plan, cublasHandle_t blas, int* blas_status, void* ws,
                                   const ExpertSet& ex, const HyperView& hv, double* rows, double* total, int* flags,
                                   cudaStream_t s) {
  *blas_status = 0;
  const long long E = ex.E;
  const int n_max = ex.n_max;
  const size_t mat = static_cast<size_t>(E) * n_max * n_max;
  double* A = static_cast<double*>(ws);
  double* Ainv = A + mat;
  double* ya = Ainv + mat;
  double** Aptr = reinterpret_cast<double**>(ya + static_cast<size_t>(E) * 2 * n_max);
  double** Cptr = Aptr + E;
  int* info = reinterpret_cast<int*>(Cptr + E);
  int* piv = info + E;
  GenParams p{};
  p.X = ex.X; p.y = ex.y; p.off = ex.off; p.n_max = n_max; p.x_in_smem = plan.x_in_smem;
  p.hv = hv; p.A = A; p.Ainv = Ainv; p.ya = plan.ya_in_ws ? ya : nullptr; p.info = info; p.out = rows; p.flags = flags;
  gen_build_kernel<<<static_cast<unsigned>(E), EX_THREADS, 0, s>>>(p, Aptr, Cptr, Ainv);
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) return e;
  cublasSetStream(blas, s);
  // K is symmetric, so cuBLAS' column-major view of the row-major buffer is the same matrix
  cublasStatus_t st = cublasDgetrfBatched(blas, n_max, Aptr, n_max, piv, info, static_cast<int>(E));
  if (st == CUBLAS_STATUS_SUCCESS)
    st = cublasDgetriBatched(blas, n_max, Aptr, n_max, piv, Cptr, n_max, info + 0, static_cast<int>(E));
  if (st != CUBLAS_STATUS_SUCCESS) { *blas_status = static_cast<int>(st); return cudaSuccess; }
  e = allow_dynamic_smem(reinterpret_cast<const void*>(gen_objective_kernel));
  if (e != cudaSuccess) return e;
  gen_objective_kernel<<<static_cast<unsigned>(E), EX_THREADS, plan.smem, s>>>(p);
  e = cudaGetLastError();
  if (e != cudaSuccess) return e;
  return launch_rows_reduce(total, rows, E, 1 + hv.n_hypers, s);
}

}  // namespace sgp
