// GreedilyOptimizingActiveSetProvider (commons/ActiveSetProvider.scala:58-139: Seeger et al. 2003 forward selection as the
// reference codes it) with RANK-1 UPDATES.  The reference rebuilds everything in every round -- one statistics pass
// (K_mn K_nm, K_mn y), two m x m inverses and three quadratic forms per candidate point: O(N m^2) per round, O(N m^3) for an
// active set of m points.  Here the cross kernel K_mn lives on the device and grows by one row per round; because
//   K_mm' = [[K_mm, c], [c', kii]]   and   A' = s2 K_mm' + G' = [[A, w], [w', s2 kii + k*.k*]],   w = s2 c + K_mn k*
// are BORDERED extensions, the inverses and the per-point quantities of ASP:109-113 follow from the previous round:
//   p_i' = p_i + (u~.k_i - k*_i)^2 / s~        u~ = inv(K_mm) c,   s~ = kii - c.u~
//   q_i' = q_i + (u.k_i  - k*_i)^2 / s         u  = inv(A) w,      s  = s2 kii + k*.k* - w.u   (s <= 0  <=>  A' not PD)
//   mu_i' = mu_i + a (u.k_i - k*_i)            a  = (u.b - k*.y) / s
// i.e. per round one kernel column (N kernel evaluations), one GEMV (K_mn k*), one N x m x 2 GEMM (K_nm [u~ u]) and an
// elementwise pass: O(N m).  The m x m bookkeeping (bordered inverse updates, O(m^2) per round) runs on the host in fp64.
// Selection semantics are the reference's: candidates folded per expert (point i belongs to expert i % E) left to right with
// later-wins ties and NaN poisoning (ASP:108-127), poisoned experts dropped (ASP:131), the FIRST expert with the maximal score
// wins (Ordering.max), already selected points are not excluded, `sigma2` is the kernel's whiteNoiseVar (ASP:76).
#include <cmath>
#include <vector>

#include "sgp_internal.h"

namespace sgp {
namespace {

// out[i] = sum_t C_t exp(-sum_k ((x_ik - x_jk) beta_tk)^2): the cross kernel of every point against point j (Eye terms add
// nothing to a cross kernel, kernel/Kernel.scala:157)
__global__ void greedy_column_kernel(double* __restrict__ out, const double* __restrict__ X, long long n, int d,
                                     long long j, const double* __restrict__ beta /*[n_terms][d]*/, const KernelFlat kf) {
  const long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x;
  if (i >= n) return;
  const double* xi = X + static_cast<size_t>(i) * d;
  const double* xj = X + static_cast<size_t>(j) * d;
  double v = 0.0;
  for (int t = 0; t < kf.n_terms; ++t) {
    double q = 0.0;
    for (int k = 0; k < d; ++k) {
      const double df = xi[k] * beta[t * d + k] - xj[k] * beta[t * d + k];      // same form as cross_kernel_kernel
      q = fma(df, df, q);
    }
    v = kf.fold_term(v, t, q);
  }
  out[i] = v;
}

// ASP:109-124 after the rank-1 update of p, q, mu.  T = [t~ | t] (column-major N x 2), t = K_nm u
__global__ void greedy_update_kernel(double* __restrict__ p, double* __restrict__ q, double* __restrict__ mu,
                                     double* __restrict__ delta, const double* __restrict__ kstar,
                                     const double* __restrict__ T, const double* __restrict__ y, long long n, int have_t,
                                     double inv_s1, double inv_s2, double a, double kii, double s2n) {
  const long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x;
  if (i >= n) return;
  const double ks = kstar[i];
  const double e1 = (have_t ? T[i] : 0.0) - ks, e2 = (have_t ? T[n + i] : 0.0) - ks;
  const double pi = p[i] + e1 * e1 * inv_s1, qi = q[i] + e2 * e2 * inv_s2, mi = mu[i] + a * e2;
  p[i] = pi; q[i] = qi; mu[i] = mi;
  const double sigma = sqrt(s2n);
  const double li = sqrt(kii - pi);
  const double r = sigma / li, r2 = r * r;
  const double ksi = 1.0 / (r2 + 1.0 - qi);
  const double kappa = ksi * (1.0 + 2.0 * r2);
  const double dy = y[i] - mi;
  delta[i] = -log(r) - (log(ksi) + ksi * (1.0 - kappa) / s2n * (dy * dy) - kappa + 2.0) / 2.0;
}

// ASP:108-127, one thread per expert: (oldMax, oldIdx) folded over the expert's points e, e + E, ... in order
__global__ void greedy_fold_kernel(double* __restrict__ best, long long* __restrict__ best_idx,
                                   const double* __restrict__ delta, long long n, long long E) {
  const long long e = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x;
  if (e >= E) return;
  double old_max = -1.7976931348623157e308;       // Double.MinValue
  long long old_idx = -1;
  bool poisoned = false;
  for (long long i = e; i < n; i += E) {
    const double dl = delta[i];
    if (!(old_max > dl) || poisoned) old_idx = i;  // a NaN on either side compares false -> i; ties -> the later point
    if (dl != dl) poisoned = true;                 // math.max(NaN, x) = NaN from here on
    else if (dl > old_max) old_max = dl;
  }
  best[e] = poisoned ? nan("") : old_max;
  best_idx[e] = old_idx;
}

// RDD.filter(!isNaN).max(): the FIRST expert with the maximal score (Ordering.max keeps x when gteq(x, y)).  One block.
__global__ void greedy_argmax_kernel(long long* __restrict__ out /*[1]: point index, -1 = empty.max*/,
                                     const double* __restrict__ best, const long long* __restrict__ best_idx, long long E) {
  __shared__ double sv[256];
  __shared__ long long se[256];
  double v = 0.0;
  long long be = -1;
  for (long long e = threadIdx.x; e < E; e += blockDim.x) {       // ascending e per thread: strict > keeps the first
    const double b = best[e];
    if (b != b) continue;
    if (be < 0 || b > v) { v = b; be = e; }
  }
  sv[threadIdx.x] = v; se[threadIdx.x] = be;
  __syncthreads();
  for (int s = blockDim.x / 2; s > 0; s >>= 1) {
    if (threadIdx.x < s) {
      const long long e2 = se[threadIdx.x + s];
      const double v2 = sv[threadIdx.x + s];
      const long long e1 = se[threadIdx.x];
      if (e2 >= 0 && (e1 < 0 || v2 > sv[threadIdx.x] || (v2 == sv[threadIdx.x] && e2 < e1))) {
        sv[threadIdx.x] = v2; se[threadIdx.x] = e2;
      }
    }
    __syncthreads();
  }
  if (threadIdx.x == 0) out[0] = se[0] >= 0 ? best_idx[se[0]] : -1;
}

#define SGP_BLAS(c, expr)                                                                              \
  do {                                                                                                 \
    cublasStatus_t st_ = (expr);                                                                       \
    if (st_ != CUBLAS_STATUS_SUCCESS)                                                                  \
      return ::sgp::fail((c), SGP_E_CUDA, std::string(#expr) + ": cuBLAS status " + std::to_string(static_cast<int>(st_))); \
  } while (0)

// inv(A) of the leading n x n block (row stride ld) through a host Cholesky factorisation; false if A is not positive definite
bool chol_inverse(const std::vector<double>& A, int n, int ld, std::vector<double>& inv) {
  std::vector<double> L(static_cast<size_t>(n) * n, 0.0), Li(static_cast<size_t>(n) * n, 0.0);
  for (int j = 0; j < n; ++j) {
    double dsum = A[static_cast<size_t>(j) * ld + j];
    for (int k = 0; k < j; ++k) dsum -= L[static_cast<size_t>(j) * n + k] * L[static_cast<size_t>(j) * n + k];
    if (!(dsum > 0.0)) return false;
    const double ljj = std::sqrt(dsum);
    L[static_cast<size_t>(j) * n + j] = ljj;
    for (int i = j + 1; i < n; ++i) {
      double v = A[static_cast<size_t>(i) * ld + j];
      const double* li = L.data() + static_cast<size_t>(i) * n;
      const double* lj = L.data() + static_cast<size_t>(j) * n;
      for (int k = 0; k < j; ++k) v -= li[k] * lj[k];
      L[static_cast<size_t>(i) * n + j] = v / ljj;
    }
  }
  for (int j = 0; j < n; ++j) {                       // Li = inv(L), column by column
    Li[static_cast<size_t>(j) * n + j] = 1.0 / L[static_cast<size_t>(j) * n + j];
    for (int i = j + 1; i < n; ++i) {
      double v = 0.0;
      const double* li = L.data() + static_cast<size_t>(i) * n;
      for (int k = j; k < i; ++k) v -= li[k] * Li[static_cast<size_t>(k) * n + j];
      Li[static_cast<size_t>(i) * n + j] = v / li[i];
    }
  }
  for (int i = 0; i < n; ++i)                         // inv(A) = Li' Li
    for (int j = 0; j <= i; ++j) {
      double v = 0.0;
      for (int k = i; k < n; ++k) v += Li[static_cast<size_t>(k) * n + i] * Li[static_cast<size_t>(k) * n + j];
      inv[static_cast<size_t>(i) * ld + j] = v;
      inv[static_cast<size_t>(j) * ld + i] = v;
    }
  return true;
}

}  // namespace

int run_greedy(Ctx* c, const KernelFlat& kf, const std::vector<double>& beta_flat /*[n_terms][d]*/, const double* X,
               const double* y, bool x_on_device, long long n, int d, long long E, long long first_index, int m_target,
               long long* indices_out) {
  const size_t N = static_cast<size_t>(n);
  // ---- device state: X, y (host input only), K_mn (row per selected point), p, q, mu, delta, [t~ t], per-expert folds --
  const size_t xy = x_on_device ? 0 : N * d + N;
  const size_t bytes = (xy + static_cast<size_t>(m_target) * N + 4 * N + 2 * N) * 8 +
                       static_cast<size_t>(E) * 16 + static_cast<size_t>(kMaxTerms) * d * 8 +
                       static_cast<size_t>(m_target) * 2 * 8 + static_cast<size_t>(m_target + 1) * 8 + 64;
  size_t free_b = 0, total_b = 0;
  SGP_CUDA(c, cudaMemGetInfo(&free_b, &total_b));
  if (bytes > free_b + c->greedy_ws.cap)
    return fail(c, SGP_E_NOMEM, "sgp_greedy_active_set: the N x m cross kernel does not fit in device memory");
  int rc = ctx_scratch(c, c->greedy_ws, bytes);
  if (rc != SGP_OK) return rc;
  double* ws = static_cast<double*>(c->greedy_ws.p);
  const double* dX = x_on_device ? X : ws;
  const double* dy = x_on_device ? y : ws + N * d;
  double* Kt = ws + xy;                                  // [m_target][N]
  double* dp = Kt + static_cast<size_t>(m_target) * N;
  double* dq = dp + N;
  double* dmu = dq + N;
  double* ddelta = dmu + N;
  double* dT = ddelta + N;                               // [2][N]
  double* dbest = dT + 2 * N;                            // [E]
  long long* dbest_idx = reinterpret_cast<long long*>(dbest + E);
  double* dbeta = reinterpret_cast<double*>(dbest_idx + E);
  double* dU = dbeta + static_cast<size_t>(kMaxTerms) * d;   // [2][m_target] column-major m_target x 2
  double* dg = dU + static_cast<size_t>(m_target) * 2;   // [m_target + 1]
  long long* dsel = reinterpret_cast<long long*>(dg + m_target + 1);
  cudaStream_t s = c->stream;
  if (!x_on_device) {
    SGP_CUDA(c, cudaMemcpyAsync(ws, X, N * d * 8, cudaMemcpyHostToDevice, s));
    SGP_CUDA(c, cudaMemcpyAsync(ws + N * d, y, N * 8, cudaMemcpyHostToDevice, s));
  }
  SGP_CUDA(c, cudaMemcpyAsync(dbeta, beta_flat.data(), beta_flat.size() * 8, cudaMemcpyHostToDevice, s));
  SGP_CUDA(c, cudaMemsetAsync(dp, 0, 3 * N * 8, s));      // p, q, mu
  SGP_BLAS(c, cublasSetStream(c->blas, s));
  SGP_BLAS(c, cublasSetPointerMode(c->blas, CUBLAS_POINTER_MODE_HOST));

  const double kii = kf.self_kernel, s2n = kf.eye_sum;    // trainingKernelDiag (Kernel.scala:111-114), whiteNoiseVar (ASP:76)

  // ---- host state: inv(K_mm), inv(A), b, magic vector --------------------------------------------------------------------
  const int M = m_target;
  std::vector<double> Kinv(static_cast<size_t>(M) * M, 0.0), Ainv(static_cast<size_t>(M) * M, 0.0), b(M, 0.0), mv(M, 0.0);
  std::vector<double> Kmm(static_cast<size_t>(M) * M, 0.0), Amat(static_cast<size_t>(M) * M, 0.0);   // explicit copies (refresh)
  std::vector<double> cvec(M), g(M + 1), ut(M), u(M), w(M), U2(static_cast<size_t>(M) * 2);
  const unsigned nblk = static_cast<unsigned>((N + 255) / 256);
  long long idx = first_index;
  for (int m = 0; m < M; ++m) {
    indices_out[m] = idx;
    if (m == M - 1) break;                                  // the last point needs no scores
    double* krow = Kt + static_cast<size_t>(m) * N;
    greedy_column_kernel<<<nblk, 256, 0, s>>>(krow, dX, n, d, idx, dbeta, kf);
    SGP_CUDA(c, cudaGetLastError());
    c->launches += 1;
    // g = K_mn k* over the m + 1 rows (the last entry is k*.k*), beta = k*.y;  c = K_mn[:, idx]
    const double one = 1.0, zero = 0.0;
    SGP_BLAS(c, cublasSetPointerMode(c->blas, CUBLAS_POINTER_MODE_HOST));
    SGP_BLAS(c, cublasDgemv(c->blas, CUBLAS_OP_T, static_cast<int>(n), m + 1, &one, Kt, static_cast<int>(n), krow, 1, &zero,
                            dg, 1));
    double bnew = 0.0;
    SGP_BLAS(c, cublasDdot(c->blas, static_cast<int>(n), krow, 1, dy, 1, &bnew));     // synchronises
    SGP_CUDA(c, cudaMemcpyAsync(g.data(), dg, static_cast<size_t>(m + 1) * 8, cudaMemcpyDeviceToHost, s));
    if (m > 0)
      SGP_CUDA(c, cudaMemcpy2DAsync(cvec.data(), 8, Kt + idx, N * 8, 8, m, cudaMemcpyDeviceToHost, s));
    SGP_CUDA(c, cudaStreamSynchronize(s));
    c->launches += 2;
    const double gamma = g[m];
    // u~ = inv(K_mm) c, u = inv(A) w
    double s1 = kii, s2 = s2n * kii + gamma, ub = 0.0;
    for (int i = 0; i < m; ++i) w[i] = s2n * cvec[i] + g[i];
    for (int i = 0; i < m; ++i) {
      double a1 = 0.0, a2 = 0.0;
      const double* kr = Kinv.data() + static_cast<size_t>(i) * M;
      const double* ar = Ainv.data() + static_cast<size_t>(i) * M;
      for (int j = 0; j < m; ++j) { a1 += kr[j] * cvec[j]; a2 += ar[j] * w[j]; }
      ut[i] = a1; u[i] = a2;
    }
    for (int i = 0; i < m; ++i) { s1 -= cvec[i] * ut[i]; s2 -= w[i] * u[i]; }
    for (int i = 0; i < m; ++i) {
      Kmm[static_cast<size_t>(m) * M + i] = Kmm[static_cast<size_t>(i) * M + m] = cvec[i];
      Amat[static_cast<size_t>(m) * M + i] = Amat[static_cast<size_t>(i) * M + m] = w[i];
    }
    Kmm[static_cast<size_t>(m) * M + m] = kii;
    Amat[static_cast<size_t>(m) * M + m] = s2n * kii + gamma;
    b[m] = bnew;
    // A Schur complement that is tiny against its diagonal entry (the reference does not exclude selected points: a repeated
    // point makes A' nearly singular) has lost its digits to cancellation: rebuild both inverses from the explicit matrices.
    // A' is positive definite iff the factorisation succeeds (the reference's check: no negative eigenvalue, PGPH:62-65).
    const bool refresh = !(s2 > 1e-7 * (s2n * kii + gamma)) || !(s1 > 1e-7 * kii);
    if (refresh) {
      if (!chol_inverse(Kmm, m + 1, M, Kinv) || !chol_inverse(Amat, m + 1, M, Ainv))
        return fail(c, SGP_E_NOT_PD, "NotPositiveDefiniteException: some eigenvalues are negative");
      s1 = 1.0 / Kinv[static_cast<size_t>(m) * M + m];
      s2 = 1.0 / Ainv[static_cast<size_t>(m) * M + m];
      for (int i = 0; i < m; ++i) {
        ut[i] = -Kinv[static_cast<size_t>(i) * M + m] * s1;
        u[i] = -Ainv[static_cast<size_t>(i) * M + m] * s2;
      }
    }
    for (int i = 0; i < m; ++i) ub += u[i] * b[i];
    const double a = (ub - bnew) / s2;
    // t~ = K_nm u~, t = K_nm u
    if (m > 0) {
      for (int i = 0; i < m; ++i) { U2[i] = ut[i]; U2[static_cast<size_t>(M) + i] = u[i]; }
      SGP_CUDA(c, cudaMemcpyAsync(dU, U2.data(), static_cast<size_t>(M) * 2 * 8, cudaMemcpyHostToDevice, s));
      SGP_BLAS(c, cublasDgemm(c->blas, CUBLAS_OP_N, CUBLAS_OP_N, static_cast<int>(n), 2, m, &one, Kt, static_cast<int>(n), dU,
                              M, &zero, dT, static_cast<int>(n)));
      c->launches += 1;
    }
    greedy_update_kernel<<<nblk, 256, 0, s>>>(dp, dq, dmu, ddelta, krow, dT, dy, n, m > 0 ? 1 : 0, 1.0 / s1, 1.0 / s2, a, kii,
                                              s2n);
    SGP_CUDA(c, cudaGetLastError());
    greedy_fold_kernel<<<static_cast<unsigned>((E + 127) / 128), 128, 0, s>>>(dbest, dbest_idx, ddelta, n, E);
    SGP_CUDA(c, cudaGetLastError());
    greedy_argmax_kernel<<<1, 256, 0, s>>>(dsel, dbest, dbest_idx, E);
    SGP_CUDA(c, cudaGetLastError());
    c->launches += 3;
    long long next = -1;
    SGP_CUDA(c, cudaMemcpyAsync(&next, dsel, 8, cudaMemcpyDeviceToHost, s));
    // bordered inverse updates while the device scores the candidates
    //   inv' = [[inv + v v'/s, -v/s], [-v'/s, 1/s]]
    if (!refresh) {
      for (int i = 0; i < m; ++i) {
        double* kr = Kinv.data() + static_cast<size_t>(i) * M;
        double* ar = Ainv.data() + static_cast<size_t>(i) * M;
        const double f1 = ut[i] / s1, f2 = u[i] / s2;
        for (int j = 0; j < m; ++j) { kr[j] += f1 * ut[j]; ar[j] += f2 * u[j]; }
        kr[m] = -f1; ar[m] = -f2;
        Kinv[static_cast<size_t>(m) * M + i] = -f1;
        Ainv[static_cast<size_t>(m) * M + i] = -f2;
      }
      Kinv[static_cast<size_t>(m) * M + m] = 1.0 / s1;
      Ainv[static_cast<size_t>(m) * M + m] = 1.0 / s2;
    }
    for (int i = 0; i < m; ++i) mv[i] += u[i] * a;
    mv[m] = -a;
    SGP_CUDA(c, cudaStreamSynchronize(s));
    if (next < 0) return fail(c, SGP_E_BADARG, "empty.max");       // every expert poisoned by a NaN score (ASP:131-135)
    idx = next;
  }
  return SGP_OK;
}

}  // namespace sgp
