// The m x m tail (fp64, one GPU) and the per-window launch of block prediction (kernels in predict.cu).
//
//   commons/ProjectedGaussianProcessHelper.scala:49-65   getMagicVector + assertSymPositiveDefinite
//   commons/GaussianProcessCommons.scala:118-126         GaussianProjectedProcessRawPredictor.predict
//
// The reference's dense linear algebra is LAPACK through Breeze (dsyevd for the PD check, dgesv for `\`,
// dgetrf+dgetri for `inv`), all on one driver thread.  Here the tail runs on the device with cuSOLVER / cuBLAS
// (plain library factorizations of an m x m matrix -- not the hot path) and is organised for latency:
//
//   fast path (every well-posed model):  A = whiteNoiseVar K_mm + G is symmetric.  A successful Cholesky
//     factorization proves that every eigenvalue is > 0, i.e. the reference's check "no eigenvalue < 0" (PGPH:63)
//     passes -- without the O(10 m^3) dsyevd that dominated round 1's tail (26.5 ms at m = 1000).  The same factors
//     give  magicVector = A \ b  and  inv(A)  (dpotrs); K_mm (SPD: a kernel matrix plus the Eye terms) is inverted the
//     same way on a SECOND stream with its own cuSOLVER handle, concurrently with the A chain.  For SPD matrices the
//     Cholesky and LU solutions agree to rounding (both backward stable; the reference's LU pivots are a no-op
//     on a diagonally dominant SPD matrix up to rounding) -- the parity tests (mean / variance <= 1e-5 vs the oracle's
//     LAPACK LU) are unchanged.
//   slow path (Cholesky of A or K_mm breaks down):  exactly the reference's sequence -- dsyevd, throw iff an
//     eigenvalue is < 0 (a semi-definite matrix passes, PGPH:63 is a strict comparison), then LU solves/inverses
//     (dgetrf / dgetrs), SGP_E_SINGULAR on a zero pivot like Breeze's MatrixSingularException.
//
// All device workspaces live in the context and are reused across calls (cudaMalloc/cudaFree synchronise the device
// and cost more than the factorizations at m = 1000).
#include "sgp_internal.h"

namespace sgp {

#define SGP_SOLVER(c, expr)                                                                    \
  do {                                                                                         \
    cusolverStatus_t st_ = (expr);                                                             \
    if (st_ != CUSOLVER_STATUS_SUCCESS)                                                        \
      return fail((c), SGP_E_CUDA, std::string(#expr) + ": cusolver status " + std::to_string((int)st_)); \
  } while (0)

// Grow-only device scratch owned by the context.  A failed cudaMalloc also records its error as the runtime's last
// error, which the launch check of the next kernel on this thread would report; it is cleared here, and an
// out-of-memory failure returns SGP_E_NOMEM.
int ctx_scratch(Ctx* c, DevScratch& s, size_t bytes) {
  if (bytes <= s.cap && s.p) return SGP_OK;
  if (s.p) {
    SGP_CUDA(c, cudaStreamSynchronize(c->stream));
    if (c->tail_stream) SGP_CUDA(c, cudaStreamSynchronize(c->tail_stream));
    cudaFree(s.p);
    s.p = nullptr; s.cap = 0;
  }
  const cudaError_t e = cudaMalloc(&s.p, bytes ? bytes : 8);
  if (e != cudaSuccess) {
    s.p = nullptr;
    cudaGetLastError();
    return fail(c, e == cudaErrorMemoryAllocation ? SGP_E_NOMEM : SGP_E_CUDA,
                "cudaMalloc of " + std::to_string(bytes >> 20) + " MiB: " + cudaGetErrorString(e));
  }
  s.cap = bytes ? bytes : 8;
  return SGP_OK;
}

static const char* kNotPdMsg =
    "Some matrix which is supposed to be positive definite is not. This probably happened due "
    "to `sigma2` parameter being too small. Try to gradually increase it.";

// The reference's own sequence on one matrix (slow path): M is overwritten by its LU factors.
// inv_out = M^-1 ; optionally rhs_vec <- M^-1 rhs_vec.
static int lu_inverse(Ctx* c, cusolverDnHandle_t h, cudaStream_t s, int m, double* M, double* inv_out, double* rhs_vec,
                      double* work, int* ipiv, int* info) {
  int hinfo = 0;
  SGP_SOLVER(c, cusolverDnDgetrf(h, m, m, M, m, work, ipiv, info));
  SGP_CUDA(c, cudaMemcpyAsync(&hinfo, info, sizeof(int), cudaMemcpyDeviceToHost, s));
  SGP_CUDA(c, cudaStreamSynchronize(s));
  if (hinfo > 0) return fail(c, SGP_E_SINGULAR, "matrix is singular (LU pivot " + std::to_string(hinfo) + ")");
  if (hinfo < 0) return fail(c, SGP_E_CUDA, "dgetrf bad argument " + std::to_string(-hinfo));
  if (rhs_vec) SGP_SOLVER(c, cusolverDnDgetrs(h, CUBLAS_OP_N, m, 1, M, m, ipiv, rhs_vec, m, info));
  SGP_CUDA(c, launch_set_identity(inv_out, m, s));
  c->launches += 1;
  SGP_SOLVER(c, cusolverDnDgetrs(h, CUBLAS_OP_N, m, m, M, m, ipiv, inv_out, m, info));
  return SGP_OK;
}

int run_tail(Ctx* c, double* magic_vector, double* magic_matrix) {
  const int m = c->m;
  const size_t mm = static_cast<size_t>(m) * m;
  cudaStream_t s = c->stream, s2 = c->tail_stream;
  double* G = c->dGb.as<double>();
  const double* b = G + mm;
  double* mvec = c->dMagicVec.as<double>();
  double* mmat = c->dMagicMat.as<double>();
  SGP_SOLVER(c, cusolverDnSetStream(c->solver, s));
  SGP_SOLVER(c, cusolverDnSetStream(c->solver2, s2));

  // ---- persistent workspaces -------------------------------------------------------------------------------
  int lw_potrf = 0, lw_eig = 0, lw_lu = 0;
  SGP_SOLVER(c, cusolverDnDpotrf_bufferSize(c->solver, CUBLAS_FILL_MODE_LOWER, m, G, m, &lw_potrf));
  SGP_SOLVER(c, cusolverDnDgetrf_bufferSize(c->solver, m, m, G, m, &lw_lu));
  int lwork = lw_potrf > lw_lu ? lw_potrf : lw_lu;
  // layout of the one scratch block: [Kmm | A | invA | invK | Acopy] (mm doubles each) [work | work2] [ipiv] [info x 4]
  const size_t need = (5 * mm + 2 * static_cast<size_t>(lwork)) * 8 + static_cast<size_t>(m) * sizeof(int) + 64;
  int rc = ctx_scratch(c, c->tail_ws, need);
  if (rc != SGP_OK) return rc;
  double* Kmm = static_cast<double*>(c->tail_ws.p);
  double* A = Kmm + mm;
  double* invA = A + mm;
  double* invK = invA + mm;
  double* Acopy = invK + mm;
  double* work = Acopy + mm;
  double* work2 = work + lwork;
  int* ipiv = reinterpret_cast<int*>(work2 + lwork);
  int* info = ipiv + m;                                               // info[0]: A chain, info[1]: K_mm chain

  const double wn = c->kf.eye_sum;                                   // kernel.whiteNoiseVar

  // K_mm = trainingKernel (PGPH:54) on the main stream; both chains need it
  SGP_CUDA(c, launch_kmm_build(Kmm, c->dZs.as<double>(), c->kf, m, c->m_pad, c->dpad, s));
  SGP_CUDA(c, launch_axpby_diag(A, Kmm, G, wn, m, s));                                                 // PGPH:55-56
  c->launches += 2;
  SGP_CUDA(c, cudaMemcpyAsync(Acopy, A, mm * 8, cudaMemcpyDeviceToDevice, s));     // kept for the slow path
  SGP_CUDA(c, cudaEventRecord(c->tail_fork, s));
  SGP_CUDA(c, cudaStreamWaitEvent(s2, c->tail_fork, 0));

  // ---- chain 2 (second stream): inv(K_mm) by Cholesky ------------------------------------------------------
  SGP_CUDA(c, cudaMemcpyAsync(invA, Kmm, mm * 8, cudaMemcpyDeviceToDevice, s2));   // invA doubles as K_mm's factor buffer
  SGP_SOLVER(c, cusolverDnDpotrf(c->solver2, CUBLAS_FILL_MODE_LOWER, m, invA, m, work2, lwork, info + 1));
  SGP_CUDA(c, launch_set_identity(invK, m, s2));
  SGP_SOLVER(c, cusolverDnDpotrs(c->solver2, CUBLAS_FILL_MODE_LOWER, m, m, invA, m, invK, m, info + 2));
  SGP_CUDA(c, cudaEventRecord(c->tail_join, s2));

  // ---- chain 1 (main stream): Cholesky of A = PD check; magicVector = A \ b -----------------------------------
  SGP_SOLVER(c, cusolverDnDpotrf(c->solver, CUBLAS_FILL_MODE_LOWER, m, A, m, work, lwork, info));
  SGP_CUDA(c, cudaMemcpyAsync(mvec, b, static_cast<size_t>(m) * 8, cudaMemcpyDeviceToDevice, s));
  SGP_SOLVER(c, cusolverDnDpotrs(c->solver, CUBLAS_FILL_MODE_LOWER, m, 1, A, m, mvec, m, info + 3));
  c->launches += 1;
  // inv(A) goes into mmat (finished in place below): invA is still K_mm's factor buffer on the other stream
  SGP_CUDA(c, launch_set_identity(mmat, m, s));
  SGP_SOLVER(c, cusolverDnDpotrs(c->solver, CUBLAS_FILL_MODE_LOWER, m, m, A, m, mmat, m, info + 3));
  c->launches += 1;

  int hinfo[2] = {0, 0};
  SGP_CUDA(c, cudaStreamWaitEvent(s, c->tail_join, 0));
  SGP_CUDA(c, cudaMemcpyAsync(hinfo, info, 2 * sizeof(int), cudaMemcpyDeviceToHost, s));
  SGP_CUDA(c, cudaStreamSynchronize(s));
  if (hinfo[0] < 0 || hinfo[1] < 0) return fail(c, SGP_E_CUDA, "dpotrf bad argument");

  bool a_done = (hinfo[0] == 0), k_done = (hinfo[1] == 0);
  c->tail_fast = a_done && k_done;
  c->has_magic_run = true;
  if (!a_done) {
    // ---- slow path for A: the reference's literal check, then LU ---------------------------------------------
    int lw = 0;
    SGP_SOLVER(c, cusolverDnDsyevd_bufferSize(c->solver, CUSOLVER_EIG_MODE_NOVECTOR, CUBLAS_FILL_MODE_LOWER, m, A, m,
                                              invA, &lw_eig));
    lw = lw_eig > lw_lu ? lw_eig : lw_lu;
    rc = ctx_scratch(c, c->tail_ws2, (static_cast<size_t>(lw) + m) * 8);
    if (rc != SGP_OK) return rc;
    double* wk = static_cast<double*>(c->tail_ws2.p);
    double* W = wk + lw;
    SGP_CUDA(c, cudaMemcpyAsync(A, Acopy, mm * 8, cudaMemcpyDeviceToDevice, s));
    SGP_SOLVER(c, cusolverDnDsyevd(c->solver, CUSOLVER_EIG_MODE_NOVECTOR, CUBLAS_FILL_MODE_LOWER, m, A, m, W, wk, lw, info));
    std::vector<double> ev(m);
    int einfo = 0;
    SGP_CUDA(c, cudaMemcpyAsync(ev.data(), W, static_cast<size_t>(m) * 8, cudaMemcpyDeviceToHost, s));
    SGP_CUDA(c, cudaMemcpyAsync(&einfo, info, sizeof(int), cudaMemcpyDeviceToHost, s));
    SGP_CUDA(c, cudaStreamSynchronize(s));
    if (einfo != 0) return fail(c, SGP_E_CUDA, "dsyevd did not converge, info=" + std::to_string(einfo));
    for (int i = 0; i < m; ++i)
      if (ev[i] < 0.0 || ev[i] != ev[i]) return fail(c, SGP_E_NOT_PD, kNotPdMsg);        // PGPH:62-65
    // semi-definite (or PD only to rounding): carry on with LU like the reference                      PGPH:59
    SGP_CUDA(c, cudaMemcpyAsync(A, Acopy, mm * 8, cudaMemcpyDeviceToDevice, s));
    SGP_CUDA(c, cudaMemcpyAsync(mvec, b, static_cast<size_t>(m) * 8, cudaMemcpyDeviceToDevice, s));
    rc = lu_inverse(c, c->solver, s, m, A, mmat, mvec, wk, ipiv, info);
    if (rc != SGP_OK) return rc;
  }
  if (!k_done) {
    // Cholesky of K_mm broke down (e.g. a kernel without any Eye term on duplicated active points): LU like the reference
    rc = ctx_scratch(c, c->tail_ws2, (static_cast<size_t>(lw_lu) + m) * 8);
    if (rc != SGP_OK) return rc;
    rc = lu_inverse(c, c->solver, s, m, Kmm, invK, nullptr, static_cast<double*>(c->tail_ws2.p), ipiv, info);
    if (rc != SGP_OK) return rc;
  }
  // magicMatrix = inv(A) * whiteNoiseVar - inv(K_mm)                                                    PGPH:59
  SGP_CUDA(c, launch_magic_matrix(mmat, mmat, invK, wn, m, s));
  c->launches += 1;

  if (magic_vector)
    SGP_CUDA(c, cudaMemcpyAsync(magic_vector, mvec, static_cast<size_t>(m) * 8, cudaMemcpyDeviceToHost, s));
  if (magic_matrix) SGP_CUDA(c, cudaMemcpyAsync(magic_matrix, mmat, mm * 8, cudaMemcpyDeviceToHost, s));
  SGP_CUDA(c, cudaStreamSynchronize(s));
  c->has_magic = true;
  c->magic_packed = false;
  return SGP_OK;
}

int predict_prepare(Ctx* c, bool with_var, int n_nodes) {
  if (!with_var) return SGP_OK;                       // the mean-only kernel needs no workspace
  int rc = ctx_scratch(c, c->predict_ws, predict_ws_bytes(predict_window_points(c->m_pad), c->m_pad));
  if (rc == SGP_OK && n_nodes > 0 && n_nodes != c->gh_nodes) {
    // once per context and rule size: a copy, not a launch, so a probability call launches what a variance call does
    std::vector<double> rule(2 * static_cast<size_t>(n_nodes));
    if (!gauss_hermite_rule(n_nodes, rule.data(), rule.data() + n_nodes))
      return fail(c, SGP_E_BADARG, "n_nodes must be in [1, " + std::to_string(kMaxHermiteNodes) + "]");
    rc = ctx_scratch(c, c->dGhRule, 2 * static_cast<size_t>(kMaxHermiteNodes) * sizeof(double));
    if (rc != SGP_OK) return rc;
    c->gh_nodes = 0;
    SGP_CUDA(c, cudaMemcpyAsync(c->dGhRule.p, rule.data(), rule.size() * sizeof(double), cudaMemcpyHostToDevice,
                                c->stream));
    SGP_CUDA(c, cudaStreamSynchronize(c->stream));    // `rule` goes out of scope here
    c->gh_nodes = n_nodes;
  }
  if (rc != SGP_OK || c->magic_packed) return rc;
  rc = ctx_scratch(c, c->dMagicPacked, static_cast<size_t>(c->m_pad) * c->m_pad * sizeof(double));
  if (rc != SGP_OK) return rc;
  SGP_CUDA(c, launch_pack_magic(c->dMagicPacked.as<double>(), c->dMagicMat.as<double>(), c->m, c->m_pad, c->stream));
  c->launches += 1;
  c->magic_packed = true;
  return SGP_OK;
}

int predict_window(Ctx* c, const void* dX, int x_is_f32, long long n, double* dMean, double* dVar, double* dP) {
  PredictArgs a{};
  a.X = dX; a.x_is_f32 = x_is_f32; a.n = n;
  a.d = c->d; a.dpad = c->dpad; a.m = c->m; a.m_pad = c->m_pad;
  a.kf = c->kf;
  a.Zc = c->dZc.as<double>(); a.beta = c->dBeta.as<double>(); a.v = c->dMagicVec.as<double>();
  a.B = c->dMagicPacked.as<double>(); a.ws = c->predict_ws.as<double>();
  a.mean = dMean; a.var = dVar;
  if (dP) {
    a.rule = c->dGhRule.as<double>(); a.n_nodes = c->gh_nodes; a.prob = dP;
  }
  SGP_CUDA(c, launch_predict(a, c->stream));
  c->launches += (dVar || dP) ? 3 : 1;
  return SGP_OK;
}

}  // namespace sgp
