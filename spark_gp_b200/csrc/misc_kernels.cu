// Small fp64 kernels around the hot path: active-set pre-scaling, K_mm (trainingKernel), the dense
// cross kernel K(X*, Z) of sgp_cross_kernel (golden-vector tests, greedy cross-check), and element-wise pieces of
// the m x m tail.  All of these are O(m^2) or O(n_test * m) -- negligible next to the Gram kernel.
#include "sgp_internal.h"

namespace sgp {
namespace {

// out[r][k] = (r < rows_in && k < d) ? in[r][k] * beta[k] : 0      (out is rows_out x dpad)
// out_centred[r][k] (optional): the same with (in[r][k] - centre[k]) * beta[k]
__global__ void scale_rows_kernel(double* __restrict__ out, double* __restrict__ out_centred,
                                  const double* __restrict__ in, const double* __restrict__ beta,
                                  const double* __restrict__ centre, int rows_in, int rows_out, int d, int dpad) {
  const size_t idx = blockIdx.x * static_cast<size_t>(blockDim.x) + threadIdx.x;
  if (idx >= static_cast<size_t>(rows_out) * dpad) return;
  const int r = static_cast<int>(idx / dpad), k = static_cast<int>(idx % dpad);
  const bool in_range = r < rows_in && k < d;
  const double v = in_range ? in[static_cast<size_t>(r) * d + k] : 0.0;
  out[idx] = in_range ? v * beta[k] : 0.0;
  if (out_centred) out_centred[idx] = in_range ? (v - centre[k]) * beta[k] : 0.0;
}

// K_mm[i][j] = sum_t C_t exp(-|z~_ti - z~_tj|^2) + (i==j) * eye_sum        kernel/Kernel.scala:151,
// kernel/ARDRBFKernel.scala:48-59, kernel/SumOfKernels.scala:45
__global__ void kmm_build_kernel(double* __restrict__ Kmm, const double* __restrict__ Zs, const KernelFlat kf, int m,
                                 int m_pad, int dpad) {
  const int j = blockIdx.x * blockDim.x + threadIdx.x;
  const int i = blockIdx.y * blockDim.y + threadIdx.y;
  if (i >= m || j >= m) return;
  double v = 0.0;
  for (int t = 0; t < kf.n_terms; ++t) {
    const double* zi = Zs + (static_cast<size_t>(t) * m_pad + i) * dpad;
    const double* zj = Zs + (static_cast<size_t>(t) * m_pad + j) * dpad;
    double q = 0.0;
    for (int k = 0; k < dpad; ++k) {
      const double df = zi[k] - zj[k];
      q = fma(df, df, q);
    }
    v = kf.fold_term(v, t, q);
  }
  if (i == j) v += kf.eye_sum;
  Kmm[static_cast<size_t>(i) * m + j] = v;
}

// K[r][j] = sum_t C_t exp(-sum_k ((x_rk * beta_tk) - z~_tjk)^2)        kernel/Kernel.scala:69-74 contract:
// rows = test vectors, cols = training (here: active-set) vectors.  Eye terms add nothing (Kernel.scala:157).
__global__ void cross_kernel_kernel(double* __restrict__ K, const double* __restrict__ X,
                                    const double* __restrict__ Zs, const double* __restrict__ beta, const KernelFlat kf,
                                    long long n, int d, int dpad, int m, int m_pad) {
  const int j = blockIdx.x * blockDim.x + threadIdx.x;
  const long long r = blockIdx.y * static_cast<long long>(blockDim.y) + threadIdx.y;
  if (r >= n || j >= m) return;
  double v = 0.0;
  for (int t = 0; t < kf.n_terms; ++t) {
    const double* zj = Zs + (static_cast<size_t>(t) * m_pad + j) * dpad;
    const double* bt = beta + t * dpad;
    const double* xr = X + static_cast<size_t>(r) * d;
    double q = 0.0;
    for (int k = 0; k < d; ++k) {
      const double df = xr[k] * bt[k] - zj[k];
      q = fma(df, df, q);
    }
    v = kf.fold_term(v, t, q);
  }
  K[static_cast<size_t>(r) * m + j] = v;
}

__global__ void axpby_kernel(double* __restrict__ A, const double* __restrict__ K, const double* __restrict__ G,
                             double wn, size_t n) {
  const size_t i = blockIdx.x * static_cast<size_t>(blockDim.x) + threadIdx.x;
  if (i < n) A[i] = wn * K[i] + G[i];     // PGPH:55-56
}

__global__ void identity_kernel(double* __restrict__ I, int m) {
  const size_t i = blockIdx.x * static_cast<size_t>(blockDim.x) + threadIdx.x;
  if (i < static_cast<size_t>(m) * m) I[i] = (i / m == i % m) ? 1.0 : 0.0;
}

// (out may alias invA: run_tail finishes inv(A) in place)
__global__ void magic_matrix_kernel(double* out, const double* invA, const double* __restrict__ invK, double wn,
                                    size_t n) {
  const size_t i = blockIdx.x * static_cast<size_t>(blockDim.x) + threadIdx.x;
  if (i < n) out[i] = invA[i] * wn - invK[i];   // PGPH:59
}

// status words that must be agreed on by every rank travel inside the all-reduced buffers as doubles
__global__ void status_to_double_kernel(double* __restrict__ dst, const int* __restrict__ flags, int mask,
                                        const double* __restrict__ norm_sum, double norm_limit) {
  double v = (flags && (*flags & mask)) ? 1.0 : 0.0;
  if (norm_sum && *norm_sum > norm_limit) v += 2.0;
  *dst = v;
}

__global__ void flags_to_double_kernel(double* __restrict__ dst, const int* __restrict__ flags, int mask, int n) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) dst[i] = (flags[i] & mask) ? 1.0 : 0.0;
}

// Expert grouping on the device (GPC:26-31): E = Math.round(N / n_e); point i (zipWithIndex order) belongs to expert
// i % E and is its (i / E)-th point.  With k = N / E and r = N % E, experts < r own k+1 points: expert e starts at
// e*k + min(e, r).  One thread per (point, feature): a strided gather from the row-major input into the expert-major
// fp64 layout the objective kernels read.
// A fold's training set (sgp_experts_upload_folds) leaves out the points listed in skip_pos (sorted): point i is then the
// training set's point i - (left-out points before i), found by a binary search over skip_pos.  Each of a point's d
// threads runs the same search; the threads of a warp read the same entries.
__global__ void group_experts_kernel(double* __restrict__ Xe, double* __restrict__ ye, const void* __restrict__ X,
                                     int x_is_f32, const double* __restrict__ y, long long n, int d, long long E,
                                     long long p0, long long cn, const long long* __restrict__ skip_pos,
                                     long long n_skip) {
  const long long idx = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x;
  if (idx >= cn * d) return;
  const long long li = idx / d;                 // point inside this chunk
  const int k = static_cast<int>(idx % d);
  long long i = p0 + li;                        // global point index, then its training rank
  if (skip_pos) {
    long long lo = 0, hi = n_skip;              // lo = number of left-out points before i
    while (lo < hi) {
      const long long mid = (lo + hi) >> 1;
      if (skip_pos[mid] < i) lo = mid + 1; else hi = mid;
    }
    if (lo < n_skip && skip_pos[lo] == i) return;
    i -= lo;
  }
  const long long e = i % E, pos = i / E;
  const long long kq = n / E, r = n % E;
  const long long dst = e * kq + (e < r ? e : r) + pos;
  const double v = x_is_f32 ? static_cast<double>(static_cast<const float*>(X)[li * d + k])
                            : static_cast<const double*>(X)[li * d + k];
  Xe[dst * d + k] = v;
  if (k == 0) ye[dst] = y[li];
}

// One thread per point: the inverse of group_experts_kernel's permutation (without skipped points).
__global__ void ungroup_experts_kernel(double* __restrict__ out, const double* __restrict__ f, long long n, long long E) {
  const long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x;
  if (i >= n) return;
  const long long e = i % E, pos = i / E;
  const long long kq = n / E, r = n % E;
  out[i] = f[e * kq + (e < r ? e : r) + pos];
}

__global__ void expert_offsets_kernel(long long* __restrict__ off, long long n, long long E, long long base) {
  const long long e = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x;
  if (e > E) return;
  const long long kq = n / E, r = n % E;
  off[e] = base + e * kq + (e < r ? e : r);
}

}  // namespace

cudaError_t launch_scale_rows(double* out, double* out_centred, const double* in, const double* beta, const double* centre,
                              int rows_in, int rows_out, int d, int dpad, cudaStream_t s) {
  const size_t n = static_cast<size_t>(rows_out) * dpad;
  scale_rows_kernel<<<static_cast<unsigned>((n + 255) / 256), 256, 0, s>>>(out, out_centred, in, beta, centre, rows_in,
                                                                            rows_out, d, dpad);
  return cudaGetLastError();
}

cudaError_t launch_kmm_build(double* Kmm, const double* Zs, const KernelFlat& kf, int m, int m_pad, int dpad,
                             cudaStream_t s) {
  dim3 block(32, 8), grid((m + 31) / 32, (m + 7) / 8);
  kmm_build_kernel<<<grid, block, 0, s>>>(Kmm, Zs, kf, m, m_pad, dpad);
  return cudaGetLastError();
}

cudaError_t launch_cross_kernel(double* K, const double* X, const double* Zs, const double* beta,
                                const KernelFlat& kf, long long n, int d, int dpad, int m, int m_pad,
                                cudaStream_t s) {
  dim3 block(32, 8), grid((m + 31) / 32, static_cast<unsigned>((n + 7) / 8));
  cross_kernel_kernel<<<grid, block, 0, s>>>(K, X, Zs, beta, kf, n, d, dpad, m, m_pad);
  return cudaGetLastError();
}

cudaError_t launch_axpby_diag(double* A, const double* K, const double* G, double wn, int m, cudaStream_t s) {
  const size_t n = static_cast<size_t>(m) * m;
  axpby_kernel<<<static_cast<unsigned>((n + 255) / 256), 256, 0, s>>>(A, K, G, wn, n);
  return cudaGetLastError();
}

cudaError_t launch_set_identity(double* I, int m, cudaStream_t s) {
  const size_t n = static_cast<size_t>(m) * m;
  identity_kernel<<<static_cast<unsigned>((n + 255) / 256), 256, 0, s>>>(I, m);
  return cudaGetLastError();
}

cudaError_t launch_magic_matrix(double* out, const double* invA, const double* invK, double wn, int m,
                                cudaStream_t s) {
  const size_t n = static_cast<size_t>(m) * m;
  magic_matrix_kernel<<<static_cast<unsigned>((n + 255) / 256), 256, 0, s>>>(out, invA, invK, wn, n);
  return cudaGetLastError();
}

cudaError_t launch_group_experts(double* Xe, double* ye, const void* dX, int x_is_f32, const double* dy, long long n, int d,
                                 long long E, long long p0, long long cn, const long long* skip_pos, long long n_skip,
                                 cudaStream_t s) {
  const long long total = cn * d;
  group_experts_kernel<<<static_cast<unsigned>((total + 255) / 256), 256, 0, s>>>(Xe, ye, dX, x_is_f32, dy, n, d, E, p0, cn,
                                                                                  skip_pos, n_skip);
  return cudaGetLastError();
}

cudaError_t launch_ungroup_experts(double* out, const double* f, long long n, long long E, cudaStream_t s) {
  ungroup_experts_kernel<<<static_cast<unsigned>((n + 255) / 256), 256, 0, s>>>(out, f, n, E);
  return cudaGetLastError();
}

cudaError_t launch_expert_offsets(long long* off, long long n, long long E, long long base, cudaStream_t s) {
  expert_offsets_kernel<<<static_cast<unsigned>((E + 1 + 255) / 256), 256, 0, s>>>(off, n, E, base);
  return cudaGetLastError();
}

cudaError_t launch_status_to_double(double* dst, const int* flags, int mask, const double* norm_sum, double norm_limit,
                                    cudaStream_t s) {
  status_to_double_kernel<<<1, 1, 0, s>>>(dst, flags, mask, norm_sum, norm_limit);
  return cudaGetLastError();
}

cudaError_t launch_flags_to_double(double* dst, const int* flags, int mask, int n, cudaStream_t s) {
  flags_to_double_kernel<<<(n + 255) / 256, 256, 0, s>>>(dst, flags, mask, n);
  return cudaGetLastError();
}

}  // namespace sgp
