// Feature standardisation (commons/util/Scaling.scala:10-25) on device-resident rows: the fixed-order column sums of
// sgp_column_sums_device and the element-wise (x - mean) / sd of sgp_scale_apply_device.  Both passes are HBM-bound.
//
// Thread layout of both kernels: a CTA takes kScaleRows consecutive rows (one row block).  Its threads cover cw =
// min(d, kScaleThreads) adjacent columns and L = kScaleThreads / cw row lanes: thread t reads column c0 + t % cw of the
// rows lane, lane + L, ... with lane = t / cw, so one step of the CTA reads L * cw consecutive elements (coalesced for
// any d, d = 16 and d = 32 included).  Columns beyond kScaleThreads are taken in chunks of cw.
//
// Sum order (column_sums_kernel + column_fold_kernel): each thread sums its rows of the block in row order, the L lane
// sums of a column are added in lane order, and the blocks' partials are added in block order.  L and the blocks depend
// on d and n alone, never on the grid or on how many CTAs run at once, so the same inputs give the same bits.
#include "sgp_internal.h"

namespace sgp {
namespace {

constexpr int kScaleThreads = 256;
constexpr int kFoldCols = 32;      // columns of one fold CTA
constexpr int kFoldBlocks = 128;   // row blocks a fold CTA stages in shared memory at a time (32 KiB)
constexpr int kUnroll = 16;        // loads a thread has in flight

struct Lanes {
  int cw, L, lane, k;              // columns per chunk, row lanes, this thread's lane and column within the chunk
  __device__ explicit Lanes(int d) {
    cw = d < kScaleThreads ? d : kScaleThreads;
    L = kScaleThreads / cw;
    lane = threadIdx.x / cw;
    k = threadIdx.x % cw;
  }
  __device__ bool active(int c0, int d) const { return lane < L && c0 + k < d; }
};

// v as the sum's term: x, or (x - c)^2 with x converted exactly to fp64 and each operation rounded once (no fma, so
// that every term is the reference formula's centred square)
__device__ __forceinline__ double term(double x, bool centred, double c) {
  if (!centred) return x;
  const double t = __dsub_rn(x, c);
  return __dmul_rn(t, t);
}

// part[b][k]: the sum over row block b of column k's terms
template <class T>
__global__ void __launch_bounds__(kScaleThreads) column_sums_kernel(const T* __restrict__ X, long long n, int d,
                                                                    const double* __restrict__ centre,
                                                                    double* __restrict__ part) {
  __shared__ double lane_sum[kScaleThreads];
  const Lanes g(d);
  const long long r0 = static_cast<long long>(blockIdx.x) * kScaleRows;
  const long long r1 = r0 + kScaleRows < n ? r0 + kScaleRows : n;
  const long long step = g.L;
  for (int c0 = 0; c0 < d; c0 += g.cw) {
    const int col = c0 + g.k;
    if (g.active(c0, d)) {
      const bool centred = centre != nullptr;
      const double c = centred ? centre[col] : 0.0;
      const T* x = X + col;
      double acc = 0.0;
      long long r = r0 + g.lane;
      for (; r + (kUnroll - 1) * step < r1; r += kUnroll * step) {
        T v[kUnroll];
#pragma unroll
        for (int u = 0; u < kUnroll; ++u) v[u] = x[(r + u * step) * d];
#pragma unroll
        for (int u = 0; u < kUnroll; ++u) acc = __dadd_rn(acc, term(static_cast<double>(v[u]), centred, c));
      }
      for (; r < r1; r += step) acc = __dadd_rn(acc, term(static_cast<double>(x[r * d]), centred, c));
      lane_sum[threadIdx.x] = acc;
    }
    __syncthreads();
    if (g.lane == 0 && col < d) {
      double s = lane_sum[g.k];
      for (int l = 1; l < g.L; ++l) s = __dadd_rn(s, lane_sum[l * g.cw + g.k]);
      part[static_cast<size_t>(blockIdx.x) * d + col] = s;
    }
    __syncthreads();
  }
}

// out[k] = part[0][k] + part[1][k] + ... + part[blocks - 1][k], added in block order.  CTA j takes the columns
// [32 j, 32 j + 32); the CTA stages kFoldBlocks partials of its columns at a time, so that one thread per column adds
// them from shared memory instead of waiting for one global load per block.
__global__ void __launch_bounds__(kScaleThreads) column_fold_kernel(const double* __restrict__ part, long long blocks,
                                                                    int d, double* __restrict__ out) {
  __shared__ double tile[kFoldBlocks][kFoldCols];
  const int c0 = blockIdx.x * kFoldCols;
  const int j = threadIdx.x % kFoldCols, b_lane = threadIdx.x / kFoldCols;
  constexpr int kLanes = kScaleThreads / kFoldCols;
  double s = 0.0;
  for (long long b0 = 0; b0 < blocks; b0 += kFoldBlocks) {
    const int nb = blocks - b0 < kFoldBlocks ? static_cast<int>(blocks - b0) : kFoldBlocks;
    for (int b = b_lane; b < nb; b += kLanes)
      tile[b][j] = c0 + j < d ? part[static_cast<size_t>(b0 + b) * d + c0 + j] : 0.0;
    __syncthreads();
    if (threadIdx.x < kFoldCols)
      for (int b = 0; b < nb; ++b) s = __dadd_rn(s, tile[b][j]);
    __syncthreads();
  }
  if (threadIdx.x < kFoldCols && c0 + j < d) out[c0 + j] = s;
}

// Y[i][k] = (x_ik - mean_k) / sd_k in fp64: a correctly rounded subtraction, then a correctly rounded division
template <class T>
__global__ void __launch_bounds__(kScaleThreads) scale_apply_kernel(const T* __restrict__ X, long long n, int d,
                                                                    const double* __restrict__ mean,
                                                                    const double* __restrict__ sd,
                                                                    double* __restrict__ Y) {
  const Lanes g(d);
  const long long r0 = static_cast<long long>(blockIdx.x) * kScaleRows;
  const long long r1 = r0 + kScaleRows < n ? r0 + kScaleRows : n;
  const long long step = g.L;
  for (int c0 = 0; c0 < d; c0 += g.cw) {
    if (!g.active(c0, d)) continue;
    const int col = c0 + g.k;
    const double mu = mean[col], s = sd[col];
    const T* x = X + col;
    double* y = Y + col;
    long long r = r0 + g.lane;
    for (; r + (kUnroll - 1) * step < r1; r += kUnroll * step) {
      T v[kUnroll];
#pragma unroll
      for (int u = 0; u < kUnroll; ++u) v[u] = x[(r + u * step) * d];
#pragma unroll
      for (int u = 0; u < kUnroll; ++u)
        y[(r + u * step) * d] = __ddiv_rn(__dsub_rn(static_cast<double>(v[u]), mu), s);
    }
    for (; r < r1; r += step) y[r * d] = __ddiv_rn(__dsub_rn(static_cast<double>(x[r * d]), mu), s);
  }
}

}  // namespace

long long scale_row_blocks(long long n) { return (n + kScaleRows - 1) / kScaleRows; }

cudaError_t launch_column_sums(const void* X, int x_is_f32, long long n, int d, const double* centre, double* part,
                               double* out, cudaStream_t s) {
  const long long blocks = scale_row_blocks(n);
  if (x_is_f32)
    column_sums_kernel<float><<<static_cast<unsigned>(blocks), kScaleThreads, 0, s>>>(static_cast<const float*>(X), n, d,
                                                                                     centre, part);
  else
    column_sums_kernel<double><<<static_cast<unsigned>(blocks), kScaleThreads, 0, s>>>(static_cast<const double*>(X), n,
                                                                                      d, centre, part);
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) return e;
  column_fold_kernel<<<(d + kFoldCols - 1) / kFoldCols, kScaleThreads, 0, s>>>(part, blocks, d, out);
  return cudaGetLastError();
}

cudaError_t launch_scale_apply(const void* X, int x_is_f32, long long n, int d, const double* mean, const double* sd,
                               double* Y, cudaStream_t s) {
  const unsigned blocks = static_cast<unsigned>(scale_row_blocks(n));
  if (x_is_f32)
    scale_apply_kernel<float><<<blocks, kScaleThreads, 0, s>>>(static_cast<const float*>(X), n, d, mean, sd, Y);
  else
    scale_apply_kernel<double><<<blocks, kScaleThreads, 0, s>>>(static_cast<const double*>(X), n, d, mean, sd, Y);
  return cudaGetLastError();
}

}  // namespace sgp
