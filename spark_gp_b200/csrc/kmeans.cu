// KMeansActiveSetProvider (commons/ActiveSetProvider.scala:22-46): Spark 3.1 MLlib KMeans with the reference's settings --
// k-means|| seeding (2 steps), a local weighted k-means++ over the distinct candidates, then Lloyd iterations that keep the
// centre of an empty cluster and stop on an absolute centre-movement rule (DESIGN.md 4.7 restates the algorithm).
//   * assignment (the hot path): point-stationary fp32 direct-form distances on the CUDA cores.  Each thread holds its
//     point's coordinates in registers (chunks of DCH for large d), centre tiles are staged in shared memory, a running
//     min / argmin keeps the lowest index on ties.  Points and centres are shifted by a common origin o and scaled by a
//     common power of two 2^s in fp64 BEFORE the fp32 rounding, so the accuracy does not depend on the data's distance
//     from the origin, and fp32 neither underflows nor overflows at the data's scale; distances are returned times 2^-2s
//     (exact).
//   * centre update: fp64 sums over the points as given, in point-index order (stable radix sort of the labels, one warp
//     per cluster), no floating-point atomics: the result does not depend on scheduling.
//   * every fp64 reduction the algorithm branches on (the k-means|| cost sum, the k-means++ walk) has a fixed order.
#include <cub/cub.cuh>

#include <algorithm>
#include <cmath>
#include <cstring>
#include <string>
#include <unordered_set>
#include <vector>

#include "sgp_internal.h"

namespace sgp {
namespace {

// The counter-based generator shared with the NumPy restatement of the algorithm: splitmix64's finaliser, chained over
// (seed, stream, i).  Streams: 0 first centre, 1 + s k-means|| step s, 100 local k-means++, 101 local empty clusters.
__host__ __device__ inline uint64_t km_mix(uint64_t z) {
  z += 0x9E3779B97F4A7C15ULL;
  z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9ULL;
  z = (z ^ (z >> 27)) * 0x94D049BB133111EBULL;
  return z ^ (z >> 31);
}
__host__ __device__ inline double km_u(uint64_t seed, uint64_t stream, uint64_t i) {
  return static_cast<double>(km_mix(km_mix(km_mix(seed) ^ stream) ^ i) >> 11) * 0x1.0p-53;
}

constexpr int kAssignThreads = 128;
constexpr int kRowPad = 64;          // centre rows of the fp32 image are padded to a multiple of the largest tile
constexpr int kSumBlocks = 264;      // fixed grid of the fixed-order reductions (2 x 132 SMs)

int dchunk(int d) { return d <= 4 ? 4 : d <= 8 ? 8 : d <= 16 ? 16 : 32; }
int cstride(int d) { const int c = dchunk(d); return (d + c - 1) / c * c; }
int rows_pad(int k) { return (k + kRowPad - 1) / kRowPad * kRowPad; }

// label[i] / dist[i] = argmin / min over the k centres of |x_i - c|^2 (fp32 on the images (x - o) scale, lowest index
// on ties; dist = min inv2 with inv2 = scale^-2); min_into: dist[i] = min(dist[i], min inv2) and no label (the k-means||
// running cost); changed (optional) is set when a label differs from the one already in label[]; *range is set when a
// point's nearest distance is not finite.  Cf: [rows_pad(k)][cstride(d)] fp32 images (c - o) scale, zero padded.
template <typename T, int DCH, int TC>
__global__ void __launch_bounds__(kAssignThreads) kmeans_assign_kernel(const T* __restrict__ X, int n, int d,
                                                                       const double* __restrict__ o, double scale,
                                                                       double inv2, const float* __restrict__ Cf, int k,
                                                                       int cs, int* __restrict__ label,
                                                                       double* __restrict__ dist, int min_into,
                                                                       int* __restrict__ changed, int* __restrict__ range) {
  __shared__ __align__(16) float sc[TC][DCH];
  const int i = blockIdx.x * kAssignThreads + threadIdx.x;
  const bool live = i < n;
  const int nch = (d + DCH - 1) / DCH;
  float xs[DCH];
  auto load_x = [&](int ch) {
#pragma unroll
    for (int kk = 0; kk < DCH; ++kk) {
      const int j = ch * DCH + kk;
      xs[kk] = (live && j < d)
                   ? static_cast<float>((static_cast<double>(X[static_cast<size_t>(i) * d + j]) - o[j]) * scale)
                   : 0.f;
    }
  };
  if (nch == 1) load_x(0);
  float best = INFINITY;
  int bi = 0;
  for (int c0 = 0; c0 < k; c0 += TC) {
    float acc[TC];
#pragma unroll
    for (int c = 0; c < TC; ++c) acc[c] = 0.f;
    for (int ch = 0; ch < nch; ++ch) {
      __syncthreads();
      for (int e = threadIdx.x; e < TC * DCH; e += kAssignThreads) {
        const int c = e / DCH, kk = e % DCH;
        sc[c][kk] = Cf[static_cast<size_t>(c0 + c) * cs + ch * DCH + kk];
      }
      __syncthreads();
      if (nch > 1) load_x(ch);
#pragma unroll
      for (int c = 0; c < TC; ++c) {
#pragma unroll
        for (int kk = 0; kk < DCH; kk += 4) {
          const float4 v = *reinterpret_cast<const float4*>(&sc[c][kk]);
          const float a = xs[kk] - v.x, b = xs[kk + 1] - v.y, e = xs[kk + 2] - v.z, f = xs[kk + 3] - v.w;
          acc[c] = fmaf(a, a, acc[c]);
          acc[c] = fmaf(b, b, acc[c]);
          acc[c] = fmaf(e, e, acc[c]);
          acc[c] = fmaf(f, f, acc[c]);
        }
      }
    }
#pragma unroll
    for (int c = 0; c < TC; ++c)
      if (c0 + c < k && acc[c] < best) { best = acc[c]; bi = c0 + c; }
  }
  if (!live) return;
  if (!(best < INFINITY)) *range = 1;
  if (min_into) {
    dist[i] = fmin(dist[i], static_cast<double>(best) * inv2);
    return;
  }
  if (changed && label[i] != bi) *changed = 1;
  label[i] = bi;
  dist[i] = static_cast<double>(best) * inv2;
}

// the data's frame for the fp32 distances: origin o (device, d entries) and the prescale sc = 2^s, inv2 = 2^-2s
struct Frame {
  const double* o;
  double sc, inv2;
  int* range;
};

template <typename T>
cudaError_t launch_assign(const T* X, int n, int d, const Frame& f, const float* Cf, int k, int* label, double* dist,
                          int min_into, int* changed, cudaStream_t s) {
  const unsigned grid = static_cast<unsigned>((n + kAssignThreads - 1) / kAssignThreads);
  const int cs = cstride(d);
#define SGP_KM_ASSIGN(DCH, TC)                                                                                             \
  kmeans_assign_kernel<T, DCH, TC><<<grid, kAssignThreads, 0, s>>>(X, n, d, f.o, f.sc, f.inv2, Cf, k, cs, label, dist,  \
                                                                   min_into, changed, f.range)
  switch (dchunk(d)) {
    case 4: SGP_KM_ASSIGN(4, 64); break;
    case 8: SGP_KM_ASSIGN(8, 64); break;
    case 16: SGP_KM_ASSIGN(16, 64); break;
    default: SGP_KM_ASSIGN(32, 32); break;
  }
#undef SGP_KM_ASSIGN
  return cudaGetLastError();
}

// Cf[r][j] = fp32((C[r][j] - o[j]) sc) for r < k, j < d; zero elsewhere in [rows_pad(k)][cstride(d)]
__global__ void kmeans_centre_f32_kernel(const double* __restrict__ Cc, int k, int d, const double* __restrict__ o,
                                         double sc, float* __restrict__ Cf, int rows, int cs) {
  const long long e = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x;
  if (e >= static_cast<long long>(rows) * cs) return;
  const int r = static_cast<int>(e / cs), j = static_cast<int>(e % cs);
  Cf[e] = (r < k && j < d) ? static_cast<float>((Cc[static_cast<size_t>(r) * d + j] - o[j]) * sc) : 0.f;
}

// per-slice column sums and sums of squares (fixed order: 8 row lanes x 32 column lanes, lanes folded in order); any
// non-finite coordinate sets *bad
template <typename T>
__global__ void __launch_bounds__(256) kmeans_colstats_kernel(const T* __restrict__ X, int n, int d, int rows_per_slice,
                                                              double* __restrict__ part /*[slices][2][d]*/, int* bad) {
  __shared__ double s1[8][32], s2[8][32];
  const int cl = threadIdx.x & 31, rl = threadIdx.x >> 5;
  const long long r0 = static_cast<long long>(blockIdx.x) * rows_per_slice;
  const long long r1 = min(static_cast<long long>(n), r0 + rows_per_slice);
  for (int c0 = 0; c0 < d; c0 += 32) {
    const int c = c0 + cl;
    double a = 0.0, b = 0.0;
    if (c < d)
      for (long long r = r0 + rl; r < r1; r += 8) {
        const double v = static_cast<double>(X[static_cast<size_t>(r) * d + c]);
        if (!isfinite(v)) *bad = 1;
        a += v;
        b = fma(v, v, b);
      }
    s1[rl][cl] = a; s2[rl][cl] = b;
    __syncthreads();
    if (rl == 0 && c < d) {
      double ta = 0.0, tb = 0.0;
      for (int q = 0; q < 8; ++q) { ta += s1[q][cl]; tb += s2[q][cl]; }
      part[static_cast<size_t>(blockIdx.x) * 2 * d + c] = ta;
      part[static_cast<size_t>(blockIdx.x) * 2 * d + d + c] = tb;
    }
    __syncthreads();
  }
}

// part[b] = sum of v over block b's fixed range, fixed tree order
__global__ void __launch_bounds__(256) kmeans_sum_kernel(const double* __restrict__ v, int n, int per,
                                                         double* __restrict__ part) {
  __shared__ double sh[256];
  const long long b0 = static_cast<long long>(blockIdx.x) * per;
  const long long b1 = min(static_cast<long long>(n), b0 + per);
  double a = 0.0;
  for (long long i = b0 + threadIdx.x; i < b1; i += 256) a += v[i];
  sh[threadIdx.x] = a;
  __syncthreads();
  for (int s = 128; s > 0; s >>= 1) {
    if (threadIdx.x < s) sh[threadIdx.x] += sh[threadIdx.x + s];
    __syncthreads();
  }
  if (threadIdx.x == 0) part[blockIdx.x] = sh[0];
}

// k-means|| step: point i (global row i0 + i) is chosen iff u(seed, stream, i0 + i) < (2k cost_i) / S (a NaN threshold
// chooses nothing)
__global__ void kmeans_sample_kernel(const double* __restrict__ cost, int n, long long i0, double two_k, double S,
                                     uint64_t seed, uint64_t stream, unsigned char* __restrict__ flag) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  flag[i] = km_u(seed, stream, static_cast<uint64_t>(i0 + i)) < (two_k * cost[i]) / S ? 1 : 0;
}

__global__ void kmeans_fill_kernel(double* __restrict__ v, int n, double x) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) v[i] = x;
}

__global__ void kmeans_iota_kernel(int* __restrict__ v, int n, int start) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) v[i] = start < 0 ? start : i;
}

// integer histogram of the labels (integer atomics: the counts do not depend on the order)
__global__ void kmeans_count_kernel(const int* __restrict__ label, int n, int* __restrict__ cnt) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) atomicAdd(cnt + label[i], 1);
}

__global__ void kmeans_to_double_kernel(const int* __restrict__ cnt, int m, double* __restrict__ w) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < m) w[i] = static_cast<double>(cnt[i]);
}

// [beg, end) of every label in the sorted labels (beg = end = 0 for an absent label: memset before)
__global__ void kmeans_bounds_kernel(const int* __restrict__ keys, int n, int* __restrict__ beg, int* __restrict__ end) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const int kk = keys[i];
  if (i == 0 || keys[i - 1] != kk) beg[kk] = i;
  if (i == n - 1 || keys[i + 1] != kk) end[kk] = i + 1;
}

// One warp per cluster j: the (weighted) sum of its members in point-index order (order[] = indices sorted stably by
// label), sum * (1 / weight) as Spark's centroid.  A cluster of zero weight keeps its centre; wsum[j] records the weight.
// *notconv is set when a moved cluster moved by more than tol2 (squared distance).
template <typename T>
__global__ void __launch_bounds__(256) kmeans_update_kernel(const T* __restrict__ X, int d, const int* __restrict__ order,
                                                            const int* __restrict__ beg, const int* __restrict__ end,
                                                            const double* __restrict__ w, int k, double* __restrict__ Cc,
                                                            double* __restrict__ wsum, double tol2, int* notconv) {
  const int j = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
  if (j >= k) return;
  const int b = beg[j], e = end[j];
  double ws = static_cast<double>(e - b);
  if (w) {
    ws = 0.0;
    for (int m = b; m < e; ++m) ws += w[order[m]];
  }
  if (lane == 0) wsum[j] = ws;
  if (ws == 0.0) return;
  const double inv = 1.0 / ws;
  double moved = 0.0;
  for (int c = lane; c < d; c += 32) {
    double s = 0.0;
#pragma unroll 4
    for (int m = b; m < e; ++m) {
      const int p = order[m];
      const double x = static_cast<double>(X[static_cast<size_t>(p) * d + c]);
      s = __dadd_rn(s, w ? __dmul_rn(w[p], x) : x);
    }
    const double nc = __dmul_rn(s, inv);
    const double df = nc - Cc[static_cast<size_t>(j) * d + c];
    moved = fma(df, df, moved);
    Cc[static_cast<size_t>(j) * d + c] = nc;
  }
  for (int off = 16; off > 0; off >>= 1) moved += __shfl_down_sync(0xffffffffu, moved, off);
  if (lane == 0 && notconv && !(moved <= tol2)) *notconv = 1;
}

// The sharded Lloyd step's two halves, split at the all-reduce.  kmeans_sums_kernel: one warp per cluster j sums its
// members on this rank in point-index order, exactly as kmeans_update_kernel without weights does, and counts them.
template <typename T>
__global__ void __launch_bounds__(256) kmeans_sums_kernel(const T* __restrict__ X, int d, const int* __restrict__ order,
                                                          const int* __restrict__ beg, const int* __restrict__ end, int k,
                                                          double* __restrict__ sums, long long* __restrict__ cnt) {
  const int j = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
  if (j >= k) return;
  const int b = beg[j], e = end[j];
  if (lane == 0) cnt[j] = e - b;
  for (int c = lane; c < d; c += 32) {
    double s = 0.0;
#pragma unroll 4
    for (int m = b; m < e; ++m) s = __dadd_rn(s, static_cast<double>(X[static_cast<size_t>(order[m]) * d + c]));
    sums[static_cast<size_t>(j) * d + c] = s;
  }
}

// kmeans_centre_kernel: the summed clusters' centres, sum * (1 / count), and the moved flag, with kmeans_update_kernel's
// arithmetic; an empty cluster keeps its centre.
__global__ void __launch_bounds__(256) kmeans_centre_kernel(const double* __restrict__ sums,
                                                            const long long* __restrict__ cnt, int k, int d,
                                                            double* __restrict__ Cc, double tol2, int* notconv) {
  const int j = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
  if (j >= k) return;
  const double ws = static_cast<double>(cnt[j]);
  if (ws == 0.0) return;
  const double inv = 1.0 / ws;
  double moved = 0.0;
  for (int c = lane; c < d; c += 32) {
    const double nc = __dmul_rn(sums[static_cast<size_t>(j) * d + c], inv);
    const double df = nc - Cc[static_cast<size_t>(j) * d + c];
    moved = fma(df, df, moved);
    Cc[static_cast<size_t>(j) * d + c] = nc;
  }
  for (int off = 16; off > 0; off >>= 1) moved += __shfl_down_sync(0xffffffffu, moved, off);
  if (lane == 0 && !(moved <= tol2)) *notconv = 1;
}

// local k-means++ (LocalKMeans.kMeansPlusPlus): a cluster of zero weight gets cand[floor(u * C)], u from stream 101 with a
// draw counter that persists across iterations.  One thread: at most k draws.
__global__ void kmeans_local_empty_kernel(const double* __restrict__ wsum, int k, const double* __restrict__ cand, int C,
                                          int d, double* __restrict__ Cc, uint64_t seed, int* counter) {
  int ctr = *counter;
  for (int j = 0; j < k; ++j) {
    if (wsum[j] != 0.0) continue;
    const int p = min(C - 1, static_cast<int>(floor(km_u(seed, 101, static_cast<uint64_t>(ctr++)) * C)));
    for (int e = 0; e < d; ++e) Cc[static_cast<size_t>(j) * d + e] = cand[static_cast<size_t>(p) * d + e];
  }
  *counter = ctr;
}

// The sequential k-means++ seeding over the C weighted candidates (LocalKMeans.kMeansPlusPlus), one persistent CTA: for
// each centre a fixed-order block scan of w_j (first centre) or w_j cost_j, the walk "cum += v_j while cum < r" as a
// search for the first prefix >= r, then cost_j = min(cost_j, |cand_j - centre|^2) in fp64.  Writes the k centres to Cc.
constexpr int kPPThreads = 1024;
__global__ void __launch_bounds__(kPPThreads) kmeans_pp_kernel(const double* __restrict__ cand, int C, int d,
                                                               const double* __restrict__ w, int k, uint64_t seed,
                                                               double* __restrict__ cost, double* __restrict__ Cc) {
  __shared__ double wtot[32];
  __shared__ int found;
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int seg = (C + kPPThreads - 1) / kPPThreads;
  const int j0 = min(C, tid * seg), j1 = min(C, j0 + seg);
  for (int j = j0; j < j1; ++j) cost[j] = INFINITY;
  for (int i = 0; i < k; ++i) {
    const bool weighted = i > 0;
    if (tid == 0) found = C;
    double loc = 0.0;
    for (int j = j0; j < j1; ++j) loc += weighted ? __dmul_rn(w[j], cost[j]) : w[j];
    double incl = loc;
    for (int o = 1; o < 32; o <<= 1) {
      const double t = __shfl_up_sync(0xffffffffu, incl, o);
      if (lane >= o) incl += t;
    }
    double excl = __shfl_up_sync(0xffffffffu, incl, 1);
    if (lane == 0) excl = 0.0;
    if (lane == 31) wtot[warp] = incl;
    __syncthreads();
    if (warp == 0) {
      double t = wtot[lane];
      for (int o = 1; o < 32; o <<= 1) {
        const double q = __shfl_up_sync(0xffffffffu, t, o);
        if (lane >= o) t += q;
      }
      wtot[lane] = t;
    }
    __syncthreads();
    const double total = wtot[31];
    const double r = km_u(seed, 100, static_cast<uint64_t>(i)) * total;
    if (r > 0.0) {
      double cum = (warp > 0 ? wtot[warp - 1] : 0.0) + excl;
      for (int j = j0; j < j1; ++j) {
        cum += weighted ? __dmul_rn(w[j], cost[j]) : w[j];
        if (cum >= r) { atomicMin(&found, j); break; }
      }
    }
    __syncthreads();
    const int p = !(r > 0.0) ? 0 : (found < C ? found : C - 1);
    const double* cp = cand + static_cast<size_t>(p) * d;
    for (int e = tid; e < d; e += kPPThreads) Cc[static_cast<size_t>(i) * d + e] = cp[e];
    for (int j = j0; j < j1; ++j) {
      const double* cj = cand + static_cast<size_t>(j) * d;
      double s = 0.0;
      for (int e = 0; e < d; ++e) {
        const double df = cj[e] - cp[e];
        s = __dadd_rn(s, __dmul_rn(df, df));
      }
      cost[j] = fmin(cost[j], s);
    }
    __syncthreads();
  }
}

unsigned blocks(long long n, int t) { return static_cast<unsigned>((n + t - 1) / t); }

// out[q][j] = X[idx[q]][j] as fp64: the rows the host reads (candidates, the origin's fallback) when X is device memory
template <typename T>
__global__ void __launch_bounds__(256) kmeans_gather_rows_kernel(const T* __restrict__ X, int d,
                                                                 const long long* __restrict__ idx, int m,
                                                                 double* __restrict__ out) {
  const long long t = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x;
  if (t >= static_cast<long long>(m) * d) return;
  const int q = static_cast<int>(t / d), j = static_cast<int>(t % d);
  out[t] = static_cast<double>(X[static_cast<size_t>(idx[q]) * d + j]);
}

// bump allocator over one scratch block (256-byte aligned pieces)
struct Carve {
  char* base;
  size_t off = 0;
  template <class P> P* take(size_t count) {
    P* p = reinterpret_cast<P*>(base ? base + off : nullptr);
    off += (count * sizeof(P) + 255) / 256 * 256;
    return p;
  }
};

int label_bits(int k) {
  int b = 1;
  while ((1LL << b) < k) ++b;
  return b;
}

template <typename T>
struct KMeansRun {
  Ctx* c;
  const T* X;      // host, or device memory where on_device
  bool on_device;
  int n, d, k;
  uint64_t seed;
  cudaStream_t s;
  // sgp_kmeans_sharded: this rank holds the global rows [off, off + n) of N; the collectives sum over c's communicator
  bool sharded = false;
  long long off = 0, N = 0;
  // point-sized workspace
  T* dX = nullptr;
  int *label = nullptr, *iota = nullptr, *sel = nullptr, *keys = nullptr, *vals = nullptr, *ints = nullptr;
  double *dist = nullptr, *cost = nullptr, *part = nullptr, *o = nullptr;
  unsigned char* flag = nullptr;
  void* cub_tmp = nullptr;
  size_t cub_bytes = 0;
  // centre workspace (k rows)
  double *Cc = nullptr, *wsum = nullptr, *sums = nullptr;
  long long* cnts = nullptr;
  float* Cf = nullptr;
  int *beg = nullptr, *end = nullptr;
  int slices = 1, rows_per_slice = 1;
  Frame fr{};                     // o, the prescale and the range flag (ints + 5), set by origin()

  int sync() { SGP_CUDA(c, cudaStreamSynchronize(s)); return SGP_OK; }

  // host values summed element-wise over the ranks (sharded only), in place
  int allsum(void* host, size_t count, ncclDataType_t type) {
    if (!sharded || count == 0) return SGP_OK;
    const size_t bytes = count * 8;                            // every type summed here is 8 bytes wide
    int rc = ctx_scratch(c, c->kmeans_comm_ws, bytes);
    if (rc != SGP_OK) return rc;
    SGP_CUDA(c, cudaMemcpyAsync(c->kmeans_comm_ws.p, host, bytes, cudaMemcpyHostToDevice, s));
    rc = comm_sum(c, c->kmeans_comm_ws.p, count, type);
    if (rc != SGP_OK) return rc;
    SGP_CUDA(c, cudaMemcpyAsync(host, c->kmeans_comm_ws.p, bytes, cudaMemcpyDeviceToHost, s));
    return sync();
  }

  // fixed_sum over the ranks: each rank's fixed-order sum, then their sum
  double global_sum(const double* v, int m, int& rc) {
    double t = fixed_sum(v, m, rc);
    if (rc == SGP_OK) rc = allsum(&t, 1, ncclDouble);
    return t;
  }

  double fixed_sum(const double* v, int m, int& rc) {
    const int per = (m + kSumBlocks - 1) / kSumBlocks;
    kmeans_sum_kernel<<<kSumBlocks, 256, 0, s>>>(v, m, per, part);
    c->launches += 1;
    std::vector<double> h(kSumBlocks);
    cudaError_t e = cudaMemcpyAsync(h.data(), part, kSumBlocks * 8, cudaMemcpyDeviceToHost, s);
    if (e == cudaSuccess) e = cudaStreamSynchronize(s);
    if (e != cudaSuccess) { rc = fail(c, SGP_E_CUDA, std::string("kmeans sum: ") + cudaGetErrorString(e)); return 0.0; }
    double t = 0.0;
    for (double x : h) t += x;
    rc = SGP_OK;
    return t;
  }

  int centre_images(const double* C, int kk, float* F) {
    const int rows = rows_pad(kk), cs = cstride(d);
    kmeans_centre_f32_kernel<<<blocks(static_cast<long long>(rows) * cs, 256), 256, 0, s>>>(C, kk, d, o, fr.sc, F, rows,
                                                                                            cs);
    SGP_CUDA(c, cudaGetLastError());
    c->launches += 1;
    return SGP_OK;
  }

  // stable sort of (label, idx) -- idx = 0..m-1 -- cluster bounds, fixed-order (weighted) means
  template <typename P>
  int update(const P* pts, int m, const int* lab, const int* idx, const double* w, int kk, double tol2, int* notconv,
             void* tmp, size_t tmp_bytes, int* kout, int* vout) {
    SGP_CUDA(c, cub::DeviceRadixSort::SortPairs(tmp, tmp_bytes, lab, kout, idx, vout, m, 0, label_bits(kk), s));
    SGP_CUDA(c, cudaMemsetAsync(beg, 0, static_cast<size_t>(kk) * sizeof(int), s));
    SGP_CUDA(c, cudaMemsetAsync(end, 0, static_cast<size_t>(kk) * sizeof(int), s));
    kmeans_bounds_kernel<<<blocks(m, 256), 256, 0, s>>>(kout, m, beg, end);
    kmeans_update_kernel<P><<<blocks(static_cast<long long>(kk) * 32, 256), 256, 0, s>>>(pts, d, vout, beg, end, w, kk, Cc,
                                                                                       wsum, tol2, notconv);
    SGP_CUDA(c, cudaGetLastError());
    c->launches += 3;
    return SGP_OK;
  }

  // the Lloyd update over the ranks: this rank's per-cluster sums (point order) and counts, summed over the ranks, then
  // every rank moves the centres from the same totals
  int update_sharded(int kk, double tol2, int* notconv) {
    SGP_CUDA(c, cudaMemsetAsync(beg, 0, static_cast<size_t>(kk) * sizeof(int), s));
    SGP_CUDA(c, cudaMemsetAsync(end, 0, static_cast<size_t>(kk) * sizeof(int), s));
    if (n > 0) {
      size_t tb = cub_bytes;
      SGP_CUDA(c, cub::DeviceRadixSort::SortPairs(cub_tmp, tb, label, keys, iota, vals, n, 0, label_bits(kk), s));
      kmeans_bounds_kernel<<<blocks(n, 256), 256, 0, s>>>(keys, n, beg, end);
      c->launches += 2;
    }
    kmeans_sums_kernel<T><<<blocks(static_cast<long long>(kk) * 32, 256), 256, 0, s>>>(dX, d, vals, beg, end, kk, sums,
                                                                                      cnts);
    SGP_CUDA(c, cudaGetLastError());
    c->launches += 1;
    int rc = comm_sum(c, sums, static_cast<size_t>(kk) * d, ncclDouble);
    if (rc == SGP_OK) rc = comm_sum(c, cnts, static_cast<size_t>(kk), ncclInt64);
    if (rc != SGP_OK) return rc;
    kmeans_centre_kernel<<<blocks(static_cast<long long>(kk) * 32, 256), 256, 0, s>>>(sums, cnts, kk, d, Cc, tol2, notconv);
    SGP_CUDA(c, cudaGetLastError());
    c->launches += 1;
    return SGP_OK;
  }

  // this rank's chosen global indices -> every rank's, in rank order (= global index order: the ranks' rows follow each
  // other in rank order)
  int gather_chosen(std::vector<long long>& chosen) {
    if (!sharded) return SGP_OK;
    const int R = c->comm ? c->nranks : 1, me = c->comm ? c->rank : 0;
    std::vector<long long> counts(static_cast<size_t>(R), 0);
    counts[me] = static_cast<long long>(chosen.size());
    int rc = allsum(counts.data(), counts.size(), ncclInt64);
    if (rc != SGP_OK) return rc;
    long long total = 0, mine = 0;
    for (int r = 0; r < R; ++r) { if (r == me) mine = total; total += counts[r]; }
    std::vector<long long> all(static_cast<size_t>(total), 0);
    std::copy(chosen.begin(), chosen.end(), all.begin() + mine);
    rc = allsum(all.data(), all.size(), ncclInt64);
    if (rc != SGP_OK) return rc;
    chosen.swap(all);
    return SGP_OK;
  }

  int setup() {
    size_t t1 = 0, t2 = 0;
    SGP_CUDA(c, cub::DeviceRadixSort::SortPairs(nullptr, t1, static_cast<int*>(nullptr), static_cast<int*>(nullptr),
                                                static_cast<int*>(nullptr), static_cast<int*>(nullptr), n, 0, 32, s));
    SGP_CUDA(c, cub::DeviceSelect::Flagged(nullptr, t2, static_cast<int*>(nullptr), static_cast<unsigned char*>(nullptr),
                                           static_cast<int*>(nullptr), static_cast<int*>(nullptr), n, s));
    cub_bytes = std::max(t1, t2);
    slices = std::min(kSumBlocks, std::max(1, (n + 1023) / 1024));
    rows_per_slice = (n + slices - 1) / slices;
    const size_t N = static_cast<size_t>(n);
    auto carve = [&](Carve& cv) {
      dX = cv.take<T>(on_device ? 0 : N * d);
      label = cv.take<int>(N); iota = cv.take<int>(N); sel = cv.take<int>(N); keys = cv.take<int>(N); vals = cv.take<int>(N);
      dist = cv.take<double>(N); cost = cv.take<double>(N); flag = cv.take<unsigned char>(N);
      part = cv.take<double>(std::max<size_t>(static_cast<size_t>(slices) * 2 * d, kSumBlocks));
      o = cv.take<double>(d); ints = cv.take<int>(8);
      cub_tmp = cv.take<char>(cub_bytes);
    };
    Carve probe{nullptr};
    carve(probe);
    int rc = ctx_scratch(c, c->kmeans_pts_ws, probe.off);
    if (rc != SGP_OK) return rc;
    Carve real{static_cast<char*>(c->kmeans_pts_ws.p)};
    carve(real);
    if (on_device) dX = const_cast<T*>(X);     // read in place, never written
    const size_t K = static_cast<size_t>(k);
    auto carve_c = [&](Carve& cv) {
      Cc = cv.take<double>(K * d); wsum = cv.take<double>(K);
      sums = cv.take<double>(sharded ? K * d : 0); cnts = cv.take<long long>(sharded ? K : 0);
      Cf = cv.take<float>(static_cast<size_t>(rows_pad(k)) * cstride(d));
      beg = cv.take<int>(K); end = cv.take<int>(K);
    };
    Carve probe2{nullptr};
    carve_c(probe2);
    rc = ctx_scratch(c, c->kmeans_cen_ws, probe2.off);
    if (rc != SGP_OK) return rc;
    Carve real2{static_cast<char*>(c->kmeans_cen_ws.p)};
    carve_c(real2);
    return SGP_OK;
  }

  // the data's origin: per column the fp64 mean rounded to a multiple of the largest power of two not above the column's
  // standard deviation (so that the shift is exact for integer data), or the first point's coordinate for a constant column
  int origin() {
    if (!on_device) SGP_CUDA(c, cudaMemcpyAsync(dX, X, static_cast<size_t>(n) * d * sizeof(T), cudaMemcpyHostToDevice, s));
    SGP_CUDA(c, cudaMemsetAsync(ints, 0, 8 * sizeof(int), s));
    kmeans_colstats_kernel<T><<<slices, 256, 0, s>>>(dX, n, d, rows_per_slice, part, ints);
    SGP_CUDA(c, cudaGetLastError());
    c->launches += 1;
    std::vector<double> h(static_cast<size_t>(slices) * 2 * d);
    int bad = 0;
    SGP_CUDA(c, cudaMemcpyAsync(h.data(), part, h.size() * 8, cudaMemcpyDeviceToHost, s));
    SGP_CUDA(c, cudaMemcpyAsync(&bad, ints, sizeof(int), cudaMemcpyDeviceToHost, s));
    SGP_CUDA(c, cudaStreamSynchronize(s));
    // [column sums; column sums of squares; non-finite flag], the slices folded in order, then summed over the ranks
    std::vector<double> ab(static_cast<size_t>(2) * d + 1, 0.0);
    for (int j = 0; j < d; ++j)
      for (int q = 0; q < slices; ++q) {
        ab[j] += h[static_cast<size_t>(q) * 2 * d + j];
        ab[d + j] += h[static_cast<size_t>(q) * 2 * d + d + j];
      }
    ab[2 * d] = bad ? 1.0 : 0.0;
    int rc = allsum(ab.data(), ab.size(), ncclDouble);
    if (rc != SGP_OK) return rc;
    if (ab[2 * d] != 0.0) return fail(c, SGP_E_BADARG, "sgp_kmeans: X contains NaN or infinity");
    std::vector<double> oh(d), x0(d);
    rc = grows({0}, x0.data());
    if (rc != SGP_OK) return rc;
    const double nt = static_cast<double>(N);
    double sdmax = 0.0;
    bool finite = true;
    for (int j = 0; j < d; ++j) {
      const double a = ab[j], b = ab[d + j];
      const double mean = a / nt, sd = std::sqrt(std::max(b / nt - mean * mean, 0.0));
      if (sd > 0.0 && std::isfinite(sd)) {
        const double q = std::ldexp(1.0, std::ilogb(sd));
        oh[j] = std::nearbyint(mean / q) * q;
        sdmax = std::max(sdmax, sd);
      } else {
        finite = finite && std::isfinite(sd);
        oh[j] = x0[j];
      }
    }
    // the prescale 2^s: none while the largest sd is within [2^-16, 2^16], else the s that brings it into [1, 2), so that
    // the fp32 squares neither underflow nor overflow at the data's scale.  |s| <= 511 keeps 2^s and 2^-2s normal fp64
    // numbers; beyond it (or where a column's sum of squares overflows fp64) the data are refused rather than collapsed.
    // Every rank derives s from the same summed statistics, so every rank refuses together.
    int sexp = 0;
    if (sdmax > 0.0 && (sdmax < 0x1.0p-16 || sdmax > 0x1.0p16)) sexp = -std::ilogb(sdmax);
    if (!finite || sexp < -511 || sexp > 511)
      return fail(c, SGP_E_RANGE, "sgp_kmeans: the data's spread is outside the range of the fp32 distances (largest "
                                  "column standard deviation outside [2^-511, 2^512), or sums of squares beyond fp64)");
    fr = Frame{o, std::ldexp(1.0, sexp), std::ldexp(1.0, -2 * sexp), ints + 5};
    SGP_CUDA(c, cudaMemcpyAsync(o, oh.data(), static_cast<size_t>(d) * 8, cudaMemcpyHostToDevice, s));
    return SGP_OK;
  }

  // the rows idx of X as fp64, row after row, into host memory
  int rows(const std::vector<long long>& idx, double* out) {
    if (!on_device) {
      for (size_t q = 0; q < idx.size(); ++q)
        for (int j = 0; j < d; ++j) out[q * d + j] = static_cast<double>(X[static_cast<size_t>(idx[q]) * d + j]);
      return SGP_OK;
    }
    const size_t m = idx.size(), ib = (m * 8 + 255) / 256 * 256;
    int rc = ctx_scratch(c, c->kmeans_rows_ws, ib + m * d * 8);
    if (rc != SGP_OK) return rc;
    long long* didx = static_cast<long long*>(c->kmeans_rows_ws.p);
    double* drows = reinterpret_cast<double*>(static_cast<char*>(c->kmeans_rows_ws.p) + ib);
    SGP_CUDA(c, cudaMemcpyAsync(didx, idx.data(), m * 8, cudaMemcpyHostToDevice, s));
    kmeans_gather_rows_kernel<T><<<blocks(static_cast<long long>(m) * d, 256), 256, 0, s>>>(X, d, didx, static_cast<int>(m),
                                                                                          drows);
    SGP_CUDA(c, cudaGetLastError());
    c->launches += 1;
    SGP_CUDA(c, cudaMemcpyAsync(out, drows, m * d * 8, cudaMemcpyDeviceToHost, s));
    return sync();
  }

  // the global rows idx as fp64 into host memory: each rank contributes the rows it holds, and the rows' bit patterns are
  // summed over the ranks as integers (exact: every other rank adds zero)
  int grows(const std::vector<long long>& idx, double* out) {
    if (!sharded) return rows(idx, out);
    std::vector<long long> mine;
    std::vector<size_t> where;
    for (size_t q = 0; q < idx.size(); ++q)
      if (idx[q] >= off && idx[q] < off + n) { mine.push_back(idx[q] - off); where.push_back(q); }
    std::vector<double> loc(mine.size() * d);
    if (!mine.empty()) {
      const int rc = rows(mine, loc.data());
      if (rc != SGP_OK) return rc;
    }
    std::vector<uint64_t> bits(idx.size() * d, 0);
    for (size_t q = 0; q < mine.size(); ++q) std::memcpy(&bits[where[q] * d], &loc[q * d], static_cast<size_t>(d) * 8);
    const int rc = allsum(bits.data(), bits.size(), ncclUint64);
    if (rc != SGP_OK) return rc;
    std::memcpy(out, bits.data(), bits.size() * 8);
    return SGP_OK;
  }

  // k-means|| (KMeans.initKMeansParallel) then, for more than k distinct candidates, the local weighted k-means++ and its
  // Lloyd iterations (LocalKMeans.kMeansPlusPlus).  Leaves the kk initial centres in Cc.
  int init_parallel(int* kk_out) {
    const long long i0 = std::min<long long>(N - 1, static_cast<long long>(std::floor(km_u(seed, 0, 0) * N)));
    std::vector<long long> cand_idx{i0}, new_idx{i0};
    if (n > 0) {
      kmeans_fill_kernel<<<blocks(n, 256), 256, 0, s>>>(cost, n, INFINITY);
      kmeans_iota_kernel<<<blocks(n, 256), 256, 0, s>>>(iota, n, 0);
      SGP_CUDA(c, cudaGetLastError());
      c->launches += 2;
    }
    std::vector<double> rows;
    for (int step = 0; step < 2; ++step) {
      const int m = static_cast<int>(new_idx.size());
      if (m > 0) {
        rows.resize(static_cast<size_t>(m) * d);
        int rc = grows(new_idx, rows.data());
        if (rc != SGP_OK) return rc;
        const size_t img = (static_cast<size_t>(rows_pad(m)) * cstride(d) * 4 + 255) / 256 * 256;
        rc = ctx_scratch(c, c->kmeans_new_ws, img + rows.size() * 8);
        if (rc != SGP_OK) return rc;
        float* F = static_cast<float*>(c->kmeans_new_ws.p);
        double* R = reinterpret_cast<double*>(static_cast<char*>(c->kmeans_new_ws.p) + img);
        SGP_CUDA(c, cudaMemcpyAsync(R, rows.data(), rows.size() * 8, cudaMemcpyHostToDevice, s));
        rc = centre_images(R, m, F);
        if (rc != SGP_OK) return rc;
        if (n > 0) {
          SGP_CUDA(c, launch_assign<T>(dX, n, d, fr, F, m, nullptr, cost, 1, nullptr, s));
          c->launches += 1;
        }
      }
      int rc = SGP_OK;
      const double S = global_sum(cost, n, rc);
      if (rc != SGP_OK) return rc;
      int cnt = 0;
      if (n > 0) {
        kmeans_sample_kernel<<<blocks(n, 256), 256, 0, s>>>(cost, n, off, 2.0 * k, S, seed, 1 + step, flag);
        SGP_CUDA(c, cudaGetLastError());
        size_t tb = cub_bytes;
        SGP_CUDA(c, cub::DeviceSelect::Flagged(cub_tmp, tb, iota, flag, sel, ints + 1, n, s));
        c->launches += 2;
        SGP_CUDA(c, cudaMemcpyAsync(&cnt, ints + 1, sizeof(int), cudaMemcpyDeviceToHost, s));
        SGP_CUDA(c, cudaStreamSynchronize(s));
      }
      std::vector<int> chosen(cnt);
      if (cnt > 0) SGP_CUDA(c, cudaMemcpyAsync(chosen.data(), sel, static_cast<size_t>(cnt) * 4, cudaMemcpyDeviceToHost, s));
      SGP_CUDA(c, cudaStreamSynchronize(s));
      new_idx.assign(chosen.begin(), chosen.end());
      for (long long& g : new_idx) g += off;
      rc = gather_chosen(new_idx);
      if (rc != SGP_OK) return rc;
      cand_idx.insert(cand_idx.end(), new_idx.begin(), new_idx.end());
    }
    // distinct candidates, first occurrence kept (-0.0 and 0.0 are equal)
    std::vector<double> cand, all(cand_idx.size() * d), r(d);
    std::unordered_set<std::string> seen;
    int rc = grows(cand_idx, all.data());
    if (rc != SGP_OK) return rc;
    for (size_t q = 0; q < cand_idx.size(); ++q) {
      std::copy(all.begin() + q * d, all.begin() + (q + 1) * d, r.begin());
      std::string key(reinterpret_cast<const char*>(r.data()), static_cast<size_t>(d) * 8);
      for (int j = 0; j < d; ++j) {
        const double z = r[j] + 0.0;
        std::memcpy(&key[static_cast<size_t>(j) * 8], &z, 8);
      }
      if (seen.insert(key).second) cand.insert(cand.end(), r.begin(), r.end());
    }
    const int C = static_cast<int>(cand.size() / d);
    if (C <= k) {
      SGP_CUDA(c, cudaMemcpyAsync(Cc, cand.data(), cand.size() * 8, cudaMemcpyHostToDevice, s));
      *kk_out = C;
      return sync();
    }
    // ---- local k-means++ over the weighted candidates ----
    size_t tsort = 0;
    SGP_CUDA(c, cub::DeviceRadixSort::SortPairs(nullptr, tsort, static_cast<int*>(nullptr), static_cast<int*>(nullptr),
                                                static_cast<int*>(nullptr), static_cast<int*>(nullptr), C, 0, 32, s));
    const size_t Cz = static_cast<size_t>(C);
    double *dcand = nullptr, *w = nullptr, *cdist = nullptr, *ccost = nullptr;
    float* CF = nullptr;
    int *cnt = nullptr, *clab = nullptr, *ckeys = nullptr, *cvals = nullptr, *cidx = nullptr;
    void* ctmp = nullptr;
    auto carve = [&](Carve& cv) {
      dcand = cv.take<double>(Cz * d); w = cv.take<double>(Cz); cdist = cv.take<double>(Cz); ccost = cv.take<double>(Cz);
      CF = cv.take<float>(static_cast<size_t>(rows_pad(C)) * cstride(d));
      cnt = cv.take<int>(Cz); clab = cv.take<int>(Cz); ckeys = cv.take<int>(Cz); cvals = cv.take<int>(Cz);
      cidx = cv.take<int>(Cz);      // the candidates' own 0..C-1 (a shard may hold fewer than C points)
      ctmp = cv.take<char>(tsort);
    };
    Carve probe{nullptr};
    carve(probe);
    rc = ctx_scratch(c, c->kmeans_cand_ws, probe.off);
    if (rc != SGP_OK) return rc;
    Carve real{static_cast<char*>(c->kmeans_cand_ws.p)};
    carve(real);
    SGP_CUDA(c, cudaMemcpyAsync(dcand, cand.data(), cand.size() * 8, cudaMemcpyHostToDevice, s));
    rc = centre_images(dcand, C, CF);
    if (rc != SGP_OK) return rc;
    // weights: how many points have each candidate as their nearest
    SGP_CUDA(c, cudaMemsetAsync(cnt, 0, Cz * sizeof(int), s));
    if (n > 0) {
      SGP_CUDA(c, launch_assign<T>(dX, n, d, fr, CF, C, label, dist, 0, nullptr, s));
      kmeans_count_kernel<<<blocks(n, 256), 256, 0, s>>>(label, n, cnt);
    }
    if (sharded) {                            // int64 counts summed over the ranks
      std::vector<int> ci(Cz);
      SGP_CUDA(c, cudaMemcpyAsync(ci.data(), cnt, Cz * sizeof(int), cudaMemcpyDeviceToHost, s));
      SGP_CUDA(c, cudaStreamSynchronize(s));
      std::vector<long long> cl(ci.begin(), ci.end());
      rc = allsum(cl.data(), cl.size(), ncclInt64);
      if (rc != SGP_OK) return rc;
      std::vector<double> wh(cl.begin(), cl.end());
      SGP_CUDA(c, cudaMemcpyAsync(w, wh.data(), Cz * 8, cudaMemcpyHostToDevice, s));
      SGP_CUDA(c, cudaStreamSynchronize(s));
    } else {
      kmeans_to_double_kernel<<<blocks(C, 256), 256, 0, s>>>(cnt, C, w);
    }
    kmeans_pp_kernel<<<1, kPPThreads, 0, s>>>(dcand, C, d, w, k, seed, ccost, Cc);
    kmeans_iota_kernel<<<blocks(C, 256), 256, 0, s>>>(clab, C, -1);
    kmeans_iota_kernel<<<blocks(C, 256), 256, 0, s>>>(cidx, C, 0);
    SGP_CUDA(c, cudaGetLastError());
    SGP_CUDA(c, cudaMemsetAsync(ints + 2, 0, 2 * sizeof(int), s));   // [2] changed, [3] empty-cluster draw counter
    c->launches += 6;
    for (int it = 0; it < 30; ++it) {
      rc = centre_images(Cc, k, Cf);
      if (rc != SGP_OK) return rc;
      SGP_CUDA(c, cudaMemsetAsync(ints + 2, 0, sizeof(int), s));
      SGP_CUDA(c, launch_assign<double>(dcand, C, d, fr, Cf, k, clab, cdist, 0, ints + 2, s));
      rc = update<double>(dcand, C, clab, cidx, w, k, 0.0, nullptr, ctmp, tsort, ckeys, cvals);
      if (rc != SGP_OK) return rc;
      kmeans_local_empty_kernel<<<1, 1, 0, s>>>(wsum, k, dcand, C, d, Cc, seed, ints + 3);
      SGP_CUDA(c, cudaGetLastError());
      c->launches += 2;
      int moved = 0;
      SGP_CUDA(c, cudaMemcpyAsync(&moved, ints + 2, sizeof(int), cudaMemcpyDeviceToHost, s));
      SGP_CUDA(c, cudaStreamSynchronize(s));
      if (!moved) break;
    }
    *kk_out = k;
    return SGP_OK;
  }

  int run(int max_iter, double tol, const double* init, double* centers_out, int* k_out, int* labels_out, int* iters_out,
          double* cost_out) {
    int rc = setup();
    if (rc == SGP_OK) rc = origin();
    if (rc != SGP_OK) return rc;
    int kk = k;
    if (init) {
      SGP_CUDA(c, cudaMemcpyAsync(Cc, init, static_cast<size_t>(k) * d * 8, cudaMemcpyHostToDevice, s));
      if (n > 0) {
        kmeans_iota_kernel<<<blocks(n, 256), 256, 0, s>>>(iota, n, 0);
        SGP_CUDA(c, cudaGetLastError());
        c->launches += 1;
      }
    } else {
      rc = init_parallel(&kk);
      if (rc != SGP_OK) return rc;
    }
    // ---- Lloyd (KMeans.runAlgorithmWithWeight) ----
    rc = centre_images(Cc, kk, Cf);
    if (rc != SGP_OK) return rc;
    int iteration = 0;
    bool converged = false;
    do {
      if (n > 0) {
        SGP_CUDA(c, launch_assign<T>(dX, n, d, fr, Cf, kk, label, dist, 0, nullptr, s));
        c->launches += 1;
      }
      if (max_iter == 0) break;
      SGP_CUDA(c, cudaMemsetAsync(ints + 4, 0, sizeof(int), s));
      rc = sharded ? update_sharded(kk, tol * tol, ints + 4)
                   : update<T>(dX, n, label, iota, nullptr, kk, tol * tol, ints + 4, cub_tmp, cub_bytes, keys, vals);
      if (rc == SGP_OK) rc = centre_images(Cc, kk, Cf);
      if (rc != SGP_OK) return rc;
      int notconv = 0;
      SGP_CUDA(c, cudaMemcpyAsync(&notconv, ints + 4, sizeof(int), cudaMemcpyDeviceToHost, s));
      SGP_CUDA(c, cudaStreamSynchronize(s));
      converged = notconv == 0;
      ++iteration;
    } while (iteration < max_iter && !converged);
    const double cost_total = global_sum(dist, n, rc);
    if (rc != SGP_OK) return rc;
    // a nearest-centre distance beyond the fp32 range even after the prescale (a centre or point far outside the data's
    // spread): refused on every rank together, rather than returning a run whose draws and costs were inf
    int fl = 0;
    SGP_CUDA(c, cudaMemcpyAsync(&fl, ints + 5, sizeof(int), cudaMemcpyDeviceToHost, s));
    SGP_CUDA(c, cudaStreamSynchronize(s));
    double far = fl ? 1.0 : 0.0;
    rc = allsum(&far, 1, ncclDouble);
    if (rc != SGP_OK) return rc;
    if (far != 0.0)
      return fail(c, SGP_E_RANGE, "sgp_kmeans: a squared distance to the nearest centre is beyond the fp32 range after the "
                                  "data's power-of-two prescale");
    SGP_CUDA(c, cudaMemcpyAsync(centers_out, Cc, static_cast<size_t>(kk) * d * 8, cudaMemcpyDeviceToHost, s));
    if (labels_out && n > 0) SGP_CUDA(c, cudaMemcpyAsync(labels_out, label, static_cast<size_t>(n) * 4, cudaMemcpyDeviceToHost, s));
    SGP_CUDA(c, cudaStreamSynchronize(s));
    *k_out = kk;
    *iters_out = iteration;
    *cost_out = cost_total;
    return SGP_OK;
  }
};

}  // namespace

int run_kmeans(Ctx* c, const void* X, int x_is_f32, bool x_on_device, long long n, int d, int k, int max_iter, double tol,
               uint64_t seed, const double* init_centers, double* centers_out, int* k_out, int* labels_out,
               int* iterations_out, double* cost_out) {
  if (x_is_f32) {
    KMeansRun<float> r{c, static_cast<const float*>(X), x_on_device, static_cast<int>(n), d, k, seed, c->stream};
    r.N = n;
    return r.run(max_iter, tol, init_centers, centers_out, k_out, labels_out, iterations_out, cost_out);
  }
  KMeansRun<double> r{c, static_cast<const double*>(X), x_on_device, static_cast<int>(n), d, k, seed, c->stream};
  r.N = n;
  return r.run(max_iter, tol, init_centers, centers_out, k_out, labels_out, iterations_out, cost_out);
}

int run_kmeans_sharded(Ctx* c, const void* X, int x_is_f32, bool x_on_device, long long n, long long offset,
                       long long n_total, int d, int k, int max_iter, double tol, uint64_t seed, const double* init_centers,
                       double* centers_out, int* k_out, int* labels_out, int* iterations_out, double* cost_out) {
  if (x_is_f32) {
    KMeansRun<float> r{c, static_cast<const float*>(X), x_on_device, static_cast<int>(n), d, k, seed, c->stream};
    r.sharded = true; r.off = offset; r.N = n_total;
    return r.run(max_iter, tol, init_centers, centers_out, k_out, labels_out, iterations_out, cost_out);
  }
  KMeansRun<double> r{c, static_cast<const double*>(X), x_on_device, static_cast<int>(n), d, k, seed, c->stream};
  r.sharded = true; r.off = offset; r.N = n_total;
  return r.run(max_iter, tol, init_centers, centers_out, k_out, labels_out, iterations_out, cost_out);
}

}  // namespace sgp
