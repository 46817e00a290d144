// Operand preparation of the int8 exact-accumulation Gram (gram_i8_wgmma.cu) and of the K_nm sweep (kmn_sweep.cu):
// fp16 hi/lo-split operand images for the tensor-core distance contraction, fp32 coordinate tiles for the direct-distance
// mode.  The images are ready-to-copy shared-memory tiles (K-major SWIZZLE_128B), moved by one bulk copy per unit.
#include <cuda_fp16.h>

#include "sgp_internal.h"

namespace sgp {
namespace {

constexpr int UP = 64;                  // points per pipeline unit
constexpr int PANEL_BYTES = 16384;      // 128 rows x 128 bytes, SWIZZLE_128B K-major
constexpr int XIMG_BYTES = 8192;        // 64 rows x 128 bytes

// byte offset of (row r, 16-byte chunk c16 in [0,8)) inside a K-major SWIZZLE_128B tile with 128-byte rows
__host__ __device__ __forceinline__ uint32_t sw128_off(int r, int c16) {
  return static_cast<uint32_t>((r >> 3) * 1024 + (r & 7) * 128 + ((c16 ^ (r & 7)) << 4));
}

// ---------------------------------------------------------------------------------------------------
// Operand preparation: fp16 hi/lo split of the scaled, centred coordinates + norm columns, written as
// ready-to-copy shared-memory images (K-major SWIZZLE_128B).  Logical K columns (dp = d padded to 16):
//   [0,dp)        A: zh_k   B: 2*xh_k          [dp,2dp)   A: zl_k   B: 2*xh_k
//   [2dp,3dp)     A: zh_k   B: 2*xl_k          [3dp,3dp+16) A: 1,1,1,c1,c2,c3,0..  B: r1,r2,r3,1,1,1,0..
// with x^ = sqrt(log2 e) * beta * (x - centre) = xh + xl (fp16 each), r = -|xh+xl|^2 = r1+r2+r3, c likewise, so
// that  sum_K A*B = 2 x^.z^ - |x^|^2 - |z^|^2 (+ xl.zl, ~1e-8)  = -q * log2(e)  of the represented points.
// ---------------------------------------------------------------------------------------------------
struct SplitRow {
  __half hi[32], lo[32];
  __half n1, n2, n3;   // three-piece fp16 expansion of -|hi+lo|^2
};

__device__ __forceinline__ void split_row(const double* v, int dp, SplitRow& s, double& norm2) {
  double acc = 0.0;
  for (int k = 0; k < dp; ++k) {
    const __half h = __double2half(v[k]);
    const __half l = __double2half(v[k] - static_cast<double>(__half2float(h)));
    s.hi[k] = h; s.lo[k] = l;
    const double r = static_cast<double>(__half2float(h)) + static_cast<double>(__half2float(l));
    acc += r * r;
  }
  norm2 = acc;
  const double n = -acc;
  s.n1 = __double2half(n);
  const double e1 = n - static_cast<double>(__half2float(s.n1));
  s.n2 = __double2half(e1);
  s.n3 = __double2half(e1 - static_cast<double>(__half2float(s.n2)));
}

template <bool IS_B>   // IS_B: point rows (B operand), else active-set rows (A operand)
__device__ __forceinline__ __half operand_col(const SplitRow& s, int dp, int L, bool valid) {
  const __half zero = __float2half(0.f), one = __float2half(1.f);
  if (L < 3 * dp) {
    if (!valid) return zero;
    const int seg = L / dp, k = L % dp;
    if (IS_B) {
      const __half h = (seg == 2) ? s.lo[k] : s.hi[k];
      return __hadd(h, h);                                   // 2*x (exact)
    }
    return (seg == 1) ? s.lo[k] : s.hi[k];
  }
  const int a = L - 3 * dp;                                   // augmented columns
  if (IS_B) {
    if (a == 0) return valid ? s.n1 : __float2half(-60000.f);  // padded point: T = -60000 -> kappa = 0
    if (a == 1) return valid ? s.n2 : zero;
    if (a == 2) return valid ? s.n3 : zero;
    if (a < 6) return one;
    return zero;
  }
  if (a < 3) return one;
  if (a == 3) return valid ? s.n1 : __float2half(-60000.f);    // padded active row
  if (a == 4) return valid ? s.n2 : zero;
  if (a == 5) return valid ? s.n3 : zero;
  return zero;
}

// X (n x d, fp32/fp64) -> images [unit][chunk][64 rows x 128 B] and ys (fp32, zero padded).  DP = d padded to 16 (16 or 32):
// everything is unrolled and stays in registers (a first version with run-time dp kept the split row in local memory and
// decoded every operand column with a division: ~170 us per 1M x 16 points, 5 % of the statistics step).
// B-operand columns (see the table above): [0,DP) 2 xh | [DP,2DP) 2 xh | [2DP,3DP) 2 xl | [3DP,3DP+16) r1 r2 r3 1 1 1 0.. | 0..
template <int DP>
__global__ void prep_points_kernel(uint8_t* __restrict__ Xt, float* __restrict__ ys, const void* __restrict__ X,
                                   int x_is_f32, const double* __restrict__ y, long long n, long long n_units,
                                   int d, const double* __restrict__ scale /*[DP]*/,
                                   const double* __restrict__ centre /*[DP]*/, int* __restrict__ flags,
                                   double* __restrict__ norm_sum, double* __restrict__ norm_sum_call) {
  // 128 threads = two 64-point units.  A thread builds the operand row of its point into shared memory; the block then
  // copies the rows out with 16-byte chunks of one 128-byte image row on consecutive threads (full-line stores).
  constexpr int NCH = (3 * DP + 16 + 63) / 64;                      // 64-column K chunks: 1 (DP = 16) or 2 (DP = 32)
  constexpr int ROW_BYTES = NCH * 128 + 16;                         // +16: the row-owner stores spread over the banks
  extern __shared__ __align__(16) uint8_t prep_smem[];
  __shared__ double warp_norm[4];
  const long long pt = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x;
  const bool in_grid = pt < n_units * UP;
  const bool valid = pt < n;
  __half2 hh[DP / 2], ll[DP / 2];                                   // 2 xh, 2 xl, two columns per register
  double acc = 0.0;
#pragma unroll
  for (int k = 0; k < DP; k += 2) {
    double v0 = 0.0, v1 = 0.0;
    if (valid && k < d) {
      const size_t off = static_cast<size_t>(pt) * d + k;
      v0 = x_is_f32 ? static_cast<double>(reinterpret_cast<const float*>(X)[off]) : reinterpret_cast<const double*>(X)[off];
      v0 = (v0 - centre[k]) * scale[k];
    }
    if (valid && k + 1 < d) {
      const size_t off = static_cast<size_t>(pt) * d + k + 1;
      v1 = x_is_f32 ? static_cast<double>(reinterpret_cast<const float*>(X)[off]) : reinterpret_cast<const double*>(X)[off];
      v1 = (v1 - centre[k + 1]) * scale[k + 1];
    }
    const __half h0 = __double2half(v0), h1 = __double2half(v1);
    const __half l0 = __double2half(v0 - static_cast<double>(__half2float(h0)));
    const __half l1 = __double2half(v1 - static_cast<double>(__half2float(h1)));
    const double r0 = static_cast<double>(__half2float(h0)) + static_cast<double>(__half2float(l0));
    const double r1 = static_cast<double>(__half2float(h1)) + static_cast<double>(__half2float(l1));
    acc = fma(r0, r0, acc);
    acc = fma(r1, r1, acc);
    hh[k / 2] = __halves2half2(__hadd(h0, h0), __hadd(h1, h1));     // 2 x (exact)
    ll[k / 2] = __halves2half2(__hadd(l0, l0), __hadd(l1, l1));
  }
  const double norm2 = acc;
  if (valid && !(norm2 <= kI8TensorR2Max)) atomicOr(flags, 1);    // out of the operand range -> caller falls back
  if (norm_sum) {                                                // sum of scaled squared norms (AUTO's magnitude gate)
    double v2 = valid ? norm2 : 0.0;
    for (int o = 16; o > 0; o >>= 1) v2 += __shfl_xor_sync(0xffffffffu, v2, o);
    if ((threadIdx.x & 31) == 0) warp_norm[threadIdx.x >> 5] = v2;     // one atomic per block (same-address atomics serialise)
  }
  if (in_grid) ys[pt] = (valid && y) ? static_cast<float>(y[pt]) : 0.f;
  // three-piece fp16 expansion of -|x^|^2; a padded point gets T = -60000 -> kappa = 0
  const double nn = -norm2;
  __half n1 = __double2half(nn);
  const double e1 = nn - static_cast<double>(__half2float(n1));
  __half n2 = __double2half(e1);
  __half n3 = __double2half(e1 - static_cast<double>(__half2float(n2)));
  const __half zero = __float2half(0.f), one = __float2half(1.f);
  if (!valid) { n1 = __float2half(-60000.f); n2 = zero; n3 = zero; }
  uint4* myrow = reinterpret_cast<uint4*>(prep_smem + threadIdx.x * ROW_BYTES);
  auto pack4 = [](const __half2* p) {
    uint4 u;
    u.x = *reinterpret_cast<const uint32_t*>(p + 0); u.y = *reinterpret_cast<const uint32_t*>(p + 1);
    u.z = *reinterpret_cast<const uint32_t*>(p + 2); u.w = *reinterpret_cast<const uint32_t*>(p + 3);
    return u;
  };
  constexpr int C = DP / 8;                                        // 16-byte chunks per DP columns
#pragma unroll
  for (int j = 0; j < C; ++j) {
    const uint4 h4 = pack4(hh + 4 * j), l4 = pack4(ll + 4 * j);
    myrow[j] = h4; myrow[C + j] = h4; myrow[2 * C + j] = l4;
  }
  {
    const __half2 a0 = __halves2half2(n1, n2), a1 = __halves2half2(n3, one), a2 = __halves2half2(one, one),
                  a3 = __halves2half2(zero, zero);
    uint4 u;
    u.x = *reinterpret_cast<const uint32_t*>(&a0); u.y = *reinterpret_cast<const uint32_t*>(&a1);
    u.z = *reinterpret_cast<const uint32_t*>(&a2); u.w = *reinterpret_cast<const uint32_t*>(&a3);
    myrow[3 * C] = u;
    myrow[3 * C + 1] = make_uint4(0u, 0u, 0u, 0u);
#pragma unroll
    for (int j = 3 * C + 2; j < NCH * 8; ++j) myrow[j] = make_uint4(0u, 0u, 0u, 0u);
  }
  __syncthreads();
  if (norm_sum && threadIdx.x == 0) {
    const double v2 = (warp_norm[0] + warp_norm[1]) + (warp_norm[2] + warp_norm[3]);
    if (v2 > 0.0) {
      atomicAdd(norm_sum, v2);
      if (norm_sum_call) atomicAdd(norm_sum_call, v2);
    }
  }
  const long long unit0 = static_cast<long long>(blockIdx.x) * 2;
  constexpr int PER_UNIT = NCH * 512;                              // 16-byte chunks per unit: [chunk][64 rows][8]
  for (int q = threadIdx.x; q < 2 * PER_UNIT; q += blockDim.x) {
    const int u = q / PER_UNIT, rem = q % PER_UNIT;
    const int c = rem >> 9, r = (rem >> 3) & 63, c16 = rem & 7;
    if (unit0 + u >= n_units) break;
    const uint4 val = *reinterpret_cast<const uint4*>(prep_smem + (u * 64 + r) * ROW_BYTES + c * 128 + c16 * 16);
    uint8_t* img = Xt + (static_cast<size_t>(unit0 + u) * NCH + c) * XIMG_BYTES;
    *reinterpret_cast<uint4*>(img + sw128_off(r, c16)) = val;
  }
}

// Z (m x d fp64) -> images [tile][chunk][128 rows x 128 B]
__global__ void prep_active_kernel(uint8_t* __restrict__ Zt, const double* __restrict__ Z, int m, int m_pad, int d,
                                   int dp, int nchunks, const double* __restrict__ scale, const double* __restrict__ centre,
                                   int* __restrict__ flags) {
  const int j = blockIdx.x * blockDim.x + threadIdx.x;
  if (j >= m_pad) return;
  const bool valid = j < m;
  double v[32];
  for (int k = 0; k < dp; ++k) v[k] = (valid && k < d) ? (Z[static_cast<size_t>(j) * d + k] - centre[k]) * scale[k] : 0.0;
  SplitRow s;
  double norm2;
  split_row(v, dp, s, norm2);
  if (valid && !(norm2 <= kI8TensorR2Max)) atomicOr(flags, 1);
  const int tile = j / kTile, r = j % kTile;
  for (int c = 0; c < nchunks; ++c) {
    uint8_t* img = Zt + (static_cast<size_t>(tile) * nchunks + c) * PANEL_BYTES;
    for (int c16 = 0; c16 < 8; ++c16) {
      __align__(16) __half h[8];
#pragma unroll
      for (int e = 0; e < 8; ++e) h[e] = operand_col<false>(s, dp, c * 64 + c16 * 8 + e, valid);
      *reinterpret_cast<uint4*>(img + sw128_off(r, c16)) = *reinterpret_cast<const uint4*>(h);
    }
  }
}

// ---------------------------------------------------------------------------------------------------
// Operand preparation for the DIRECT-distance mode of the Gram kernel (gram_i8_wgmma.cu): fp32 coordinate tiles, centred
// on the active-set mean and pre-scaled per kernel term by sqrt(log2 e) * beta_tk, so that the epilogue's direct-form
// sum_k (x~_k - z~_k)^2 is the base-2 exponent.  Points: [unit][term][dpad4][64]; active set: [tile][term][dpad4][128 rows], stored NEGATED (the inner loop adds).  Padding points carry +inf on coordinate 0: their kernel values are 0.
// ---------------------------------------------------------------------------------------------------
__global__ void prep_points_direct_kernel(float* __restrict__ Xd, float* __restrict__ ys, const void* __restrict__ X,
                                          int x_is_f32, const double* __restrict__ y, long long n, long long n_units, int d,
                                          int dpad4, int n_terms, const double* __restrict__ scale /*[n_terms][dpad4]*/,
                                          const double* __restrict__ centre /*[dpad4]*/, int* __restrict__ flags,
                                          float r2max, double* __restrict__ norm_sum, double* __restrict__ norm_sum_call) {
  __shared__ double warp_norm[4];
  const long long pt = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x;
  const bool in_grid = pt < n_units * UP;
  const bool valid = pt < n;
  const long long unit = pt / UP;
  const int pp = static_cast<int>(pt % UP);
  float r2[kMaxTerms] = {0.f, 0.f, 0.f, 0.f};
  for (int k = 0; k < dpad4 && in_grid; ++k) {
    double x = 0.0;
    if (valid && k < d) {
      const size_t off = static_cast<size_t>(pt) * d + k;
      x = (x_is_f32 ? static_cast<double>(reinterpret_cast<const float*>(X)[off]) : reinterpret_cast<const double*>(X)[off]) -
          centre[k];
    }
    for (int t = 0; t < n_terms; ++t) {
      float v = static_cast<float>(x * scale[t * dpad4 + k]);
      r2[t] = fmaf(v, v, r2[t]);
      if (!valid) v = (k == 0) ? __int_as_float(0x7f800000) : 0.f;     // +inf: kernel value exactly 0 against any active row
      Xd[((static_cast<size_t>(unit) * n_terms + t) * dpad4 + k) * UP + pp] = v;
    }
  }
  // fp32 coordinates: the exponent's rounding error grows like 2^-24 * sqrt(q) * (|x~| + |z~|)
  if (valid && !(fmaxf(fmaxf(r2[0], r2[1]), fmaxf(r2[2], r2[3])) <= r2max)) atomicOr(flags, 4);
  if (ys && in_grid) ys[pt] = (valid && y) ? static_cast<float>(y[pt]) : 0.f;
  if (norm_sum) {                               // AUTO's magnitude budget: scaled squared norm under the WIDEST term
    float rmin = r2[0];
    for (int t = 1; t < n_terms; ++t) rmin = fminf(rmin, r2[t]);
    double v2 = valid ? static_cast<double>(rmin) : 0.0;
    for (int o = 16; o > 0; o >>= 1) v2 += __shfl_xor_sync(0xffffffffu, v2, o);
    if ((threadIdx.x & 31) == 0) warp_norm[threadIdx.x >> 5] = v2;
    __syncthreads();
    if (threadIdx.x == 0) {
      const double tot = (warp_norm[0] + warp_norm[1]) + (warp_norm[2] + warp_norm[3]);
      if (tot > 0.0) {
        atomicAdd(norm_sum, tot);
        if (norm_sum_call) atomicAdd(norm_sum_call, tot);
      }
    }
  }
}

__global__ void prep_active_direct_kernel(float* __restrict__ Zd, const double* __restrict__ Z, int m, int m_pad, int d,
                                          int dpad4, int n_terms, const double* __restrict__ scale,
                                          const double* __restrict__ centre, int* __restrict__ flags, float r2max) {
  const int j = blockIdx.x * blockDim.x + threadIdx.x;
  if (j >= m_pad) return;
  const bool valid = j < m;
  const int tile = j / kTile, r = j % kTile;
  for (int t = 0; t < n_terms; ++t) {
    float* col = Zd + (static_cast<size_t>(tile) * n_terms + t) * dpad4 * kTile + r;
    float r2 = 0.f;
    for (int k = 0; k < dpad4; ++k) {
      float v = 0.f;
      if (valid && k < d) v = -static_cast<float>((Z[static_cast<size_t>(j) * d + k] - centre[k]) * scale[t * dpad4 + k]);
      r2 = fmaf(v, v, r2);
      col[static_cast<size_t>(k) * kTile] = v;                   // padding rows: zeros (their Gram rows are never read)
    }
    if (valid && !(r2 <= r2max)) atomicOr(flags, 4);
  }
}

}  // namespace

// -------------------------------------------------------------------------------------------------------
// host side
// -------------------------------------------------------------------------------------------------------
size_t i8_points_scratch_bytes(long long n, int nchunks) {
  const long long units = (n + UP - 1) / UP;
  return static_cast<size_t>(units) * nchunks * XIMG_BYTES;
}
size_t i8_active_scratch_bytes(int m_pad, int nchunks) {
  return static_cast<size_t>(m_pad / kTile) * nchunks * PANEL_BYTES;
}
int i8_nchunks(int d) {
  const int dp = (d + 15) / 16 * 16;
  return (3 * dp + 16 + 63) / 64;
}

cudaError_t launch_i8_prep_active(uint8_t* Zt, const double* dZ, int m, int m_pad, int d, const double* dScale,
                                  const double* dCentre, int* dFlags, cudaStream_t s) {
  const int dp = (d + 15) / 16 * 16;
  prep_active_kernel<<<(m_pad + 127) / 128, 128, 0, s>>>(Zt, dZ, m, m_pad, d, dp, i8_nchunks(d), dScale, dCentre, dFlags);
  return cudaGetLastError();
}

cudaError_t launch_i8_prep_points(uint8_t* Xt, float* ys, const void* dX, int x_is_f32, const double* dy, long long n,
                                  int d, const double* dScale, const double* dCentre, int* dFlags, double* dNormSum,
                                  double* dNormSumCall, cudaStream_t s) {
  const long long units = (n + UP - 1) / UP;
  const long long threads = units * UP;
  const unsigned grid = static_cast<unsigned>((threads + 127) / 128);
  if (d <= 16)
    prep_points_kernel<16><<<grid, 128, 128 * (1 * 128 + 16), s>>>(Xt, ys, dX, x_is_f32, dy, n, units, d, dScale, dCentre, dFlags,
                                                                  dNormSum, dNormSumCall);
  else
    prep_points_kernel<32><<<grid, 128, 128 * (2 * 128 + 16), s>>>(Xt, ys, dX, x_is_f32, dy, n, units, d, dScale, dCentre, dFlags,
                                                                  dNormSum, dNormSumCall);
  return cudaGetLastError();
}

cudaError_t launch_i8_prep_active_direct(float* Zd, const double* dZ, int m, int m_pad, int d, int dpad4, int n_terms,
                                         const double* dScale, const double* dCentre, int* flags, float r2max,
                                         cudaStream_t s) {
  prep_active_direct_kernel<<<(m_pad + 127) / 128, 128, 0, s>>>(Zd, dZ, m, m_pad, d, dpad4, n_terms, dScale, dCentre, flags,
                                                                r2max);
  return cudaGetLastError();
}

cudaError_t launch_i8_prep_points_direct(float* Xd, float* ys, const void* dX, int x_is_f32, const double* dy, long long n,
                                         int d, int dpad4, int n_terms, const double* dScale, const double* dCentre, int* flags,
                                         float r2max, double* dNormSum, double* dNormSumCall, cudaStream_t s) {
  const long long units = (n + UP - 1) / UP;
  const long long threads = units * UP;
  prep_points_direct_kernel<<<static_cast<unsigned>((threads + 127) / 128), 128, 0, s>>>(Xd, ys, dX, x_is_f32, dy, n, units, d,
                                                                                       dpad4, n_terms, dScale, dCentre, flags, r2max, dNormSum,
                                                                                       dNormSumCall);
  return cudaGetLastError();
}

}  // namespace sgp
