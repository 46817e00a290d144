// K_mn + Gram on the Hopper tensor cores (wgmma), exact-accumulation path: a digit-plane producer and an int8 Gram.
//
// Same contract as gram_f64.cu (one shard of points -> per-slice partial tiles of G = sum_n k_n k_n^T and
// b = sum_n k_n y_n; replaces commons/ProjectedGaussianProcessHelper.scala:27-29 and the crossKernel chain
// kernel/ARDRBFKernel.scala:81-89 / RBFKernel.scala:66-76 / ScalarTimesKernel.scala:24 / SumOfKernels.scala:57-58).
//
// Why integers.  tools/precision_study.py: the posterior mean only matches the fp64 reference to 1e-5 if the Gram is
// ACCUMULATED better than fp32, while fp32-accurate *elements* are 50x inside it.  Integer wgmma accumulates in int32,
// which is exact.  Every kernel element kappa in (0,1] becomes a 23-bit fixed-point integer u = rint(kappa * C0) written
// in balanced digits u = s2*2^15 + s1*2^7 + s0 (s2 in [0,255]: the unsigned operand range, s1 in [-128,127], s0 in
// [-64,63]); the stored planes P2 = s2, P1 = s1, P0 = 2 s0 are the base-256 digits of W = 2u and
//     4 sum_n u_ni u_nj = 2^32 [P2'P2] + 2^24 [P2'P1 + P1'P2] + 2^16 [P2'P0 + P0'P2 + P1'P1] + (dropped)
// is six int8 products into three int32 accumulators.  The dropped products (weights 2^8, 2^0) are zero-mean because the
// low digits are balanced; they bound this path's accuracy (posterior mean within ~2e-6 of fp64, DESIGN.md section 3).
//
// Two kernels, so that every kernel element is computed once per unit (not once per CTA whose tile holds its row):
//   kmn_i8_planes_kernel   one CTA (two warpgroups, 64 rows each) per (active tile of 128 rows, point slice).  Per
//              64-point unit: distances (tensor mode: T = -q*log2(e) as ONE fp16 wgmma contraction over the hi/lo split
//              of the scaled, centred coordinates with the norms folded in as extra K columns, images from
//              launch_i8_prep_points / launch_i8_prep_active; direct mode: sum of up to 4 terms of 2^(-|x~ - z~|^2) from
//              fp32 coordinates on the CUDA cores), then ex2 -> fixed point via one FFMA against 2^23 -> byte planes
//              (PRMT) in shared memory, in exactly the K-major SWIZZLE_64B byte image the Gram reads, and one 24 KB bulk
//              store of the tile's three planes to the plane workspace [unit][tile][3][128 x 64].  b += kappa*y for the
//              tile's rows (fp32 per unit, fp64 across units).
//   gram_i8_kernel   one CTA per (tile pair I >= J of the upper block triangle, point slice), warp specialised: one
//              thread of the copy warpgroup streams the I and J plane images of each unit into a ring of stages
//              (cp.async.bulk, mbarrier completion, released by the consumers through a second mbarrier); two consumer
//              warpgroups (64 rows of I each, all 128 columns of J) issue twelve int8 wgmma m64n128k32 per unit into three
//              int32 accumulators (192 registers, handed over from the copy warpgroup with setmaxnreg).  Every 400 units
//              the accumulators are folded into the fp64 partial tile (no overflow possible).
#include <cuda_fp16.h>

#include <algorithm>

#include "hopper.cuh"
#include "sgp_internal.h"

namespace sgp {
namespace {

using namespace hop;

constexpr int UP = 64;                  // points per pipeline unit
constexpr int NTHREADS = 256;           // producer: two warpgroups
constexpr int XSTAGES = 4;              // producer: ring of point stages
constexpr int ZPANEL_BYTES = 16384;     // fp16 active-set operand image: 128 rows x 128 bytes, SWIZZLE_128B K-major
constexpr int XIMG_BYTES = 8192;        // fp16 point operand image: 64 rows x 128 bytes
constexpr int PLANE = 8192;             // int8 digit plane of one tile: 128 rows x 64 points, K-major SWIZZLE_64B
constexpr int TILE_PLANES = 3 * PLANE;  // the three planes of one (unit, tile): one bulk copy
static_assert(TILE_PLANES == kI8PlaneBytes, "plane workspace stride");
constexpr int GTHREADS = 384;           // Gram: copy warpgroup + two consumer warpgroups
constexpr int GSTAGES = 4;              // Gram: ring of [I planes | J planes] stages, 48 KB each
constexpr int COPY_REGS = 24, MMA_REGS = 240;   // setmaxnreg split: 128 x 24 + 256 x 240 <= 65536
constexpr int FLUSH_UNITS = 400;        // |ACC4| <= 255^2 n, |ACC3| <= 2*255*128 n, |ACC2| <= (2*255*128 + 128^2) n < 2^31
// Fixed point: mantissa(kappa * C0 + MAGIC) = u + 0x4040, and the bytes of (that << 1) are (2 s0 + 128, s1 + 128, s2).
constexpr float C0 = 8355000.0f;        // u <= C0*(1+2e-3) keeps u + 0x4040 < 2^23
constexpr float MAGIC = 8388608.0f + 16448.0f;   // 2^23 + 0x4040

__device__ __forceinline__ uint32_t fixed_word(float kappa) { return __float_as_uint(fmaf(kappa, C0, MAGIC)) << 1; }
__device__ __forceinline__ uint32_t prmt(uint32_t a, uint32_t b, uint32_t sel) {
  uint32_t d;
  asm("prmt.b32 %0, %1, %2, %3;" : "=r"(d) : "r"(a), "r"(b), "r"(sel));
  return d;
}
// byte offset of (row r, byte k in [0,64)) inside a K-major SWIZZLE_64B tile with 64-byte rows
__device__ __forceinline__ uint32_t sw64_off(int r, int k) {
  return static_cast<uint32_t>((r >> 3) * 512 + (r & 7) * 64 + ((((k >> 4) ^ ((r >> 1) & 3))) << 4) + (k & 15));
}
// two neighbouring points (kappa words w0, w1) of one row -> the three digit planes at byte k, k+1
__device__ __forceinline__ void store_digits(uint8_t* planes, int plane_bytes, int r, int k, uint32_t w0, uint32_t w1) {
  const uint32_t off = sw64_off(r, k);
  *reinterpret_cast<uint16_t*>(planes + off) = static_cast<uint16_t>(prmt(w0, w1, 0x0040) ^ 0x8080u);                 // P0
  *reinterpret_cast<uint16_t*>(planes + plane_bytes + off) = static_cast<uint16_t>(prmt(w0, w1, 0x0051) ^ 0x8080u);   // P1
  *reinterpret_cast<uint16_t*>(planes + 2 * plane_bytes + off) = static_cast<uint16_t>(prmt(w0, w1, 0x0062));         // P2
}

// units [u_lo, u_lo + nu) of point slice `slice` of n_slices (the producer and the Gram each split a launch their own way)
__device__ __forceinline__ long long slice_units(long long n_units, int n_slices, int slice, long long* u_lo) {
  const long long ups = (n_units + n_slices - 1) / n_slices;
  *u_lo = ups * slice;
  long long u_hi = *u_lo + ups;
  if (u_hi > n_units) u_hi = n_units;
  return u_hi > *u_lo ? u_hi - *u_lo : 0;
}

struct PlaneParams {
  const uint8_t* Xt;    // tensor mode: [n_units][nchunks][8192] fp16 images; direct: [n_units][n_terms][dpad4][64] fp32
  const float* ys;      // [n_units*64]
  const uint8_t* Zt;    // tensor mode: [nt][nchunks][16384]; direct: [nt][n_terms][dpad4][128 rows] fp32, negated
  long long n_units;
  uint32_t xbytes, zbytes;
  int n_terms, dpad4;   // direct mode
  float w[4];           // term weights C_t / sum_t C_t
  int m_pad, nt, n_slices;
  uint8_t* planes;      // [n_units][nt][TILE_PLANES]
  double* bpart;        // [n_slices][m_pad]
  double bscale;        // C
  int accumulate;       // 0: store b, 1: add to it (later windows of one call)
  float* dbg_T;         // optional [128*64] : T of tile 0, unit 0
  uint32_t* dbg_w;      // optional [128*64] : fixed-point words of the same tile
};

// KS: 16-column k-steps of the tensor-mode distance contraction (4 for d <= 16, 7 for d <= 32; unused in direct mode).
template <bool DIRECT, int KS>
__global__ void __launch_bounds__(NTHREADS, 1) kmn_i8_planes_kernel(const PlaneParams p) {
  extern __shared__ uint8_t smem_raw[];
  const uint32_t raw = smem_u32(smem_raw);
  const uint32_t base = (raw + 1023u) & ~1023u;
  uint8_t* sm = smem_raw + (base - raw);
  const uint32_t s_pl = base;                                 // [2 buffers][P0 P1 P2]
  const uint32_t s_zt = s_pl + 2 * TILE_PLANES;               // active tile
  const uint32_t s_xs = s_zt + p.zbytes;                      // [XSTAGES][xbytes]
  const uint32_t s_ys = s_xs + XSTAGES * p.xbytes;            // [XSTAGES][64] float
  const uint32_t s_bar = s_ys + XSTAGES * UP * 4;             // zfull, xfull[XSTAGES]
  const uint32_t b_zfull = s_bar, b_xfull = s_bar + 8;

  const int tid = threadIdx.x, wg = tid >> 7, wq = (tid >> 5) & 3, lane = tid & 31;
  const int ti = blockIdx.x;
  long long u_lo;
  const long long nu = slice_units(p.n_units, p.n_slices, blockIdx.y, &u_lo);
  double* bp = p.bpart + static_cast<size_t>(blockIdx.y) * p.m_pad + ti * kTile;
  if (nu == 0) {   // empty slice: its b partial must still be defined
    if (!p.accumulate && tid < kTile) bp[tid] = 0.0;
    return;
  }

  auto issue_unit = [&](long long i, int s) {
    mbar_expect_tx(b_xfull + 8 * s, p.xbytes + UP * 4);
    bulk_g2s(s_xs + s * p.xbytes, p.Xt + static_cast<size_t>(u_lo + i) * p.xbytes, p.xbytes, b_xfull + 8 * s);
    bulk_g2s(s_ys + s * UP * 4, p.ys + static_cast<size_t>(u_lo + i) * UP, UP * 4, b_xfull + 8 * s);
  };
  if (tid == 0) {
    mbar_init(b_zfull, 1);
    for (int s = 0; s < XSTAGES; ++s) mbar_init(b_xfull + 8 * s, 1);
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();
  if (tid == 0) {
    mbar_expect_tx(b_zfull, p.zbytes);
    bulk_g2s(s_zt, p.Zt + static_cast<size_t>(ti) * p.zbytes, p.zbytes, b_zfull);
    for (long long i = 0; i < XSTAGES && i < nu; ++i) issue_unit(i, static_cast<int>(i));
  }

  // fragment coordinates of a wgmma m64n64 accumulator: element 4j+e sits at row r0 (+8 if e >= 2), point 8j + c0 + (e & 1)
  const int r0 = 16 * wq + (lane >> 2), c0 = 2 * (lane & 3);
  const int R = 64 * wg + r0;             // tile row (of 128) of this thread's first fragment row
  double bsum0 = 0.0, bsum1 = 0.0;

  mbar_wait(b_zfull, 0);
  for (long long i = 0; i < nu; ++i) {
    const int s = static_cast<int>(i % XSTAGES);
    mbar_wait(b_xfull + 8 * s, static_cast<uint32_t>((i / XSTAGES) & 1));
    const uint32_t xst = s_xs + s * p.xbytes;

    float T[32];
    if constexpr (!DIRECT) {
      wg_fence();
#pragma unroll
      for (int k = 0; k < KS; ++k) {
        const uint32_t za = s_zt + (k >> 2) * ZPANEL_BYTES + wg * 8192 + (k & 3) * 32;
        const uint32_t xb = xst + (k >> 2) * XIMG_BYTES + (k & 3) * 32;
        wgmma_f16_n64(T, desc_sw128(za), desc_sw128(xb), k > 0);
      }
      wg_commit();
      wg_wait<0>();
      if (p.dbg_T && i == 0 && blockIdx.x == 0 && blockIdx.y == 0) {
#pragma unroll
        for (int e = 0; e < 32; ++e) p.dbg_T[(R + ((e & 2) ? 8 : 0)) * UP + 8 * (e >> 2) + c0 + (e & 1)] = T[e];
      }
#pragma unroll
      for (int e = 0; e < 32; ++e) T[e] = ex2f(T[e]);
    } else {
#pragma unroll
      for (int e = 0; e < 32; ++e) T[e] = 0.f;
      // kappa = sum_t w_t 2^(-|x~_t - z~_t|^2), direct form (no cancellation: any norms)
      const float* xs = reinterpret_cast<const float*>(sm + (xst - base));
      const float* zt = reinterpret_cast<const float*>(sm + (s_zt - base));
      for (int t = 0; t < p.n_terms; ++t) {
        float q[32];
#pragma unroll
        for (int e = 0; e < 32; ++e) q[e] = 0.f;
        const float* xt = xs + t * p.dpad4 * UP;
        const float* ztt = zt + t * p.dpad4 * kTile;
#pragma unroll 2
        for (int k = 0; k < p.dpad4; ++k) {
          const float a0 = ztt[k * kTile + R], a1 = ztt[k * kTile + R + 8];      // stored negated
          const float* xk = xt + k * UP + c0;
#pragma unroll
          for (int j = 0; j < 8; ++j) {
            const float2 x = *reinterpret_cast<const float2*>(xk + 8 * j);
            float e0 = x.x + a0, e1 = x.y + a0, e2 = x.x + a1, e3 = x.y + a1;
            q[4 * j + 0] = fmaf(e0, e0, q[4 * j + 0]); q[4 * j + 1] = fmaf(e1, e1, q[4 * j + 1]);
            q[4 * j + 2] = fmaf(e2, e2, q[4 * j + 2]); q[4 * j + 3] = fmaf(e3, e3, q[4 * j + 3]);
          }
        }
        const float wt = p.w[t];
#pragma unroll
        for (int e = 0; e < 32; ++e) T[e] = fmaf(wt, ex2f(-q[e]), T[e]);
      }
    }

    {   // b: fp32 over the unit's points, fp64 across units
      const float* yv = reinterpret_cast<const float*>(sm + (s_ys - base)) + s * UP + c0;
      float b0 = 0.f, b1 = 0.f;
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        const float2 y2 = *reinterpret_cast<const float2*>(yv + 8 * j);
        b0 = fmaf(T[4 * j + 0], y2.x, fmaf(T[4 * j + 1], y2.y, b0));
        b1 = fmaf(T[4 * j + 2], y2.x, fmaf(T[4 * j + 3], y2.y, b1));
      }
      bsum0 += static_cast<double>(b0);
      bsum1 += static_cast<double>(b1);
    }

    // point stage s is consumed; plane buffer i&1 is free once the bulk store of unit i-2 has read it
    if (tid == 0) bulk_wait_read<1>();
    __syncthreads();
    if (tid == 0 && i + XSTAGES < nu) issue_unit(i + XSTAGES, s);

    uint8_t* planes = sm + (s_pl - base) + static_cast<int>(i & 1) * TILE_PLANES;
    const bool dbg = p.dbg_w != nullptr && i == 0 && blockIdx.x == 0 && blockIdx.y == 0;
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      const uint32_t w0 = fixed_word(T[4 * j + 0]), w1 = fixed_word(T[4 * j + 1]);
      const uint32_t w2 = fixed_word(T[4 * j + 2]), w3 = fixed_word(T[4 * j + 3]);
      store_digits(planes, PLANE, R, 8 * j + c0, w0, w1);
      store_digits(planes, PLANE, R + 8, 8 * j + c0, w2, w3);
      if (dbg) {
        const int k = 8 * j + c0;
        p.dbg_w[R * UP + k] = w0 >> 1; p.dbg_w[R * UP + k + 1] = w1 >> 1;
        p.dbg_w[(R + 8) * UP + k] = w2 >> 1; p.dbg_w[(R + 8) * UP + k + 1] = w3 >> 1;
      }
    }
    fence_proxy_async();
    __syncthreads();     // planes of unit i complete
    if (tid == 0) {
      bulk_s2g(p.planes + (static_cast<size_t>(u_lo + i) * p.nt + ti) * TILE_PLANES,
               s_pl + static_cast<uint32_t>(i & 1) * TILE_PLANES, TILE_PLANES);
      bulk_commit();
    }
  }
  if (tid == 0) bulk_wait<0>();

  // a row's 64 points are spread over the 4 lanes of a quad
  bsum0 += __shfl_xor_sync(0xffffffffu, bsum0, 1);
  bsum0 += __shfl_xor_sync(0xffffffffu, bsum0, 2);
  bsum1 += __shfl_xor_sync(0xffffffffu, bsum1, 1);
  bsum1 += __shfl_xor_sync(0xffffffffu, bsum1, 2);
  if ((lane & 3) == 0) {
    if (p.accumulate) {
      bp[R] += p.bscale * bsum0;
      bp[R + 8] += p.bscale * bsum1;
    } else {
      bp[R] = p.bscale * bsum0;
      bp[R + 8] = p.bscale * bsum1;
    }
  }
}

struct GramI8Params {
  const uint8_t* planes;   // [n_units][nt][TILE_PLANES]
  long long n_units;
  int m_pad, nt, n_slices;
  double* Gpart;           // [n_slices][m_pad*m_pad]
  double gscale;           // C^2 / (4 C0^2)
  int accumulate;          // 0: the first fold stores, 1: every fold adds (later windows of one call)
};

__global__ void __launch_bounds__(GTHREADS, 1) gram_i8_kernel(const GramI8Params p) {
  extern __shared__ uint8_t smem_raw[];
  const uint32_t raw = smem_u32(smem_raw);
  const uint32_t base = (raw + 1023u) & ~1023u;
  const uint32_t s_st = base;                                  // [GSTAGES][I planes | J planes]
  const uint32_t b_full = s_st + GSTAGES * 2 * TILE_PLANES;    // [GSTAGES]
  const uint32_t b_empty = b_full + 8 * GSTAGES;               // [GSTAGES]

  const int tid = threadIdx.x, wg = tid >> 7, wq = (tid >> 5) & 3, lane = tid & 31;
  int ti, tj;
  {
    int t = blockIdx.x;
    tj = 0;
    while (t >= p.nt - tj) { t -= p.nt - tj; ++tj; }
    ti = tj + t;
  }
  const bool diag = ti == tj;
  long long u_lo;
  const long long nu = slice_units(p.n_units, p.n_slices, blockIdx.y, &u_lo);

  // partial tile stored TRANSPOSED (mirror position, upper block triangle; gram_reduce_upper reads it):
  // element (row R of tile I, column c of tile J) at Gp[(tj*128 + c) * m_pad + ti*128 + R]
  double* gtile = p.Gpart + static_cast<size_t>(blockIdx.y) * p.m_pad * p.m_pad +
                  static_cast<size_t>(tj * kTile) * p.m_pad + ti * kTile;
  if (nu == 0) {   // empty slice: the partial tile must still be defined
    if (!p.accumulate)
      for (int e = tid; e < kTile * kTile; e += GTHREADS) gtile[static_cast<size_t>(e / kTile) * p.m_pad + (e % kTile)] = 0.0;
    return;
  }

  if (tid == 0) {
    for (int s = 0; s < GSTAGES; ++s) {
      mbar_init(b_full + 8 * s, 1);
      mbar_init(b_empty + 8 * s, 2);      // one arrival per consumer warpgroup
    }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();

  if (wg == 0) {   // ---- copy warpgroup: one thread streams the plane images of tiles I and J -------------------------
    setmaxnreg_dec<COPY_REGS>();
    if (tid == 0) {
      const uint32_t bytes = diag ? TILE_PLANES : 2 * TILE_PLANES;
      for (long long i = 0; i < nu; ++i) {
        const int s = static_cast<int>(i % GSTAGES);
        if (i >= GSTAGES) mbar_wait(b_empty + 8 * s, static_cast<uint32_t>(((i / GSTAGES) & 1) ^ 1));
        const uint8_t* src = p.planes + static_cast<size_t>(u_lo + i) * p.nt * TILE_PLANES;
        const uint32_t dst = s_st + s * 2 * TILE_PLANES;
        mbar_expect_tx(b_full + 8 * s, bytes);
        bulk_g2s(dst, src + static_cast<size_t>(ti) * TILE_PLANES, TILE_PLANES, b_full + 8 * s);
        if (!diag) bulk_g2s(dst + TILE_PLANES, src + static_cast<size_t>(tj) * TILE_PLANES, TILE_PLANES, b_full + 8 * s);
      }
      // the consumers spin on the full barriers without a bound: waiting here for their release of the last stages
      // keeps a copy that never lands a trap, not a hang
      for (long long i = nu > GSTAGES ? nu - GSTAGES : 0; i < nu; ++i)
        mbar_wait(b_empty + 8 * static_cast<int>(i % GSTAGES), static_cast<uint32_t>((i / GSTAGES) & 1));
    }
    return;
  }

  // ---- consumer warpgroups: rows 64 cw .. 64 cw + 63 of tile I against the 128 rows of tile J --------------------------
  setmaxnreg_inc<MMA_REGS>();
  const int cw = wg - 1;
  // fragment coordinates of a wgmma m64n128 accumulator: element 4j+e sits at row r0 (+8 if e >= 2), column 8j + c0 + (e & 1)
  const int r0 = 16 * wq + (lane >> 2), c0 = 2 * (lane & 3);
  const int R = 64 * cw + r0;
  int acc4[64], acc3[64], acc2[64];    // restarted (not zeroed) by the first MMAs after each fold
  int until_flush = FLUSH_UNITS;
  bool first_flush = !p.accumulate, fresh = true;

  for (long long i = 0; i < nu; ++i) {
    const int s = static_cast<int>(i % GSTAGES);
    mbar_wait_spin(b_full + 8 * s, static_cast<uint32_t>((i / GSTAGES) & 1));
    const uint32_t st = s_st + s * 2 * TILE_PLANES;
    const uint32_t a_base = st + cw * 4096;                    // 64 rows of the I planes
    const uint32_t b_base = diag ? st : st + TILE_PLANES;      // all 128 rows of the J planes
    wg_fence();
#pragma unroll
    for (int ks = 0; ks < 2; ++ks) {   // 2 k-steps of 32 points
      const uint64_t A0 = desc_sw64(a_base + 32 * ks), A1 = desc_sw64(a_base + PLANE + 32 * ks),
                     A2 = desc_sw64(a_base + 2 * PLANE + 32 * ks);
      const uint64_t B0 = desc_sw64(b_base + 32 * ks), B1 = desc_sw64(b_base + PLANE + 32 * ks),
                     B2 = desc_sw64(b_base + 2 * PLANE + 32 * ks);
      const int acc = (ks == 0 && fresh) ? 0 : 1;
      wgmma_uu(acc4, A2, B2, acc);              // weight 2^32 : P2'P2
      wgmma_us(acc3, A2, B1, acc);              // weight 2^24 : P2'P1 + P1'P2
      wgmma_su(acc3, A1, B2, 1);
      wgmma_us(acc2, A2, B0, acc);              // weight 2^16 : P2'P0 + P0'P2 + P1'P1
      wgmma_su(acc2, A0, B2, 1);
      wgmma_ss(acc2, A1, B1, 1);
    }
    wg_commit();
    fresh = false;
    wg_wait<1>();                               // the MMAs of unit i-1 are done: release its stage
    if (i >= 1 && (tid & 127) == 0) mbar_arrive(b_empty + 8 * static_cast<int>((i - 1) % GSTAGES));

    if (--until_flush == 0 || i == nu - 1) {
      // ---- fold the exact int32 accumulators into the fp64 partial tile -----------------------------------------
      until_flush = FLUSH_UNITS;
      wg_wait<0>();
      // the row stride, read through an opaque move: the column addresses are formed here, not hoisted out of the
      // unit loop into registers the accumulators need
      uint32_t ld;
      asm volatile("mov.b32 %0, %1;" : "=r"(ld) : "r"(static_cast<uint32_t>(p.m_pad)));
      double* const trow = gtile + R;
      const auto at = [&](int e) {
        return trow + static_cast<size_t>(8 * (e >> 2) + c0 + (e & 1)) * ld + ((e & 2) ? 8 : 0);
      };
      // the compiler cannot tell the elements' addresses apart, so a load after a store waits for it: each batch reads
      // all its old values before it writes any, FB loads in flight instead of one (in the registers of the accumulators
      // already folded; a batch of 16 spills under MMA_REGS)
      constexpr int FB = 8;
#pragma unroll
      for (int e0 = 0; e0 < 64; e0 += FB) {
        double old[FB];
#pragma unroll
        for (int k = 0; k < FB; ++k) old[k] = first_flush ? 0.0 : *at(e0 + k);
#pragma unroll
        for (int k = 0; k < FB; ++k) {
          const int e = e0 + k;
          const double v = p.gscale * (4294967296.0 * static_cast<double>(acc4[e]) + 16777216.0 * static_cast<double>(acc3[e]) +
                                       65536.0 * static_cast<double>(acc2[e]));
          *at(e) = first_flush ? v : old[k] + v;
        }
      }
      first_flush = false;
      fresh = true;
    }
  }
  if ((tid & 127) == 0) mbar_arrive(b_empty + 8 * static_cast<int>((nu - 1) % GSTAGES));   // the last unit's stage
}

}  // namespace

// Point slices of the Gram: pick the slice count (<= 16) that minimises (waves x units per slice), counting two CTA
// slots per tile of the upper block triangle.  The Gram kernel runs one CTA per tile, so its grid is half that count:
// configs[1] (m_pad = 1024) gets 11 slices x 36 tiles = 396 CTAs, three full waves on 132 SMs.
int i8_slices(int m_pad, int num_sms, long long n_units) {
  const int nt = m_pad / kTile;
  const long long ctas = static_cast<long long>(nt) * (nt + 1);
  int best = 1;
  long long best_cost = -1;
  for (int s = 1; s <= 16 && s <= n_units; ++s) {
    const long long waves = (ctas * s + num_sms - 1) / num_sms;
    const long long cost = waves * ((n_units + s - 1) / s);
    if (best_cost < 0 || cost < best_cost) { best = s; best_cost = cost; }
  }
  return best;
}

namespace {
// the producer variant of a launch: its kernel, point and active-tile image bytes, and dynamic shared memory
const void* plane_kernel(int d, const I8Direct& direct, uint32_t* xbytes, uint32_t* zbytes, size_t* smem) {
  const int nchunks = i8_nchunks(d);    // 64-column K chunks of the distance contraction (1 or 2)
  *xbytes = static_cast<uint32_t>(nchunks * XIMG_BYTES);
  *zbytes = static_cast<uint32_t>(nchunks * ZPANEL_BYTES);
  if (direct.on) {
    *xbytes = static_cast<uint32_t>(direct.n_terms * UP * direct.dpad4 * sizeof(float));
    *zbytes = static_cast<uint32_t>(direct.n_terms * kTile * direct.dpad4 * sizeof(float));
  }
  *smem = 1024 + 2 * TILE_PLANES + *zbytes + XSTAGES * (*xbytes + UP * 4) + 8 * (XSTAGES + 1);
  const int dp = (d + 15) / 16 * 16;
  return direct.on ? reinterpret_cast<const void*>(kmn_i8_planes_kernel<true, 0>)
         : (3 * dp + 16) / 16 == 4 ? reinterpret_cast<const void*>(kmn_i8_planes_kernel<false, 4>)
                                   : reinterpret_cast<const void*>(kmn_i8_planes_kernel<false, 7>);
}
}  // namespace

// Point slices of the producer: the planes are indexed by global unit, so its split need not match the Gram's.  The
// grid (active tiles x slices) is the largest that runs in one wave at the occupancy the variant's shared memory allows:
// configs[1] (8 tiles, d = 16: two CTAs per SM) gets 33 slices = 264 CTAs on 132 SMs, where the Gram's split gave 88.
cudaError_t i8_plane_slices(int m_pad, int num_sms, long long n_units, int d, const I8Direct& direct, int* n_slices) {
  uint32_t xbytes, zbytes;
  size_t smem;
  const void* fn = plane_kernel(d, direct, &xbytes, &zbytes, &smem);
  if (smem > kSmemOptInMax) return cudaErrorInvalidConfiguration;
  cudaError_t e = allow_dynamic_smem(fn);
  if (e != cudaSuccess) return e;
  int per_sm = 0;
  e = cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, fn, NTHREADS, smem);
  if (e != cudaSuccess) return e;
  if (per_sm < 1) return cudaErrorInvalidConfiguration;
  const long long s = std::min<long long>(static_cast<long long>(num_sms) * per_sm / (m_pad / kTile), n_units);
  *n_slices = static_cast<int>(std::max<long long>(s, 1));
  return cudaSuccess;
}

cudaError_t launch_i8_planes(const uint8_t* Xt, const float* ys, const uint8_t* Zt, long long n_units, int d, int m_pad,
                             int n_slices, const I8Direct& direct, double C, bool accumulate, uint8_t* planes,
                             double* bpart, float* dbg_T, uint32_t* dbg_w, cudaStream_t s) {
  PlaneParams p{};
  p.Xt = Xt; p.ys = ys; p.Zt = Zt;
  p.n_units = n_units;
  p.m_pad = m_pad; p.nt = m_pad / kTile; p.n_slices = n_slices;
  p.planes = planes; p.bpart = bpart;
  p.bscale = C;
  p.accumulate = accumulate ? 1 : 0;
  p.dbg_T = dbg_T; p.dbg_w = dbg_w;
  if (direct.on) {
    p.n_terms = direct.n_terms; p.dpad4 = direct.dpad4;
    for (int t = 0; t < 4; ++t) p.w[t] = direct.w[t];
  }
  size_t smem;
  const void* fn = plane_kernel(d, direct, &p.xbytes, &p.zbytes, &smem);
  if (smem > kSmemOptInMax) return cudaErrorInvalidConfiguration;
  // the cap is per device and shared by every context on it (one per task thread, on one or several GPUs): set on
  // every launch, to the one value allow_dynamic_smem gives every launch of this kernel, never to this launch's smem
  cudaError_t e = allow_dynamic_smem(fn);
  if (e != cudaSuccess) return e;
  dim3 grid(p.nt, n_slices);
  void* args[] = {&p};
  return cudaLaunchKernel(fn, grid, dim3(NTHREADS), args, smem, s);
}

cudaError_t launch_gram_i8(const uint8_t* planes, long long n_units, int m_pad, int n_slices, double C, bool accumulate,
                           double* Gpart, cudaStream_t s) {
  GramI8Params p{};
  p.planes = planes;
  p.n_units = n_units;
  p.m_pad = m_pad; p.nt = m_pad / kTile; p.n_slices = n_slices;
  p.Gpart = Gpart;
  p.gscale = C * C / (4.0 * static_cast<double>(C0) * static_cast<double>(C0));      // the planes are the digits of 2 u
  p.accumulate = accumulate ? 1 : 0;
  const size_t smem = 1024 + GSTAGES * 2 * TILE_PLANES + 16 * GSTAGES;
  const void* fn = reinterpret_cast<const void*>(gram_i8_kernel);
  cudaError_t e = allow_dynamic_smem(fn);
  if (e != cudaSuccess) return e;
  dim3 grid(p.nt * (p.nt + 1) / 2, n_slices);
  void* args[] = {&p};
  return cudaLaunchKernel(fn, grid, dim3(GTHREADS), args, smem, s);
}

}  // namespace sgp
