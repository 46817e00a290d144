// Fused K_mn + Gram kernel on the Hopper tensor cores (wgmma), exact-accumulation path.
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
// One CTA (256 threads = two warpgroups) owns the half tile  rows I-tile (128 active points) x 64 columns (half h of
// J-tile), I >= J, and a slice of the shard's 64-point units; its three 64 x 64 int32 accumulators per warpgroup live in
// registers (96 per thread).  Per unit:
//   distances  tensor mode: T = -q*log2(e) as ONE fp16 wgmma contraction over the hi/lo split of the scaled, centred
//              coordinates with the norms folded in as extra K columns (images from launch_i8_prep_points); panel I
//              (warpgroup w: rows 64w.., m64n64) and, off the diagonal, the 64 rows of panel J (warpgroup w: points 32w..,
//              m64n32).  Direct mode: sum of up to 4 terms of 2^(-|x~ - z~|^2) from fp32 coordinates on the CUDA cores,
//              at the same fragment positions.
//   epilogue   ex2 -> fixed point via one FFMA against 2^23 -> byte planes (PRMT) -> K-major SWIZZLE_64B int8 planes in
//              shared memory (double buffered), b += kappa*y on diagonal tiles.
//   Gram       12 int8 wgmma m64n64k32 per warpgroup (6 products x 2 k-steps of 32 points), issued asynchronously: they
//              run while the next unit's distances are contracted.  Every 400 units the accumulators are folded into
//              the fp64 partial tile (no overflow possible).
// Operands arrive by bulk copy (cp.async.bulk, completion on an mbarrier) into a ring of point stages.
#include <cuda_fp16.h>

#include "hopper.cuh"
#include "sgp_internal.h"

namespace sgp {
namespace {

using namespace hop;

constexpr int UP = 64;                  // points per pipeline unit
constexpr int NTHREADS = 256;           // two warpgroups
constexpr int XSTAGES_MAX = 8;
constexpr int ZPANEL_BYTES = 16384;     // fp16 active-set operand image: 128 rows x 128 bytes, SWIZZLE_128B K-major
constexpr int XIMG_BYTES = 8192;        // fp16 point operand image: 64 rows x 128 bytes
constexpr int PLANE_I = 8192;           // int8 digit plane of panel I: 128 rows x 64 points, K-major SWIZZLE_64B
constexpr int PLANE_J = 4096;           // ... of the 64 rows of panel J this CTA multiplies with
constexpr int PLANES_BYTES = 3 * PLANE_I + 3 * PLANE_J;
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

struct I8Params {
  const uint8_t* Xt;    // tensor mode: [n_units][nchunks][8192] fp16 images; direct: [n_units][n_terms][dpad4][64] fp32
  const float* ys;      // [n_units*64]
  const uint8_t* Zt;    // tensor mode: [nt][nchunks][16384]; direct: [nt][n_terms][dpad4][128 rows] fp32, negated
  long long n_units;
  uint32_t xbytes, zbytes;
  int n_terms, dpad4;   // direct mode
  float w[4];           // term weights C_t / sum_t C_t
  int xstages;
  int m_pad, nt, n_slices;
  double* Gpart;        // [n_slices][m_pad*m_pad]
  double* bpart;        // [n_slices][m_pad]
  double gscale;        // C^2 / (4 C0^2)
  double bscale;        // C
  float* dbg_T;         // optional [128*64] : T of the first distance tile of CTA (0,0)
  uint32_t* dbg_w;      // optional [128*64] : fixed-point words of the same tile
};

// KS: 16-column k-steps of the tensor-mode distance contraction (4 for d <= 16, 7 for d <= 32; unused in direct mode).
// Every MMA of a unit is issued unconditionally (a branch around wgmma makes ptxas serialise them): on diagonal tiles the
// panel-J contraction runs against panel I and its result is not used.
template <bool DIRECT, int KS>
__global__ void __launch_bounds__(NTHREADS, 1) kmn_gram_i8_wgmma_kernel(const I8Params p) {
  extern __shared__ uint8_t smem_raw[];
  const uint32_t raw = smem_u32(smem_raw);
  const uint32_t base = (raw + 1023u) & ~1023u;
  uint8_t* sm = smem_raw + (base - raw);
  const uint32_t s_zi = base, s_zj = s_zi + p.zbytes;                 // active tiles I and J
  const uint32_t s_pl = s_zj + p.zbytes;                              // [2 buffers][PI0 PI1 PI2 PJ0 PJ1 PJ2]
  const uint32_t s_xs = s_pl + 2 * PLANES_BYTES;                      // [xstages][xbytes]
  const uint32_t s_ys = s_xs + p.xstages * p.xbytes;                  // [xstages][64] float
  const uint32_t s_bar = s_ys + p.xstages * UP * 4;                   // zfull, xfull[xstages]
  const uint32_t b_zfull = s_bar, b_xfull = s_bar + 8;

  const int tid = threadIdx.x, wg = tid >> 7, wq = (tid >> 5) & 3, lane = tid & 31;
  const int h = blockIdx.x & 1;
  int ti, tj;
  {
    int t = blockIdx.x >> 1;
    tj = 0;
    while (t >= p.nt - tj) { t -= p.nt - tj; ++tj; }
    ti = tj + t;
  }
  const bool diag = ti == tj;

  const long long ups = (p.n_units + p.n_slices - 1) / p.n_slices;
  const long long u_lo = ups * blockIdx.y;
  long long u_hi = u_lo + ups;
  if (u_hi > p.n_units) u_hi = p.n_units;
  const long long nu = u_hi > u_lo ? u_hi - u_lo : 0;

  double* Gp = p.Gpart + static_cast<size_t>(blockIdx.y) * p.m_pad * p.m_pad;
  double* bp = p.bpart + static_cast<size_t>(blockIdx.y) * p.m_pad;
  // partial tile stored TRANSPOSED (mirror position, upper block triangle; gram_reduce_upper reads it):
  // element (row R of tile I, column c of half h of tile J) at Gp[(tj*128 + 64h + c) * m_pad + ti*128 + R]
  double* gtile = Gp + static_cast<size_t>(tj * kTile + 64 * h) * p.m_pad + ti * kTile;

  if (nu == 0) {   // empty slice: the partial tile must still be defined
    for (int e = tid; e < 64 * kTile; e += NTHREADS) gtile[static_cast<size_t>(e / kTile) * p.m_pad + (e % kTile)] = 0.0;
    if (diag && h == 0 && tid < kTile) bp[ti * kTile + tid] = 0.0;
    return;
  }

  const int xs_n = p.xstages;
  auto issue_unit = [&](long long i, int s) {
    mbar_expect_tx(b_xfull + 8 * s, p.xbytes + UP * 4);
    bulk_g2s(s_xs + s * p.xbytes, p.Xt + static_cast<size_t>(u_lo + i) * p.xbytes, p.xbytes, b_xfull + 8 * s);
    bulk_g2s(s_ys + s * UP * 4, p.ys + static_cast<size_t>(u_lo + i) * UP, UP * 4, b_xfull + 8 * s);
  };
  if (tid == 0) {
    mbar_init(b_zfull, 1);
    for (int s = 0; s < xs_n; ++s) mbar_init(b_xfull + 8 * s, 1);
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();
  if (tid == 0) {
    mbar_expect_tx(b_zfull, diag ? p.zbytes : 2 * p.zbytes);
    bulk_g2s(s_zi, p.Zt + static_cast<size_t>(ti) * p.zbytes, p.zbytes, b_zfull);
    if (!diag) bulk_g2s(s_zj, p.Zt + static_cast<size_t>(tj) * p.zbytes, p.zbytes, b_zfull);
    for (long long i = 0; i < xs_n && i < nu; ++i) issue_unit(i, static_cast<int>(i));
  }

  // fragment coordinates of a wgmma m64nN accumulator: element 4j+e sits at row r0 (+8 if e >= 2), column 8j + c0 + (e & 1)
  const int r0 = 16 * wq + (lane >> 2), c0 = 2 * (lane & 3);
  const int RI = 64 * wg + r0;            // panel-I row (of 128) of this thread's first fragment row

  int acc4[32], acc3[32], acc2[32];
#pragma unroll
  for (int e = 0; e < 32; ++e) acc4[e] = acc3[e] = acc2[e] = 0;
  double bsum0 = 0.0, bsum1 = 0.0;
  int until_flush = FLUSH_UNITS;
  bool first_flush = true;
  const bool want_b = diag && h == 0;

  mbar_wait(b_zfull, 0);
  for (long long i = 0; i < nu; ++i) {
    const int s = static_cast<int>(i % xs_n);
    // stage (i-1) % xs_n was released by every thread at the barrier of unit i-1
    if (tid == 0 && i >= 1 && i + xs_n - 1 < nu) issue_unit(i + xs_n - 1, static_cast<int>((i - 1) % xs_n));
    mbar_wait(b_xfull + 8 * s, static_cast<uint32_t>((i / xs_n) & 1));
    const uint32_t xst = s_xs + s * p.xbytes;

    float TI[32], TJ[16];
    if constexpr (!DIRECT) {
      const uint32_t za = s_zi + wg * 8192, zja = (diag ? s_zi : s_zj) + h * 8192;
      wg_fence();
#pragma unroll
      for (int k = 0; k < KS; ++k) {
        const uint32_t off = (k >> 2) * ZPANEL_BYTES + (k & 3) * 32, xoff = (k >> 2) * XIMG_BYTES + (k & 3) * 32;
        wgmma_f16_n64(TI, desc_sw128(za + off), desc_sw128(xst + xoff), k > 0);
        wgmma_f16_n32(TJ, desc_sw128(zja + off), desc_sw128(xst + wg * 4096 + xoff), k > 0);
      }
      wg_commit();
      wg_wait<0>();      // also drains this warpgroup's Gram MMAs of unit i-1
      if (p.dbg_T && i == 0 && blockIdx.x == 0 && blockIdx.y == 0) {
#pragma unroll
        for (int e = 0; e < 32; ++e) p.dbg_T[(RI + ((e & 2) ? 8 : 0)) * UP + 8 * (e >> 2) + c0 + (e & 1)] = TI[e];
      }
#pragma unroll
      for (int e = 0; e < 32; ++e) TI[e] = ex2f(TI[e]);
#pragma unroll
      for (int e = 0; e < 16; ++e) TJ[e] = ex2f(TJ[e]);
    } else {
#pragma unroll
      for (int e = 0; e < 32; ++e) TI[e] = 0.f;
#pragma unroll
      for (int e = 0; e < 16; ++e) TJ[e] = 0.f;
      wg_wait<0>();
      // kappa = sum_t w_t 2^(-|x~_t - z~_t|^2), direct form (no cancellation: any norms)
      const float* xs = reinterpret_cast<const float*>(sm + (xst - base));
      const float* zi = reinterpret_cast<const float*>(sm + (s_zi - base));
      const float* zj = reinterpret_cast<const float*>(sm + ((diag ? s_zi : s_zj) - base));
      const int pi0 = RI, pi1 = RI + 8, pj0 = 64 * h + r0, pj1 = 64 * h + r0 + 8;
      for (int t = 0; t < p.n_terms; ++t) {
        float qi[32], qj[16];
#pragma unroll
        for (int e = 0; e < 32; ++e) qi[e] = 0.f;
#pragma unroll
        for (int e = 0; e < 16; ++e) qj[e] = 0.f;
        const float* xt = xs + t * p.dpad4 * UP;
        const float* zit = zi + t * p.dpad4 * kTile;
        const float* zjt = zj + t * p.dpad4 * kTile;
#pragma unroll 2
        for (int k = 0; k < p.dpad4; ++k) {
          const float a0 = zit[k * kTile + pi0], a1 = zit[k * kTile + pi1];      // stored negated
          const float* xk = xt + k * UP + c0;
#pragma unroll
          for (int j = 0; j < 8; ++j) {
            const float2 x = *reinterpret_cast<const float2*>(xk + 8 * j);
            float e0 = x.x + a0, e1 = x.y + a0, e2 = x.x + a1, e3 = x.y + a1;
            qi[4 * j + 0] = fmaf(e0, e0, qi[4 * j + 0]); qi[4 * j + 1] = fmaf(e1, e1, qi[4 * j + 1]);
            qi[4 * j + 2] = fmaf(e2, e2, qi[4 * j + 2]); qi[4 * j + 3] = fmaf(e3, e3, qi[4 * j + 3]);
          }
          if (!diag) {
            const float b0 = zjt[k * kTile + pj0], b1 = zjt[k * kTile + pj1];
#pragma unroll
            for (int j = 0; j < 4; ++j) {
              const float2 x = *reinterpret_cast<const float2*>(xk + 32 * wg + 8 * j);
              float e0 = x.x + b0, e1 = x.y + b0, e2 = x.x + b1, e3 = x.y + b1;
              qj[4 * j + 0] = fmaf(e0, e0, qj[4 * j + 0]); qj[4 * j + 1] = fmaf(e1, e1, qj[4 * j + 1]);
              qj[4 * j + 2] = fmaf(e2, e2, qj[4 * j + 2]); qj[4 * j + 3] = fmaf(e3, e3, qj[4 * j + 3]);
            }
          }
        }
        const float wt = p.w[t];
#pragma unroll
        for (int e = 0; e < 32; ++e) TI[e] = fmaf(wt, ex2f(-qi[e]), TI[e]);
#pragma unroll
        for (int e = 0; e < 16; ++e) TJ[e] = fmaf(wt, ex2f(-qj[e]), TJ[e]);
      }
    }

    // ---- epilogue: b on diagonal tiles, digit planes of panel I (and of the 64 rows of panel J) ----------------
    uint8_t* planes = sm + (s_pl - base) + static_cast<int>(i & 1) * PLANES_BYTES;
    if (want_b) {
      const float* yv = reinterpret_cast<const float*>(sm + (s_ys - base)) + s * UP + c0;
      float b0 = 0.f, b1 = 0.f;
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        const float2 y2 = *reinterpret_cast<const float2*>(yv + 8 * j);
        b0 = fmaf(TI[4 * j + 0], y2.x, fmaf(TI[4 * j + 1], y2.y, b0));
        b1 = fmaf(TI[4 * j + 2], y2.x, fmaf(TI[4 * j + 3], y2.y, b1));
      }
      bsum0 += static_cast<double>(b0);
      bsum1 += static_cast<double>(b1);
    }
    const bool dbg = p.dbg_w != nullptr && i == 0 && blockIdx.x == 0 && blockIdx.y == 0;
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      const uint32_t w0 = fixed_word(TI[4 * j + 0]), w1 = fixed_word(TI[4 * j + 1]);
      const uint32_t w2 = fixed_word(TI[4 * j + 2]), w3 = fixed_word(TI[4 * j + 3]);
      store_digits(planes, PLANE_I, RI, 8 * j + c0, w0, w1);
      store_digits(planes, PLANE_I, RI + 8, 8 * j + c0, w2, w3);
      if (dbg) {
        const int k = 8 * j + c0;
        p.dbg_w[RI * UP + k] = w0 >> 1; p.dbg_w[RI * UP + k + 1] = w1 >> 1;
        p.dbg_w[(RI + 8) * UP + k] = w2 >> 1; p.dbg_w[(RI + 8) * UP + k + 1] = w3 >> 1;
      }
    }
    if (!diag) {
      uint8_t* pj = planes + 3 * PLANE_I;
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        const int k = 32 * wg + 8 * j + c0;
        store_digits(pj, PLANE_J, r0, k, fixed_word(TJ[4 * j + 0]), fixed_word(TJ[4 * j + 1]));
        store_digits(pj, PLANE_J, r0 + 8, k, fixed_word(TJ[4 * j + 2]), fixed_word(TJ[4 * j + 3]));
      }
    }
    fence_proxy_async();
    __syncthreads();     // planes complete (both warpgroups); point stage s and its y released

    // ---- Gram: 6 products x 2 k-steps of 32 points, asynchronous -------------------------------------------------
    {
      const uint32_t pl = s_pl + static_cast<uint32_t>(i & 1) * PLANES_BYTES;
      const uint32_t a_base = pl + wg * 4096;
      const uint32_t b_base = diag ? pl + h * 4096 : pl + 3 * PLANE_I;
      const uint32_t b_stride = diag ? PLANE_I : PLANE_J;
      wg_fence();
#pragma unroll
      for (int ks = 0; ks < 2; ++ks) {
        const uint64_t A0 = desc_sw64(a_base + 32 * ks), A1 = desc_sw64(a_base + PLANE_I + 32 * ks),
                       A2 = desc_sw64(a_base + 2 * PLANE_I + 32 * ks);
        const uint64_t B0 = desc_sw64(b_base + 32 * ks), B1 = desc_sw64(b_base + b_stride + 32 * ks),
                       B2 = desc_sw64(b_base + 2 * b_stride + 32 * ks);
        wgmma_uu(acc4, A2, B2);                   // weight 2^32 : P2'P2
        wgmma_us(acc3, A2, B1);                   // weight 2^24 : P2'P1 + P1'P2
        wgmma_su(acc3, A1, B2);
        wgmma_us(acc2, A2, B0);                   // weight 2^16 : P2'P0 + P0'P2 + P1'P1
        wgmma_su(acc2, A0, B2);
        wgmma_ss(acc2, A1, B1);
      }
      wg_commit();
    }

    if (--until_flush == 0 || i == nu - 1) {
      // ---- fold the exact int32 accumulators into the fp64 partial tile ---------------------------------------
      until_flush = FLUSH_UNITS;
      wg_wait<0>();
#pragma unroll
      for (int e = 0; e < 32; ++e) {
        const int R = RI + ((e & 2) ? 8 : 0), c = 8 * (e >> 2) + c0 + (e & 1);
        const double v = p.gscale * (4294967296.0 * static_cast<double>(acc4[e]) + 16777216.0 * static_cast<double>(acc3[e]) +
                                     65536.0 * static_cast<double>(acc2[e]));
        double* dst = gtile + static_cast<size_t>(c) * p.m_pad + R;
        if (first_flush) *dst = v;
        else *dst += v;
        acc4[e] = acc3[e] = acc2[e] = 0;
      }
      first_flush = false;
    }
  }
  if (want_b) {
    // a row's 64 points are spread over the 4 lanes of a quad
    bsum0 += __shfl_xor_sync(0xffffffffu, bsum0, 1);
    bsum0 += __shfl_xor_sync(0xffffffffu, bsum0, 2);
    bsum1 += __shfl_xor_sync(0xffffffffu, bsum1, 1);
    bsum1 += __shfl_xor_sync(0xffffffffu, bsum1, 2);
    if ((lane & 3) == 0) {
      bp[ti * kTile + RI] = p.bscale * bsum0;
      bp[ti * kTile + RI + 8] = p.bscale * bsum1;
    }
  }
}

}  // namespace

// Point slices of one launch: the grid has 2 * nt(nt+1)/2 CTAs per slice, one CTA per SM; pick the slice count (<= 16)
// that minimises (waves x units per slice).
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

cudaError_t launch_gram_i8(const uint8_t* Xt, const float* ys, const uint8_t* Zt, long long n, int d, int m_pad,
                           int n_slices, const I8Direct& direct, double* Gpart, double* bpart, double C, float* dbg_T,
                           uint32_t* dbg_w, cudaStream_t s) {
  I8Params p{};
  const int dp = (d + 15) / 16 * 16;
  p.Xt = Xt; p.ys = ys; p.Zt = Zt;
  p.n_units = (n + UP - 1) / UP;
  const int nchunks = i8_nchunks(d);    // 64-column K chunks of the distance contraction (1 or 2)
  p.m_pad = m_pad; p.nt = m_pad / kTile; p.n_slices = n_slices;
  p.Gpart = Gpart; p.bpart = bpart;
  p.dbg_T = dbg_T; p.dbg_w = dbg_w;
  p.xbytes = static_cast<uint32_t>(nchunks * XIMG_BYTES);
  p.zbytes = static_cast<uint32_t>(nchunks * ZPANEL_BYTES);
  if (direct.on) {
    p.n_terms = direct.n_terms; p.dpad4 = direct.dpad4;
    for (int t = 0; t < 4; ++t) p.w[t] = direct.w[t];
    p.xbytes = static_cast<uint32_t>(direct.n_terms * UP * direct.dpad4 * sizeof(float));
    p.zbytes = static_cast<uint32_t>(direct.n_terms * kTile * direct.dpad4 * sizeof(float));
    C = direct.csum;
  }
  p.gscale = C * C / (4.0 * static_cast<double>(C0) * static_cast<double>(C0));      // the planes are the digits of 2 u
  p.bscale = C;
  const long fixed = 1024 + 2L * p.zbytes + 2L * PLANES_BYTES + 8 * (XSTAGES_MAX + 1);
  long xs = (static_cast<long>(kSmemOptInMax) - fixed) / static_cast<long>(p.xbytes + UP * 4);
  if (xs > XSTAGES_MAX) xs = XSTAGES_MAX;
  if (xs < 2) return cudaErrorInvalidConfiguration;
  p.xstages = static_cast<int>(xs);
  const size_t smem = fixed + xs * (p.xbytes + UP * 4);
  const void* fn = direct.on ? reinterpret_cast<const void*>(kmn_gram_i8_wgmma_kernel<true, 0>)
                   : (3 * dp + 16) / 16 == 4 ? reinterpret_cast<const void*>(kmn_gram_i8_wgmma_kernel<false, 4>)
                                             : reinterpret_cast<const void*>(kmn_gram_i8_wgmma_kernel<false, 7>);
  // per-device attribute: set on every launch (contexts on several GPUs may live in one process)
  cudaError_t e = cudaFuncSetAttribute(fn, cudaFuncAttributeMaxDynamicSharedMemorySize, static_cast<int>(smem));
  if (e != cudaSuccess) return e;
  dim3 grid(p.nt * (p.nt + 1), n_slices);
  void* args[] = {&p};
  return cudaLaunchKernel(fn, grid, dim3(NTHREADS), args, smem, s);
}

}  // namespace sgp
