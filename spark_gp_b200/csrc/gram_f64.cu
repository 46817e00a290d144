// Fused K_mn + Gram kernel, parity-grade path (fp64 DMMA accumulation).
//
// Replaces, for one shard of points, the per-expert body of
//   commons/ProjectedGaussianProcessHelper.scala:27-29   (crossKernel; K_mn*K_mn^T; K_mn*y)
// including the kernel-DSL evaluation it calls
//   kernel/ARDRBFKernel.scala:43-46,81-89, kernel/RBFKernel.scala:66-76,
//   kernel/ScalarTimesKernel.scala:24, kernel/SumOfKernels.scala:57-58, kernel/Kernel.scala:157 (Eye -> 0).
//
// Decomposition.  G = sum_n k_n k_n^T with k_n = k(Z, x_n) in R^m is a plain sum over points (expert
// boundaries are irrelevant to it), so a CTA owns one 128x128 tile (I,J), I>=J, of the lower block
// triangle of G and one contiguous slice of the shard's points.  Per block of 16 points it
//   (1) evaluates the two panels P_I[16][128], P_J[16][128] of the cross kernel into shared memory
//       (direct-form sum_k (x~_k - z~_k)^2 on centred, pre-scaled coordinates x~ = (x - c)*beta with c within half
//       a standard deviation of the active-set mean; fp32 with ex2.approx (2 ulp, results below 2^-126 flushed to 0) by
//       default, fp64 with CUDA's exp in strict mode; the term scale C_t multiplies in fp64; Eye terms contribute nothing),
//   (2) accumulates  acc += P_I^T P_J  with fp64 tensor-core MMAs (mma.sync m8n8k4 f64), accumulators in
//       registers for the CTA's whole lifetime, and (diagonal tiles only) b_I += P_I^T y.
// At the end every CTA stores its tile into its slice's private partial buffer; a second tiny kernel sums
// the slices in a fixed order, mirrors the lower triangle and adds into the persistent fp64 [G;b]
// (deterministic: no atomics anywhere).
//
// Tile shapes.  Strict mode keeps the 128x128 tile (128 accumulator registers per thread, one CTA per SM).  The default
// mode uses 128x64 tiles (TN = 64): 64 accumulator registers per thread, so TWO CTAs fit on an SM and the panel phase
// (FMA / XU pipes) of one overlaps the DMMA phase of the other -- with one CTA per SM the two phases alternate.  Column tiles of 64 inside the 128-row
// diagonal block reuse the I panel (no second panel); the tile map is the staircase tj <= 2 ti + 1.
//
// Why fp64 accumulation: tools/precision_study.py -- the posterior mean needs the Gram accumulated to
// better than fp32 (fp16 hi/lo operands + fp32 accumulators already sit AT the 1e-5 parity bound for
// N=1e5 and degrade with N), while fp32-accurate *elements* with exact accumulation are 50x inside it.
#include <type_traits>

#include "sgp_internal.h"

namespace sgp {
namespace {

// f32x2 helpers on two scalar lanes (Hopper has no packed fp32 FADD/FFMA); round-to-nearest like the scalar ops
__device__ __forceinline__ float2 fadd2(float2 a, float2 b) { return make_float2(__fadd_rn(a.x, b.x), __fadd_rn(a.y, b.y)); }
__device__ __forceinline__ float2 ffma2(float2 a, float2 b, float2 c) {
  return make_float2(__fmaf_rn(a.x, b.x, c.x), __fmaf_rn(a.y, b.y, c.y));
}

constexpr int PB = 16;            // points per block (DMMA k extent per block = 4 steps of k=4)
constexpr int PS = kTile + 4;     // panel row stride (doubles): 132 -> conflict-free 8-byte fragment loads
constexpr int DC = 32;            // feature dims staged per chunk
constexpr int NT = 256;           // threads per CTA (8 warps: 4 x 2 grid of 32x64 warp tiles)

template <typename ET> struct ElemOps;
template <> struct ElemOps<float> {
  // coordinates are pre-scaled by sqrt(log2 e) at staging time, so exp(-q) = 2^(-q'): one MUFU.EX2 (2 ulp)
  static constexpr double kPrescale = kSqrtLog2e;
  static __device__ __forceinline__ float ex(float q) {
    float y;
    asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(-q));
    return y;
  }
  static __device__ __forceinline__ void ld4(const float* p, float (&v)[4]) {
    float4 t = *reinterpret_cast<const float4*>(p);
    v[0] = t.x; v[1] = t.y; v[2] = t.z; v[3] = t.w;
  }
};
template <> struct ElemOps<double> {
  static constexpr double kPrescale = 1.0;
  static __device__ __forceinline__ double ex(double q) { return exp(-q); }
  static __device__ __forceinline__ void ld4(const double* p, double (&v)[4]) {
    double2 a = *reinterpret_cast<const double2*>(p);
    double2 b = *reinterpret_cast<const double2*>(p + 2);
    v[0] = a.x; v[1] = a.y; v[2] = b.x; v[3] = b.y;
  }
};

__device__ __forceinline__ void dmma_m8n8k4(double (&c)[2], double a, double b) {
  asm volatile("mma.sync.aligned.m8n8k4.row.col.f64.f64.f64.f64 {%0,%1}, {%2}, {%3}, {%0,%1};\n"
               : "+d"(c[0]), "+d"(c[1])
               : "d"(a), "d"(b));
}

template <typename ET>
constexpr size_t gram_smem_bytes() {
  constexpr int NBUF = (sizeof(ET) == 4) ? 2 : 1;     // fp32 elements: panels and x staging are double buffered (pipelined loop)
  return sizeof(double) * (NBUF * 2 * PB * PS + 2 * PB) + sizeof(ET) * (DC * 256 + NBUF * PB * DC);
}

template <typename ET, int TN>
__global__ void __launch_bounds__(NT, (TN == 64) ? 2 : 1) kmn_gram_f64_kernel(const GramParams p) {
  constexpr int NJ = TN / 16;                                // 8-column B fragments per warp (warp tile 32 x TN/2)
  extern __shared__ __align__(16) unsigned char smem_raw[];
  constexpr int NBUF = (sizeof(ET) == 4) ? 2 : 1;
  double* panel = reinterpret_cast<double*>(smem_raw);      // [NBUF][2][PB][PS]
  double* ys2 = panel + NBUF * 2 * PB * PS;                  // [2][PB] (double buffered by block parity)
  ET* zs = reinterpret_cast<ET*>(ys2 + 2 * PB);              // [DC/4][256][4]
  ET* xs = zs + DC * 256;                                    // [NBUF][PB][DC]

  const int tid = threadIdx.x;
  const int lane = tid & 31, warp = tid >> 5;
  const int wr = warp >> 1, wc = warp & 1;

  // tile decode.  TN = 128: t -> (ti, tj), ti >= tj (triangular).  TN = 64: staircase, row tile ti owns column tiles
  // tj = 0 .. 2 ti + 1 (ti (ti + 1) tiles precede row ti).
  int ti, tj;
  {
    const int t = blockIdx.x;
    if (TN == 128) {
      ti = static_cast<int>((sqrtf(8.0f * t + 1.0f) - 1.0f) * 0.5f);
      while ((ti + 1) * (ti + 2) / 2 <= t) ++ti;
      while (ti * (ti + 1) / 2 > t) --ti;
      tj = t - ti * (ti + 1) / 2;
    } else {
      ti = static_cast<int>((sqrtf(4.0f * t + 1.0f) - 1.0f) * 0.5f);
      while ((ti + 1) * (ti + 2) <= t) ++ti;
      while (ti * (ti + 1) > t) --ti;
      tj = t - ti * (ti + 1);
    }
  }
  // column tiles inside the diagonal block read their B operand from the I panel
  const bool diag = (TN == 128) ? (ti == tj) : (tj >= 2 * ti);
  const int joff = (TN == 128) ? 0 : (tj - 2 * ti) * TN;      // offset of the J columns inside the I panel (diag only)
  const bool owns_b = (TN == 128) ? diag : (tj == 2 * ti);   // one tile per row tile accumulates b_I
  const int col = tid & 127, pan = tid >> 7;
  const int zrow = pan ? (tj * TN + col) : (ti * kTile + col);   // active-set index of this thread's column
  const bool zvalid = zrow < p.m;
  const bool elem_active = (pan == 0) || (!diag && col < TN);

  // slice of points
  const long long total_blocks = (p.n + PB - 1) / PB;
  const long long bps = (total_blocks + p.n_slices - 1) / p.n_slices;
  const long long blk_lo = bps * blockIdx.y;
  long long blk_hi = blk_lo + bps;
  if (blk_hi > total_blocks) blk_hi = total_blocks;

  constexpr bool kPacked = sizeof(ET) == 4;                  // fp32 elements: f32x2 arithmetic, z staged negated
  constexpr double kZSign = kPacked ? -1.0 : 1.0;
  const bool z_resident = (p.n_terms == 1 && p.dpad <= DC);

  // Both operands are centred on c (the row after the kMaxTerms beta rows of p.beta; within half a standard deviation of
  // the active-set mean) in fp64 before they are rounded to ET: x~ = (x - c) beta here, z~ = (Z - c) beta once per
  // begin() (p.Zc).  Uncentred, the rounding error of every staged coordinate would grow with |x| beta -- the distance
  // from the origin in length scales -- instead of with the spread of the data.
  static_assert(NT % DC == 0, "a thread stages the same feature dim of every point it stages");
  const double* centre = p.beta + kMaxTerms * p.dpad;
  const int kx = tid % DC;
  auto load_z_chunk = [&](int term, int c0, int clen) {
    // (threads 192..255 of a 128x64 tile have no column: their zrow may point past the padded active set)
    const bool in_range = zrow < p.m_pad;
    const double* src = p.Zc + (static_cast<size_t>(term) * p.m_pad + (in_range ? zrow : 0)) * p.dpad + c0;
    for (int k = 0; k < clen; ++k) zs[((k >> 2) * 256 + tid) * 4 + (k & 3)] = in_range ? static_cast<ET>(kZSign * ElemOps<ET>::kPrescale * src[k]) : ET(0);
  };
  auto load_x_chunk = [&](long long pt0, int term, int c0, int clen) {
    const int k = kx;
    const bool k_in = k < clen && c0 + k < p.d;
    const double ck = k_in ? centre[c0 + k] : 0.0;
    const double sk = k_in ? p.beta[term * p.dpad + c0 + k] * ElemOps<ET>::kPrescale : 0.0;
    for (int e = tid; e < PB * DC; e += NT) {
      const int pp = e / DC;
      const long long pt = pt0 + pp;
      double v = 0.0;
      if (k_in && pt < p.n) {
        const size_t off = static_cast<size_t>(pt) * p.d + c0 + k;
        v = p.x_is_f32 ? static_cast<double>(reinterpret_cast<const float*>(p.X)[off])
                       : reinterpret_cast<const double*>(p.X)[off];
        v = (v - ck) * sk;
      }
      xs[pp * DC + k] = static_cast<ET>(v);
    }
  };

  if (z_resident) load_z_chunk(0, 0, p.dpad);   // visible after the first __syncthreads below

  double acc[4][NJ][2];
#pragma unroll
  for (int i = 0; i < 4; ++i)
#pragma unroll
    for (int j = 0; j < NJ; ++j) acc[i][j][0] = acc[i][j][1] = 0.0;
  double bacc = 0.0;


  // ================= pipelined loop (fp32 elements, one kernel term, d <= 32: the common case) =========================
  // With the panel phase and the DMMA phase separated by barriers the tensor pipe idles while panels are built -- and
  // two co-resident CTAs do not fix that: they phase-lock (both share the pipe in the DMMA phase, finish together, then
  // both build panels): measured 45 % DMMA utilisation either way.  Here the DMMAs of block i and the panel build of
  // block i+1 sit in the same barrier-free region (double-buffered panels / x staging, ONE __syncthreads per block),
  // so warps drift apart and FFMA / MUFU work of some warps fills the issue slots of warps blocked on the tensor pipe.
  if constexpr (kPacked) {
    if (z_resident) {
      const int nk4 = p.dpad >> 2;                               // <= 8
      // this thread's two elements of a 16-point x 32-dim staging tile (both in feature dim kx)
      const int e0 = tid, e1 = tid + NT;
      const double ck = kx < p.d ? centre[kx] : 0.0, bk = kx < p.d ? p.beta[kx] : 0.0;
      auto fetch_x = [&](long long blk, int e) -> float {
        const int pp = e / DC, k = kx;
        const long long pt = blk * PB + pp;
        if (blk < blk_hi && k < p.d && pt < p.n) {
          const size_t off = static_cast<size_t>(pt) * p.d + k;
          const double v = p.x_is_f32 ? static_cast<double>(reinterpret_cast<const float*>(p.X)[off])
                                      : reinterpret_cast<const double*>(p.X)[off];
          return static_cast<float>((v - ck) * bk * ElemOps<ET>::kPrescale);
        }
        return 0.f;
      };
      auto panel_block = [&](long long blk, const float* xb, double* pbuf, int k4_lo, int k4_hi, float2 (&q)[PB]) {
        for (int k4 = k4_lo; k4 < k4_hi; ++k4) {
          const float4 z = *reinterpret_cast<const float4*>(zs + (k4 * 256 + tid) * 4);      // negated at staging
          const float2 z01 = make_float2(z.x, z.y), z23 = make_float2(z.z, z.w);
#pragma unroll
          for (int pp = 0; pp < PB; ++pp) {
            const float4 x = *reinterpret_cast<const float4*>(xb + pp * DC + k4 * 4);         // warp-wide broadcast
            const float2 d01 = fadd2(make_float2(x.x, x.y), z01), d23 = fadd2(make_float2(x.z, x.w), z23);
            q[pp] = ffma2(d01, d01, q[pp]);
            q[pp] = ffma2(d23, d23, q[pp]);
          }
        }
        (void)blk; (void)pbuf;
      };
      auto panel_store = [&](long long blk, double* pbuf, const float2 (&q)[PB]) {
        const double sc = p.scale[0];                            // applied in fp64: no overflow, no fp32 underflow
        double* dst = pbuf + pan * PB * PS + col;
        const long long pt0 = blk * PB;
#pragma unroll
        for (int pp = 0; pp < PB; ++pp)
          dst[pp * PS] = (zvalid && pt0 + pp < p.n) ? static_cast<double>(ElemOps<ET>::ex(q[pp].x + q[pp].y)) * sc : 0.0;
      };
      // ---- prologue: x(blk_lo) -> xs[0]; panel(blk_lo) -> panel[0]; x(blk_lo+1) -> xs[1]
      xs[e0] = fetch_x(blk_lo, e0); xs[e1] = fetch_x(blk_lo, e1);
      if (tid < PB) ys2[tid] = (blk_lo * PB + tid < p.n) ? p.y[blk_lo * PB + tid] : 0.0;
      __syncthreads();
      if (blk_lo < blk_hi && elem_active) {
        float2 q[PB];
#pragma unroll
        for (int i = 0; i < PB; ++i) q[i] = make_float2(0.f, 0.f);
        panel_block(blk_lo, xs, panel, 0, nk4, q);
        panel_store(blk_lo, panel, q);
      }
      xs[PB * DC + e0] = fetch_x(blk_lo + 1, e0); xs[PB * DC + e1] = fetch_x(blk_lo + 1, e1);
      __syncthreads();
      for (long long blk = blk_lo; blk < blk_hi; ++blk) {
        const int cur = static_cast<int>((blk - blk_lo) & 1), nxt = cur ^ 1;
        const double* pcur = panel + cur * 2 * PB * PS;
        double* pnxt = panel + nxt * 2 * PB * PS;
        const float* xnxt = xs + nxt * PB * DC;
        const bool has_next = blk + 1 < blk_hi;
        // global loads for block blk+2 are issued first and stored at the end of the region
        const float xa = fetch_x(blk + 2, e0), xb2 = fetch_x(blk + 2, e1);
        double ynext = 0.0;
        if (tid < PB && has_next) ynext = ((blk + 1) * PB + tid < p.n) ? p.y[(blk + 1) * PB + tid] : 0.0;
        if (owns_b && tid < kTile) {
          const double* ys = ys2 + cur * PB;
#pragma unroll
          for (int pp = 0; pp < PB; ++pp) bacc = fma(pcur[pp * PS + tid], ys[pp], bacc);
        }
        float2 q[PB];
#pragma unroll
        for (int i = 0; i < PB; ++i) q[i] = make_float2(0.f, 0.f);
        const bool build = has_next && elem_active;
        const double* PA = pcur;
        const double* PBm = diag ? pcur + joff : pcur + PB * PS;
#pragma unroll
        for (int ks = 0; ks < 4; ++ks) {
          // panel work of block blk+1 spread over the four DMMA k-steps of block blk
          if (build) panel_block(blk + 1, xnxt, pnxt, (ks * nk4) >> 2, ((ks + 1) * nk4) >> 2, q);
          const int k0 = ks * 4;
          double a[4], b[NJ];
          const double* pa = PA + (k0 + (lane & 3)) * PS + wr * 32 + (lane >> 2);
          const double* pb = PBm + (k0 + (lane & 3)) * PS + wc * (TN / 2) + (lane >> 2);
#pragma unroll
          for (int i = 0; i < 4; ++i) a[i] = pa[i * 8];
#pragma unroll
          for (int j = 0; j < NJ; ++j) b[j] = pb[j * 8];
#pragma unroll
          for (int i = 0; i < 4; ++i)
#pragma unroll
            for (int j = 0; j < NJ; ++j) dmma_m8n8k4(acc[i][j], a[i], b[j]);
        }
        if (build) panel_store(blk + 1, pnxt, q);
        float* xdst = xs + cur * PB * DC;                        // consumed in the previous region
        xdst[e0] = xa; xdst[e1] = xb2;
        if (tid < PB && has_next) ys2[nxt * PB + tid] = ynext;
        __syncthreads();
      }
      blk_hi = blk_lo;                                           // the generic loop below has nothing left to do
    }
  }

  for (long long blk = blk_lo; blk < blk_hi; ++blk) {
    const long long pt0 = blk * PB;
    // ---------------- phase 1: panels -----------------------------------------------------------
    // fp32 elements: q is accumulated as float2 (even / odd feature dims, two independent chains); per-term results go
    // straight into the panel (the thread owns its column).
    double* ys = ys2 + ((blk - blk_lo) & 1) * PB;   // stragglers of block k-1 may still read the other half
    if (tid < PB) ys[tid] = (pt0 + tid < p.n) ? p.y[pt0 + tid] : 0.0;
    double* dst = panel + pan * PB * PS + col;
    for (int term = 0; term < p.n_terms; ++term) {
      typename std::conditional<kPacked, float2, ET>::type q[PB];
#pragma unroll
      for (int i = 0; i < PB; ++i) {
        if constexpr (kPacked) q[i] = make_float2(0.f, 0.f); else q[i] = ET(0);
      }
      for (int c0 = 0; c0 < p.dpad; c0 += DC) {
        const int clen = (p.dpad - c0 < DC) ? (p.dpad - c0) : DC;
        __syncthreads();                       // previous users of xs/zs (and of the panels) are done
        if (!z_resident) load_z_chunk(term, c0, clen);
        load_x_chunk(pt0, term, c0, clen);
        __syncthreads();
        if (elem_active) {
          for (int k4 = 0; k4 < (clen >> 2); ++k4) {
            if constexpr (kPacked) {
              const float4 z = *reinterpret_cast<const float4*>(zs + (k4 * 256 + tid) * 4);      // already negated
              const float2 z01 = make_float2(z.x, z.y), z23 = make_float2(z.z, z.w);
#pragma unroll
              for (int pp = 0; pp < PB; ++pp) {
                const float4 x = *reinterpret_cast<const float4*>(xs + pp * DC + k4 * 4);          // warp-wide broadcast
                const float2 d01 = fadd2(make_float2(x.x, x.y), z01), d23 = fadd2(make_float2(x.z, x.w), z23);
                q[pp] = ffma2(d01, d01, q[pp]);
                q[pp] = ffma2(d23, d23, q[pp]);
              }
            } else {
              ET z4[4];
              ElemOps<ET>::ld4(zs + (k4 * 256 + tid) * 4, z4);
#pragma unroll
              for (int pp = 0; pp < PB; ++pp) {
                ET x4[4];
                ElemOps<ET>::ld4(xs + pp * DC + k4 * 4, x4);   // warp-wide broadcast
#pragma unroll
                for (int c = 0; c < 4; ++c) {
                  const ET df = x4[c] - z4[c];
                  q[pp] = fma(df, df, q[pp]);
                }
              }
            }
          }
        }
      }
      if (elem_active) {
        const double sc = p.scale[term];                         // the term scale in fp64 after the exponential
#pragma unroll
        for (int pp = 0; pp < PB; ++pp) {
          ET qq;
          if constexpr (kPacked) qq = q[pp].x + q[pp].y; else qq = q[pp];
          const double v = (zvalid && pt0 + pp < p.n) ? static_cast<double>(ElemOps<ET>::ex(qq)) * sc : 0.0;
          dst[pp * PS] = (term == 0) ? v : dst[pp * PS] + v;
        }
      }
    }
    __syncthreads();
    // ---------------- b_I += P_I^T y (diagonal tiles) ----------------------------------------------
    if (owns_b && tid < kTile) {
#pragma unroll
      for (int pp = 0; pp < PB; ++pp) bacc = fma(panel[pp * PS + tid], ys[pp], bacc);
    }
    // ---------------- phase 2: acc += P_I^T P_J  (fp64 tensor cores) --------------------------------
    const double* PA = panel;
    const double* PBm = diag ? panel + joff : panel + PB * PS;
#pragma unroll
    for (int k0 = 0; k0 < PB; k0 += 4) {
      double a[4], b[NJ];
      const double* pa = PA + (k0 + (lane & 3)) * PS + wr * 32 + (lane >> 2);
      const double* pb = PBm + (k0 + (lane & 3)) * PS + wc * (TN / 2) + (lane >> 2);
#pragma unroll
      for (int i = 0; i < 4; ++i) a[i] = pa[i * 8];
#pragma unroll
      for (int j = 0; j < NJ; ++j) b[j] = pb[j * 8];
#pragma unroll
      for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int j = 0; j < NJ; ++j) dmma_m8n8k4(acc[i][j], a[i], b[j]);
    }
    // the __syncthreads at the top of the next block's chunk loop protects the panels
  }

  // ---------------- flush the tile into this slice's partial buffer ---------------------------------
  double* Gp = p.Gpart + static_cast<size_t>(blockIdx.y) * p.m_pad * p.m_pad;
#pragma unroll
  for (int i = 0; i < 4; ++i)
#pragma unroll
    for (int j = 0; j < NJ; ++j) {
      const int row = ti * kTile + wr * 32 + i * 8 + (lane >> 2);
      const int cc = tj * TN + wc * (TN / 2) + j * 8 + 2 * (lane & 3);
      *reinterpret_cast<double2*>(Gp + static_cast<size_t>(row) * p.m_pad + cc) =
          make_double2(acc[i][j][0], acc[i][j][1]);
    }
  if (owns_b && tid < kTile) p.bpart[static_cast<size_t>(blockIdx.y) * p.m_pad + ti * kTile + tid] = bacc;
}

// G[i][j] (+ mirror) += sum_s Gpart[s][i][j] for i >= j ;  b[i] += sum_s bpart[s][i]
__global__ void gram_reduce_kernel(double* __restrict__ G, double* __restrict__ b,
                                   const double* __restrict__ Gpart, const double* __restrict__ bpart,
                                   int n_slices, int m, int m_pad) {
  const int j = blockIdx.x * blockDim.x + threadIdx.x;
  const int i = blockIdx.y * blockDim.y + threadIdx.y;
  if (j >= m) return;
  if (i < m && j <= i) {
    double v = 0.0;
    const size_t stride = static_cast<size_t>(m_pad) * m_pad;
    for (int s = 0; s < n_slices; ++s) v += Gpart[s * stride + static_cast<size_t>(i) * m_pad + j];
    G[static_cast<size_t>(i) * m + j] += v;
    if (i != j) G[static_cast<size_t>(j) * m + i] += v;
  }
  if (blockIdx.y == 0 && threadIdx.y == 0) {
    double v = 0.0;
    for (int s = 0; s < n_slices; ++s) v += bpart[static_cast<size_t>(s) * m_pad + j];
    b[j] += v;
  }
}

// Same for partial tiles stored at the MIRROR position (upper block triangle; the int8 kernel folds its accumulators
// transposed so that its global writes coalesce): G[i][j] (+ mirror) += sum_s Gpart[s][i][j] for j >= i.  The int8 Gram
// and its digit-plane producer split the points into different slice counts.
__global__ void gram_reduce_upper_kernel(double* __restrict__ G, double* __restrict__ b,
                                         const double* __restrict__ Gpart, const double* __restrict__ bpart,
                                         int g_slices, int b_slices, int m, int m_pad) {
  const int j = blockIdx.x * blockDim.x + threadIdx.x;
  const int i = blockIdx.y * blockDim.y + threadIdx.y;
  if (i < m && j < m && j >= i) {
    double v = 0.0;
    const size_t stride = static_cast<size_t>(m_pad) * m_pad;
    for (int s = 0; s < g_slices; ++s) v += Gpart[s * stride + static_cast<size_t>(i) * m_pad + j];
    G[static_cast<size_t>(i) * m + j] += v;
    if (i != j) G[static_cast<size_t>(j) * m + i] += v;
  }
  if (blockIdx.y == 0 && threadIdx.y == 0 && j < m) {
    double v = 0.0;
    for (int s = 0; s < b_slices; ++s) v += bpart[static_cast<size_t>(s) * m_pad + j];
    b[j] += v;
  }
}

}  // namespace

cudaError_t launch_gram_reduce_upper(double* G, double* b, const double* Gpart, const double* bpart, int g_slices,
                                     int b_slices, int m, int m_pad, cudaStream_t s) {
  dim3 block(32, 8);
  dim3 grid((m + 31) / 32, (m + 7) / 8);
  gram_reduce_upper_kernel<<<grid, block, 0, s>>>(G, b, Gpart, bpart, g_slices, b_slices, m, m_pad);
  return cudaGetLastError();
}

cudaError_t launch_gram_f64(const GramParams& p, bool strict_elements, cudaStream_t s) {
  if (strict_elements) {
    const int nt = p.n_tiles_1d * (p.n_tiles_1d + 1) / 2;
    dim3 grid(nt, p.n_slices);
    constexpr size_t smem = gram_smem_bytes<double>();
    {   // the cap is per DEVICE and shared by every context on it (one JVM holds one per task thread, on one or several
        // GPUs): set it on every launch, to the one value allow_dynamic_smem gives this kernel; it is cheap
      cudaError_t e = allow_dynamic_smem(reinterpret_cast<const void*>(kmn_gram_f64_kernel<double, 128>));
      if (e != cudaSuccess) return e;
    }
    kmn_gram_f64_kernel<double, 128><<<grid, NT, smem, s>>>(p);
  } else {
    const int nt = p.n_tiles_1d * (p.n_tiles_1d + 1);       // 128 x 64 staircase; two CTAs per SM
    dim3 grid(nt, p.n_slices);
    constexpr size_t smem = gram_smem_bytes<float>();
    {
      cudaError_t e = allow_dynamic_smem(reinterpret_cast<const void*>(kmn_gram_f64_kernel<float, 64>));
      if (e != cudaSuccess) return e;
    }
    kmn_gram_f64_kernel<float, 64><<<grid, NT, smem, s>>>(p);
  }
  return cudaGetLastError();
}

cudaError_t launch_gram_reduce(double* G, double* b, const double* Gpart, const double* bpart, int n_slices,
                               int m, int m_pad, cudaStream_t s) {
  dim3 block(32, 8);
  dim3 grid((m + 31) / 32, (m + 7) / 8);
  gram_reduce_kernel<<<grid, block, 0, s>>>(G, b, Gpart, bpart, n_slices, m, m_pad);
  return cudaGetLastError();
}

}  // namespace sgp
