// K_nm sweep: materialise the cross kernel  K[i][j] = C * exp(-sum_k beta_k^2 (x_ik - z_jk)^2)  of a block of points
// against the active set, in fp32, row-major n x m (the reference's `crossKernel(test)` orientation: test.length x
// train.length, kernel/Kernel.scala:69-74 -- here test = the points, train = the active set, i.e. the transpose of the
// per-expert K_mn that commons/ActiveSetProvider.scala:90-92 materialises and caches and that
// commons/GaussianProcessCommons.scala:121-125 evaluates row by row).
//
// This is the HBM-bound member of the family (BASELINE configs[4]: "K_nm sweep vs roofline"): algorithmic bytes per point
// are d*4 read + m*4 written, the tensor-core work (the same fp16-split distance contraction as the fused Gram kernel,
// gram_i8_wgmma.cu) is a few % of the store time.  One CTA (two warpgroups, 64 active rows each) owns an active tile (128
// columns of K) and a slice of the points; per 64-point unit: bulk copy of the pre-swizzled point image into a 4-deep
// ring, ONE fp16 wgmma contraction (m64n64, fp32 accumulators in registers), epilogue ex2 -> * C -> st.global.  Two CTAs
// per SM keep the stores of one CTA in flight while the other contracts.
#include <cuda_fp16.h>

#include "hopper.cuh"
#include "sgp_internal.h"

namespace sgp {
namespace {

using namespace hop;

constexpr int UP = 64;
constexpr int XSTAGES = 4;
constexpr int NTHREADS = 256;
constexpr int ZPANEL_BYTES = 16384, XIMG_BYTES = 8192;

struct SweepParams {
  const uint8_t* Xt;    // [n_units][nchunks][8192]   fp16 point images (launch_i8_prep_points)
  const uint8_t* Zt;    // [n_tiles_1d][nchunks][16384]
  long long n, n_units;
  int nchunks;
  int m, nt, n_slices;
  float scale;          // C
  float* K;             // [n][m] row-major
};

template <int KS>   // 16-column k-steps of the distance contraction: 4 (d <= 16) or 7 (d <= 32)
__global__ void __launch_bounds__(NTHREADS, 2) kmn_sweep_kernel(const SweepParams p) {
  extern __shared__ uint8_t smem_raw[];
  const uint32_t raw = smem_u32(smem_raw);
  const uint32_t base = (raw + 1023u) & ~1023u;
  const uint32_t xbytes = static_cast<uint32_t>(p.nchunks * XIMG_BYTES);
  const uint32_t s_zt = base;                                             // [nchunks][16384]
  const uint32_t s_xs = s_zt + p.nchunks * ZPANEL_BYTES;                  // [XSTAGES][nchunks][8192]
  const uint32_t s_bar = s_xs + XSTAGES * xbytes;
  const uint32_t b_zfull = s_bar, b_xfull = s_bar + 8;
  const int tid = threadIdx.x, wg = tid >> 7, wq = (tid >> 5) & 3, lane = tid & 31;
  const int ti = blockIdx.x;

  const long long ups = (p.n_units + p.n_slices - 1) / p.n_slices;
  const long long u_lo = ups * blockIdx.y;
  long long u_hi = u_lo + ups;
  if (u_hi > p.n_units) u_hi = p.n_units;
  const long long nu = u_hi > u_lo ? u_hi - u_lo : 0;
  if (nu == 0) return;

  auto issue_unit = [&](long long i, int s) {
    mbar_expect_tx(b_xfull + 8 * s, xbytes);
    bulk_g2s(s_xs + s * xbytes, p.Xt + static_cast<size_t>(u_lo + i) * xbytes, xbytes, b_xfull + 8 * s);
  };
  if (tid == 0) {
    mbar_init(b_zfull, 1);
    for (int s = 0; s < XSTAGES; ++s) mbar_init(b_xfull + 8 * s, 1);
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();
  if (tid == 0) {
    mbar_expect_tx(b_zfull, static_cast<uint32_t>(p.nchunks * ZPANEL_BYTES));
    bulk_g2s(s_zt, p.Zt + static_cast<size_t>(ti) * p.nchunks * ZPANEL_BYTES, static_cast<uint32_t>(p.nchunks * ZPANEL_BYTES),
             b_zfull);
    for (long long i = 0; i < XSTAGES && i < nu; ++i) issue_unit(i, static_cast<int>(i));
  }
  // accumulator fragment: element 4j+e at row r0 (+8 if e >= 2), point 8j + c0 + (e & 1)
  const int r0 = 16 * wq + (lane >> 2), c0 = 2 * (lane & 3);
  const int col0 = ti * kTile + 64 * wg + r0, col1 = col0 + 8;             // columns of K
  mbar_wait(b_zfull, 0);
  for (long long i = 0; i < nu; ++i) {
    const int s = static_cast<int>(i % XSTAGES);
    if (tid == 0 && i >= 1 && i + XSTAGES - 1 < nu) issue_unit(i + XSTAGES - 1, static_cast<int>((i - 1) % XSTAGES));
    mbar_wait(b_xfull + 8 * s, static_cast<uint32_t>((i / XSTAGES) & 1));
    float T[32];
    wg_fence();
#pragma unroll
    for (int k = 0; k < KS; ++k) {
      const uint32_t za = s_zt + (k >> 2) * ZPANEL_BYTES + wg * 8192 + (k & 3) * 32;
      const uint32_t xb = s_xs + s * xbytes + (k >> 2) * XIMG_BYTES + (k & 3) * 32;
      wgmma_f16_n64(T, desc_sw128(za), desc_sw128(xb), k > 0);
    }
    wg_commit();
    wg_wait<0>();
    __syncthreads();     // point stage s released (both warpgroups' contractions have completed)
    const long long pt0 = (u_lo + i) * UP + c0;
#pragma unroll
    for (int e = 0; e < 32; ++e) {
      const long long pt = pt0 + 8 * (e >> 2) + (e & 1);
      const int col = (e & 2) ? col1 : col0;
      // the 8 lanes of a quad column write 8 consecutive floats of row pt
      if (col < p.m && pt < p.n) p.K[static_cast<size_t>(pt) * p.m + col] = p.scale * ex2f(T[e]);
    }
  }
}

}  // namespace

cudaError_t launch_kmn_sweep(const uint8_t* Xt, const uint8_t* Zt, long long n, int d, int m, int m_pad, int num_sms, double C,
                             float* K, cudaStream_t s) {
  SweepParams p{};
  const int dp = (d + 15) / 16 * 16;
  p.Xt = Xt; p.Zt = Zt; p.n = n; p.n_units = (n + UP - 1) / UP;
  p.nchunks = i8_nchunks(d);
  p.m = m; p.nt = m_pad / kTile;
  p.scale = static_cast<float>(C);
  p.K = K;
  // tiles x point slices: enough CTAs to fill the SMs a few times over (no co-residency requirement here)
  int slices = (4 * num_sms + p.nt - 1) / p.nt;
  if (slices > p.n_units) slices = static_cast<int>(p.n_units > 0 ? p.n_units : 1);
  if (slices < 1) slices = 1;
  p.n_slices = slices;
  const size_t smem = 1024 + p.nchunks * ZPANEL_BYTES + XSTAGES * p.nchunks * XIMG_BYTES + 8 * (XSTAGES + 1);
  const void* fn = (3 * dp + 16) / 16 == 4 ? reinterpret_cast<const void*>(kmn_sweep_kernel<4>)
                                           : reinterpret_cast<const void*>(kmn_sweep_kernel<7>);
  cudaError_t e = allow_dynamic_smem(fn);
  if (e != cudaSuccess) return e;
  dim3 grid(p.nt, slices);
  void* args[] = {&p};
  e = cudaLaunchKernel(fn, grid, dim3(NTHREADS), args, smem, s);
  if (e != cudaSuccess) return e;
  return cudaGetLastError();
}

}  // namespace sgp
