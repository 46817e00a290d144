// Per-expert Laplace approximation for experts of any size (fp64): laplace_kernel's work with the matrices in global
// memory, on a persistent grid.
//
// The arithmetic is laplace_kernel's (laplace.cu): the Newton iteration with the reference's step halving and warm start
// (GPCls:79-111), the post-loop pi, W, L, a and grad log p of the LAST iteration (computed from the f before that
// iteration's update), d3logP from the final f with the reference's sign (GPCls:118), and the gradient as one pair-weight
// sweep (ex_descriptor_gradient) with the same W_ab.  What changes is where the matrices live and how the cubic steps run:
//   - a work item is one (slot, expert) pair; CTA b runs the items b, b + gridDim.x, ... and owns one slice of a global
//     workspace: K (full symmetric), M (B -> L -> L^-1 -> B^-1), a 32-row panel P and the vectors;
//   - the matrices are tiled in 32 x 32 blocks over np = n rounded up to 32 (B padded with an identity block, K, W and
//     the vectors with zeros: the padding adds exact zeros and ones only);
//   - the Cholesky of B is blocked and right-looking (diagonal block in shared memory, triangular solve of the panel
//     below on the CUDA cores, trailing update on fp64 tensor cores, mma.sync.m8n8k4.f64); L^-1, B^-1 = L^-T L^-1 and
//     diag(C^T C), C = L^-1 sqrtW K, are blocked on the tensor cores too;
//   - the level-2 steps (K b, the two triangular solves, K a, K s2, R t1) stay on the CUDA cores.
// Every sum has a fixed order and the tiling depends on the expert's own n only, so a work item's bits do not depend on
// the CTA that runs it, the grid size, n_max or the other experts and slots of the launch.
// Slots as laplace_kernel's: item (s, x) is expert first[sets[s]] + x of slot s's set (items past the set's expert count
// are skipped), its modes are indexed from the set's first row, its row is [s][x].
#include "expert_common.cuh"

namespace sgp {
namespace {

constexpr int GT = EX_THREADS;        // threads per CTA (8 warps)
constexpr int GW = EX_WARPS;
constexpr int NB = 32;                // tile edge: panel width of the factorisation, warp tile of the tensor-core steps
constexpr int DS = NB + 1;            // shared-memory stride of a diagonal block
constexpr int kLgVectors = 12;        // f, y, pi, sqrtW, grad log p, b, a, f candidate, t1, t2, s2, W

// One CTA's workspace slice, row stride ld = n_max rounded up to NB: K and M (ld x ld each), the panel P (NB x ld) and
// the vectors (kLgVectors x ld).
__host__ __device__ constexpr int lg_ld(int n_max) { return (n_max + NB - 1) / NB * NB; }
__host__ __device__ constexpr size_t lg_cta_doubles(int ld) {
  return static_cast<size_t>(ld) * (2 * static_cast<size_t>(ld) + NB + kLgVectors);
}

struct LapGlobalParams {
  const double* X; const double* y; double* f; const long long* off;
  long long E;               // experts per slot: the largest expert count over the listed sets
  int n_slots;
  int ldw;                   // workspace row stride: n_max rounded up to NB
  HyperView hv;              // slot 0's view (as laplace_kernel's)
  const int* cls;            // [n_slots] class of each slot; < 0: labels as uploaded
  const int* mode;           // [n_slots] mode slot of each slot
  const KernelFlat* kf;      // [n_slots]
  long long slot_stride;
  long long n;               // stride of the per-slot modes
  const int* sets;           // [n_slots] expert set of each slot
  const long long* first;    // [n_sets + 1] first expert of each set
  double tol;
  double* ws;                // [gridDim.x][lg_cta_doubles(ldw)]
  double* out;               // [n_slots][E][1 + n_hypers]
  int* flags;                // [n_slots]  bit 0: Cholesky pivot not positive
};

__device__ __forceinline__ double lg_sigmoid(double x) { return 1.0 / (1.0 + exp(-x)); }

__device__ __forceinline__ void dmma_m8n8k4(double (&c)[2], double a, double b) {
  asm volatile("mma.sync.aligned.m8n8k4.row.col.f64.f64.f64.f64 {%0,%1}, {%2}, {%3}, {%0,%1};\n"
               : "+d"(c[0]), "+d"(c[1])
               : "d"(a), "d"(b));
}

__device__ __forceinline__ double* row_ptr(double* A, int r, int ld) { return A + static_cast<size_t>(r) * ld; }
__device__ __forceinline__ const double* row_ptr(const double* A, int r, int ld) { return A + static_cast<size_t>(r) * ld; }

// 32 x 32 warp tile on the tensor cores: the m8n8k4 accumulator layout gives lane l the rows i*8 + l/4 and the columns
// j*8 + 2*(l%4) + {0, 1} of its tile.
struct WarpTile {
  double c[4][4][2];
  __device__ __forceinline__ void zero() {
#pragma unroll
    for (int i = 0; i < 4; ++i)
#pragma unroll
      for (int j = 0; j < 4; ++j) c[i][j][0] = c[i][j][1] = 0.0;
  }
  // the tile at (r0, c0) of the row-major matrix A
  __device__ __forceinline__ void store(double* A, int ld, int r0, int c0) const {
    const int lane = threadIdx.x & 31;
#pragma unroll
    for (int i = 0; i < 4; ++i)
#pragma unroll
      for (int j = 0; j < 4; ++j)
        *reinterpret_cast<double2*>(A + static_cast<size_t>(r0 + i * 8 + (lane >> 2)) * ld + c0 + j * 8 + 2 * (lane & 3)) =
            make_double2(c[i][j][0], c[i][j][1]);
  }
  // c += A B over k = 0..3 of one step: a(i) is A[i*8 + l/4][l%4], b(j) is B[l%4][j*8 + l/4]
  template <class FA, class FB>
  __device__ __forceinline__ void step(FA a_of, FB b_of) {
    double a[4], b[4];
#pragma unroll
    for (int i = 0; i < 4; ++i) a[i] = a_of(i);
#pragma unroll
    for (int j = 0; j < 4; ++j) b[j] = b_of(j);
#pragma unroll
    for (int i = 0; i < 4; ++i)
#pragma unroll
      for (int j = 0; j < 4; ++j) dmma_m8n8k4(c[i][j], a[i], b[j]);
  }
};

// Lower-triangular tile pairs (I, J), j0 <= J <= I < nb, dealt to the warps in row-major order.
template <class F>
__device__ __forceinline__ void for_lower_tiles(int j0, int nb, F fn) {
  const int warp = threadIdx.x >> 5;
  int t = 0;
  for (int I = j0; I < nb; ++I)
    for (int J = j0; J <= I; ++J, ++t)
      if ((t % GW) == warp) fn(I, J);
}

// Loads the lower triangle of the diagonal block at (k0, k0) into D (upper triangle zero).
__device__ __forceinline__ void load_diag_block(const double* M, int ld, int k0, double* D) {
  for (int idx = threadIdx.x; idx < NB * NB; idx += GT) {
    const int r = idx / NB, c = idx % NB;
    D[r * DS + c] = (c <= r) ? row_ptr(M, k0 + r, ld)[k0 + c] : 0.0;
  }
}

// Xs = D^-1 for the lower-triangular 32 x 32 block D (upper triangle of Xs zero); one warp, lane c forms column c by
// forward substitution.
__device__ __forceinline__ void warp_invert_lower(const double* D, double* Xs) {
  const int c = threadIdx.x & 31;
  for (int r = 0; r < NB; ++r) {
    double v = 0.0;
    if (r == c) {
      v = 1.0 / D[r * DS + r];
    } else if (r > c) {
      double s = 0.0;
      for (int k = c; k < r; ++k) s = fma(D[r * DS + k], Xs[k * DS + c], s);
      v = -s / D[r * DS + r];
    }
    Xs[r * DS + c] = v;
  }
  __syncwarp();
}

// In-place blocked lower Cholesky of the np x np matrix M (right-looking).  Pivots follow ex_cholesky: a pivot that is
// not positive sets `bad` (thread 0 always sees it) and is replaced by 1.  Returns sum(log diag L) over the first n rows.
__device__ double lg_cholesky(double* M, int n, int np, int ld, double* D, double* Xs, double* red, bool& bad) {
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int nb = np / NB;
  for (int kb = 0; kb < nb; ++kb) {
    const int k0 = kb * NB;
    load_diag_block(M, ld, k0, D);
    __syncthreads();
    if (warp == 0) {                                         // the diagonal block, one lane per row
      for (int j = 0; j < NB; ++j) {
        const double djj = D[j * DS + j];
        if (!(djj > 0.0)) bad = true;
        const double dd = djj > 0.0 ? djj : 1.0;
        const double inv = rsqrt(dd);
        __syncwarp();
        if (lane == j) D[j * DS + j] = dd * inv;
        if (lane > j) D[lane * DS + j] *= inv;
        __syncwarp();
        if (lane > j) {
          const double lij = D[lane * DS + j];
          for (int k = j + 1; k <= lane; ++k) D[lane * DS + k] = fma(-lij, D[k * DS + j], D[lane * DS + k]);
        }
        __syncwarp();
      }
      warp_invert_lower(D, Xs);                              // L11^-1 for the panel below
    }
    __syncthreads();
    for (int idx = tid; idx < NB * NB; idx += GT) {         // L11 back (upper triangle of the block: zero)
      const int r = idx / NB, c = idx % NB;
      row_ptr(M, k0 + r, ld)[k0 + c] = D[r * DS + c];
    }
    // panel below: L21 = A21 L11^-T, one 32 x 32 tile per warp on the tensor cores
    for (int I = kb + 1 + warp; I < nb; I += GW) {
      WarpTile t;
      t.zero();
#pragma unroll
      for (int k4 = 0; k4 < NB; k4 += 4) {
        const int kc = k4 + (lane & 3);
        t.step([&](int i) { return row_ptr(M, I * NB + i * 8 + (lane >> 2), ld)[k0 + kc]; },
               [&](int j) { return Xs[(j * 8 + (lane >> 2)) * DS + kc]; });
      }
      t.store(M, ld, I * NB, k0);
    }
    __syncthreads();
    // trailing update A22 -= L21 L21^T on the lower tiles (diagonal tiles: their lower triangle)
    for_lower_tiles(kb + 1, nb, [&](int I, int J) {
      WarpTile t;
      const int rr = lane >> 2, cc = 2 * (lane & 3);
#pragma unroll
      for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j) {
          const double2 v = *reinterpret_cast<const double2*>(row_ptr(M, I * NB + i * 8 + rr, ld) + J * NB + j * 8 + cc);
          t.c[i][j][0] = v.x; t.c[i][j][1] = v.y;
        }
#pragma unroll
      for (int k4 = 0; k4 < NB; k4 += 4) {
        const int kc = k0 + k4 + (lane & 3);
        t.step([&](int i) { return -row_ptr(M, I * NB + i * 8 + rr, ld)[kc]; },
               [&](int j) { return row_ptr(M, J * NB + j * 8 + rr, ld)[kc]; });
      }
#pragma unroll
      for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j) {
          const int r = i * 8 + rr, c = j * 8 + cc;
          double* dst = row_ptr(M, I * NB + r, ld) + J * NB + c;
          if (I != J || c <= r) dst[0] = t.c[i][j][0];
          if (I != J || c + 1 <= r) dst[1] = t.c[i][j][1];
        }
    });
    __syncthreads();
  }
  double part = 0.0;
  for (int j = tid; j < n; j += GT) part += log(row_ptr(M, j, ld)[j]);
  return ex_block_sum(part, red);
}

// x <- L^-1 x over np rows (blocked: the diagonal block by warp 0, then the rows below it)
__device__ void lg_fwd_solve(const double* L, int np, int ld, double* x, double* D) {
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  for (int k0 = 0; k0 < np; k0 += NB) {
    load_diag_block(L, ld, k0, D);
    __syncthreads();
    if (warp == 0) {
      double xl = x[k0 + lane];
      for (int j = 0; j < NB; ++j) {
        if (lane == j) xl /= D[j * DS + j];
        const double xj = __shfl_sync(0xffffffffu, xl, j);
        if (lane > j) xl -= D[lane * DS + j] * xj;
      }
      x[k0 + lane] = xl;
    }
    __syncthreads();
    for (int i = k0 + NB + tid; i < np; i += GT) {
      const double* lr = row_ptr(L, i, ld) + k0;
      double s = x[i];
      for (int k = 0; k < NB; ++k) s -= lr[k] * x[k0 + k];
      x[i] = s;
    }
    __syncthreads();
  }
}

// x <- L^-T x over np rows
__device__ void lg_bwd_solve(const double* L, int np, int ld, double* x, double* D) {
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  for (int k0 = np - NB; k0 >= 0; k0 -= NB) {
    load_diag_block(L, ld, k0, D);
    __syncthreads();
    if (warp == 0) {
      double xl = x[k0 + lane];
      for (int j = NB - 1; j >= 0; --j) {
        if (lane == j) xl /= D[j * DS + j];
        const double xj = __shfl_sync(0xffffffffu, xl, j);
        if (lane < j) xl -= D[j * DS + lane] * xj;
      }
      x[k0 + lane] = xl;
    }
    __syncthreads();
    for (int i = tid; i < k0; i += GT) {
      double s = x[i];
      for (int k = 0; k < NB; ++k) s -= row_ptr(L, k0 + k, ld)[i] * x[k0 + k];
      x[i] = s;
    }
    __syncthreads();
  }
}

// out[i] = sum_{k < n} A[k][i] v[k] for i < np (A symmetric: a coalesced column read of row i)
__device__ __forceinline__ void lg_symv(const double* A, int n, int np, int ld, const double* v, double* out) {
  for (int i = threadIdx.x; i < np; i += GT) {
    double s = 0.0;
    for (int k = 0; k < n; ++k) s += A[static_cast<size_t>(k) * ld + i] * v[k];
    out[i] = s;
  }
}

// L -> L^-1 in place (np x np, lower; the upper triangle of the diagonal blocks becomes zero).  Row block I, top-down:
// X_II = L_II^-1 (warp 0, in shared memory), T_IJ = sum_{K=J}^{I-1} L_IK X_KJ into the panel P, X_IJ = -X_II T_IJ.
__device__ void lg_invert_lower(double* M, int np, int ld, double* P, double* D, double* Xs) {
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int nb = np / NB, rr = lane >> 2;
  for (int I = 0; I < nb; ++I) {
    load_diag_block(M, ld, I * NB, D);
    __syncthreads();
    if (warp == 0) warp_invert_lower(D, Xs);                 // X_II
    for (int J = warp; J < I; J += GW) {                     // T_IJ
      WarpTile t;
      t.zero();
      for (int K = J; K < I; ++K)
#pragma unroll
        for (int k4 = 0; k4 < NB; k4 += 4) {
          const int kc = K * NB + k4 + (lane & 3);
          t.step([&](int i) { return row_ptr(M, I * NB + i * 8 + rr, ld)[kc]; },
                 [&](int j) { return row_ptr(M, kc, ld)[J * NB + j * 8 + rr]; });
        }
      t.store(P, ld, 0, J * NB);
    }
    __syncthreads();
    for (int J = warp; J < I; J += GW) {                     // X_IJ = -X_II T_IJ
      WarpTile t;
      t.zero();
#pragma unroll
      for (int k4 = 0; k4 < NB; k4 += 4) {
        const int kc = k4 + (lane & 3);
        t.step([&](int i) { return -Xs[(i * 8 + rr) * DS + kc]; },
               [&](int j) { return row_ptr(P, kc, ld)[J * NB + j * 8 + rr]; });
      }
      t.store(M, ld, I * NB, J * NB);
    }
    for (int idx = tid; idx < NB * NB; idx += GT) {
      const int r = idx / NB, c = idx % NB;
      row_ptr(M, I * NB + r, ld)[I * NB + c] = Xs[r * DS + c];
    }
    __syncthreads();
  }
}

// cc[j] = sum_r C[r][j]^2 for j < np, C = X S with X = L^-1 (lower, in M) and S = sqrtW K.  Warp w owns the column
// blocks J = w, w + 8, ...; the squares are summed over the row blocks I in order, then over the lanes of a column.
__device__ void lg_diag_ctc(const double* M, const double* K, const double* sw, int np, int ld, double* cc_out) {
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int nb = np / NB, rr = lane >> 2;
  for (int J = warp; J < nb; J += GW) {
    double cs[4][2];
#pragma unroll
    for (int j = 0; j < 4; ++j) cs[j][0] = cs[j][1] = 0.0;
    for (int I = 0; I < nb; ++I) {
      WarpTile t;
      t.zero();
      for (int Kb = 0; Kb <= I; ++Kb)
#pragma unroll
        for (int k4 = 0; k4 < NB; k4 += 4) {
          const int kc = Kb * NB + k4 + (lane & 3);
          const double swk = sw[kc];
          t.step([&](int i) { return row_ptr(M, I * NB + i * 8 + rr, ld)[kc]; },
                 [&](int j) { return swk * row_ptr(K, kc, ld)[J * NB + j * 8 + rr]; });
        }
#pragma unroll
      for (int j = 0; j < 4; ++j)
#pragma unroll
        for (int h = 0; h < 2; ++h)
#pragma unroll
          for (int i = 0; i < 4; ++i) cs[j][h] = fma(t.c[i][j][h], t.c[i][j][h], cs[j][h]);
    }
#pragma unroll
    for (int j = 0; j < 4; ++j)
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        double v = cs[j][h];
        for (int o = 4; o < 32; o <<= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
        if (rr == 0) cc_out[J * NB + j * 8 + 2 * lane + h] = v;
      }
  }
}

// X = L^-1 -> B^-1 = X^T X in place, both triangles.  Row block I, top-down (it reads rows >= I only):
// R_IJ = sum_{K>=I} X_KI^T X_KJ for J <= I into the panel P, then row block I and its mirror are written.
__device__ void lg_ltl(double* M, int np, int ld, double* P) {
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int nb = np / NB, rr = lane >> 2;
  for (int I = 0; I < nb; ++I) {
    for (int J = warp; J <= I; J += GW) {
      WarpTile t;
      t.zero();
      for (int Kb = I; Kb < nb; ++Kb)
#pragma unroll
        for (int k4 = 0; k4 < NB; k4 += 4) {
          const double* xr = row_ptr(M, Kb * NB + k4 + (lane & 3), ld);
          t.step([&](int i) { return xr[I * NB + i * 8 + rr]; }, [&](int j) { return xr[J * NB + j * 8 + rr]; });
        }
      t.store(P, ld, 0, J * NB);
    }
    __syncthreads();
    const int w = (I + 1) * NB;
    for (int idx = tid; idx < NB * w; idx += GT) {
      const int r = idx / w, c = idx % w, a = I * NB + r;
      if (c > a) continue;                                   // the diagonal tile: its lower triangle, mirrored
      const double v = row_ptr(P, r, ld)[c];
      row_ptr(M, a, ld)[c] = v;
      row_ptr(M, c, ld)[a] = v;
    }
    __syncthreads();
  }
}

__global__ void __launch_bounds__(GT, 1) laplace_global_kernel(const LapGlobalParams p) {
  __shared__ double D[NB * DS], Xs[NB * DS], red[8], sums[EX_SUMS];
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int ld = p.ldw;
  double* K = p.ws + static_cast<size_t>(blockIdx.x) * lg_cta_doubles(ld);
  double* M = K + static_cast<size_t>(ld) * ld;
  double* P = M + static_cast<size_t>(ld) * ld;
  double* v = P + static_cast<size_t>(NB) * ld;
  double *f = v, *yv = v + ld, *pi = v + 2 * ld, *sw = v + 3 * ld, *glp = v + 4 * ld, *bv = v + 5 * ld,
         *av = v + 6 * ld, *nf = v + 7 * ld, *t1 = v + 8 * ld, *t2 = v + 9 * ld, *s2 = v + 10 * ld, *wv = v + 11 * ld;
  const long long items = p.E * p.n_slots;
  for (long long w = blockIdx.x; w < items; w += gridDim.x) {
    const int slot = static_cast<int>(w / p.E);
    long long e = w % p.E;
    const long long first = p.first[p.sets[slot]];
    if (e >= p.first[p.sets[slot] + 1] - first) continue;   // the whole CTA skips the item
    e += first;
    const long long fr = p.off[first];                   // row of the modes that belong to the set's first row
    const long long r0 = p.off[e];
    const int n = static_cast<int>(p.off[e + 1] - r0);
    const int np = (n + NB - 1) / NB * NB;
    HyperView hv = p.hv;
    const double cls = p.cls[slot];                      // < 0: labels as uploaded
    double* fg = p.f + static_cast<size_t>(p.mode[slot]) * p.n;
    hv.kf = p.kf[slot];
    hv.beta += slot * p.slot_stride; hv.h_coef += slot * p.slot_stride; hv.h_value += slot * p.slot_stride;
    const double* Xe = p.X + static_cast<size_t>(r0) * hv.d;
    __syncthreads();                                     // the previous item is done with the workspace
    for (int i = tid; i < np; i += GT) {
      f[i] = (i < n) ? fg[r0 - fr + i] : 0.0;
      yv[i] = (i >= n) ? 0.0 : (cls < 0.0) ? p.y[r0 + i] : (p.y[r0 + i] == cls ? 1.0 : 0.0);
    }
    ex_build_kernel<true>(hv, Xe, hv.d, n, K, ld);       // K, both triangles (laplace_kernel's elements)
    for (int a = warp; a < np; a += GW)                  // zero padding rows and columns
      for (int b = lane; b < np; b += 32)
        if (a >= n || b >= n) row_ptr(K, a, ld)[b] = 0.0;
    __syncthreads();

    // ---- Newton iteration for the mode (GPCls:79-111) ----------------------------------------------------------------
    double old_obj = -INFINITY, new_obj = -1.7976931348623157e308;   // Double.NegativeInfinity, Double.MinValue
    double step = 1.0, sumlogL = 0.0;
    bool bad = false;
    while (fabs(old_obj - new_obj) > p.tol && step > p.tol) {
      for (int i = tid; i < np; i += GT) {
        const double s = (i < n) ? lg_sigmoid(f[i]) : 0.0;
        const double wi = (i < n) ? s * (1.0 - s) : 0.0;
        pi[i] = s;
        wv[i] = wi;
        sw[i] = sqrt(wi);
        glp[i] = yv[i] - s;
      }
      __syncthreads();
      for (int a = warp; a < np; a += GW) {              // B = I + sqrtW K sqrtW   (GPCls:95-97), lower
        const double* kr = row_ptr(K, a, ld);
        double* mr = row_ptr(M, a, ld);
        for (int b = lane; b <= a; b += 32) mr[b] = sw[a] * sw[b] * kr[b] + (a == b ? 1.0 : 0.0);
      }
      __syncthreads();
      sumlogL = lg_cholesky(M, n, np, ld, D, Xs, red, bad);          // GPCls:98
      for (int i = tid; i < np; i += GT) bv[i] = wv[i] * f[i] + glp[i];  // b = W f + grad log p   (:100)
      __syncthreads();
      lg_symv(K, n, np, ld, bv, t1);                     // rhs = sqrtW (K b)
      for (int i = tid; i < np; i += GT) t1[i] *= sw[i];
      __syncthreads();
      lg_fwd_solve(M, np, ld, t1, D);                    // L \ rhs
      lg_bwd_solve(M, np, ld, t1, D);                    // L^T \ .
      for (int i = tid; i < np; i += GT) av[i] = bv[i] - sw[i] * t1[i];   // a   (:101)
      __syncthreads();
      double part = 0.0;
      for (int i = tid; i < n; i += GT) {                // f_candidate = (1-step) f + step K a   (:102)
        double s = 0.0;
        for (int k = 0; k < n; ++k) s += K[static_cast<size_t>(k) * ld + i] * av[k];
        const double c = (1.0 - step) * f[i] + step * s;
        nf[i] = c;
        part += -0.5 * av[i] * c + log(lg_sigmoid((yv[i] * 2.0 - 1.0) * c));   // (:103)
      }
      const double cand = ex_block_sum(part, red);
      if (cand > old_obj) {                              // (:104-107)
        for (int i = tid; i < n; i += GT) f[i] = nf[i];
        old_obj = new_obj;
        new_obj = cand;
      } else {
        step *= 0.5;
      }
      __syncthreads();
    }
    if (bad && tid == 0) atomicOr(p.flags + slot, 1);
    for (int i = tid; i < n; i += GT) fg[r0 - fr + i] = f[i];   // the mode persists (warm start of the next evaluation)

    // ---- log Z and gradient (GPCls:114-128) ------------------------------------------------------------------------
    double* out = p.out + (static_cast<size_t>(slot) * p.E + w % p.E) * (1 + hv.n_hypers);   // row [slot][x]
    if (tid == 0) out[0] = -(new_obj - sumlogL);
    lg_invert_lower(M, np, ld, P, D, Xs);                // L^-1 in place
    lg_diag_ctc(M, K, sw, np, ld, t2);                   // diag(C^T C), C = L^-1 (sqrtW K)   (GPCls:117,119)
    __syncthreads();
    for (int i = tid; i < np; i += GT) {
      double s = 0.0;
      if (i < n) {
        const double d3 = -(2.0 * pi[i] - 1.0) * pi[i] * pi[i] * exp(-f[i]);   // (:118) sign as in the reference
        s = -0.5 * (row_ptr(K, i, ld)[i] - t2[i]) * d3;                      // (:119)
      }
      s2[i] = s;
    }
    __syncthreads();
    lg_ltl(M, np, ld, P);                                // B^-1 = L^-T L^-1;  R = sqrtW B^-1 sqrtW   (GPCls:116)
    // GPCls:121-126 as in laplace_kernel: W = 1/2 (a a' - R) + 1/2 (u glp' + glp u'),  u = s2 - R K s2
    lg_symv(K, n, np, ld, s2, t1);                       // t1 = K s2
    __syncthreads();
    for (int a = tid; a < np; a += GT) {                 // t2 = u = s2 - R t1
      double s = 0.0;
      for (int b = 0; b < n; ++b) s += sw[a] * sw[b] * M[static_cast<size_t>(b) * ld + a] * t1[b];
      t2[a] = s2[a] - s;
    }
    __syncthreads();
    ex_descriptor_gradient(
        hv, Xe, hv.d, n,
        [&](int a, int b) {
          return 0.5 * (av[a] * av[b] - sw[a] * sw[b] * row_ptr(M, a, ld)[b]) + 0.5 * (t2[a] * glp[b] + t2[b] * glp[a]);
        },
        -1.0, out + 1, sums, red);                       // -gradLogZ
  }
}

}  // namespace

size_t laplace_global_cta_bytes(int n_max) {
  return sizeof(double) * lg_cta_doubles(lg_ld(n_max));
}

int laplace_global_ctas_per_sm() {
  int per_sm = 0;
  if (cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, laplace_global_kernel, GT, 0) != cudaSuccess) return 1;
  return per_sm > 0 ? per_sm : 1;
}

long long laplace_global_grid(long long items, long long resident, size_t cta_bytes, size_t budget) {
  long long g = items < resident ? items : resident;
  const long long by_ws = static_cast<long long>(budget / cta_bytes);
  if (by_ws < g) g = by_ws;
  return g > 0 ? g : 1;
}

cudaError_t launch_laplace_global(const ExpertSet& ex, const HyperView& hv, double tol, double* ws, long long grid,
                                  const ObjectiveSlots& sl, double* rows, double* total, int* flags, cudaStream_t s) {
  LapGlobalParams p{};
  p.X = ex.X; p.y = ex.y; p.f = sl.f; p.off = ex.off; p.E = sl.E_max; p.n_slots = sl.n_slots; p.ldw = lg_ld(ex.n_max);
  p.hv = hv; p.cls = sl.cls; p.mode = sl.mode; p.kf = sl.kf; p.slot_stride = sl.slot_stride; p.n = sl.f_stride;
  p.sets = sl.sets; p.first = sl.first; p.tol = tol; p.ws = ws; p.out = rows; p.flags = flags;
  laplace_global_kernel<<<static_cast<unsigned>(grid), GT, 0, s>>>(p);
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) return e;
  return launch_rows_reduce(total, rows, p.E, 1 + hv.n_hypers, s, p.n_slots, p.sets, p.first);
}

}  // namespace sgp
