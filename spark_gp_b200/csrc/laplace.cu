// Batched per-expert Laplace approximation for binary GP classification (fp64), one CTA per expert.
//
// Replaces, for all experts of a rank at once, classification/GaussianProcessClassifier.scala:74-129
// `likelihoodAndGradient`: the Newton iteration for the mode of q(f | X, y) (Rasmussen & Williams Alg. 3.1) WITH the
// reference's step halving and its warm start (f persists across objective evaluations, GPCls:53-55,105), then the
// approximate log marginal likelihood and its gradient (R&W Alg. 5.1) -- including the reference's quirks: the
// post-loop quantities (pi, W, L, a, grad log p) are the ones of the LAST Newton iteration, i.e. computed from the f
// before that iteration's update, while d3logP (GPCls:118, sign as in the reference) uses exp(-f) of the final f.
// Summed over experts like commons/GaussianProcessCommons.scala:73-78.
//
// Slots (ObjectiveSlots): a second grid dimension runs several binary problems in one launch (sgp_laplace_nll is one
// slot on the whole upload, its labels as uploaded).  Block (x, s) evaluates expert first[sets[s]] + x for the s-th
// listed slot, of class c and mode slot m: labels (y == c) (c < 0: as uploaded), modes f + m * f_stride indexed from the
// set's first row, its own flattened kernel and hyper-parameter block, output row [s][x]; a block past the set's expert
// count returns before its first barrier.  The one-vs-rest entries pass m = c.  The arithmetic does not depend on the
// slot, and n_max and x_in_smem only move addresses: every loop runs over the expert's own n.  So a slot's rows equal,
// bit for bit, those of a one-slot launch on an upload of the labels (y == c) of that set alone with the same modes.
#include "expert_common.cuh"

namespace sgp {
namespace {

constexpr int LT = EX_THREADS;     // threads per CTA

struct LapParams {
  const double* X; const double* y; double* f; const long long* off;
  int n_max, x_in_smem;
  HyperView hv;              // slot 0's view; slot s reads kf[s] and the descriptor values s * slot_stride doubles on
  const int* cls;            // [n_slots] class of each slot (one-vs-rest); < 0: labels as uploaded
  const int* mode;           // [n_slots] mode slot of each slot: its modes are f + mode[s] * n
  const KernelFlat* kf;      // [n_slots] flattened kernel of each slot
  long long slot_stride;     // doubles between two slots' [beta | coef | value] blocks
  long long n;               // the stride of the per-slot modes f
  const int* sets;           // [n_slots] expert set of each slot
  const long long* first;    // [n_sets + 1] first expert of each set
  double tol;
  double* out;               // [n_slots][E][1 + n_hypers]  (-logZ, -gradLogZ)
  int* flags;                // [n_slots]  bit 0: Cholesky pivot not positive
};

__device__ __forceinline__ double sigmoid(double x) { return 1.0 / (1.0 + exp(-x)); }

// x <- L^-1 x  (forward substitution, column oriented)
__device__ void fwd_solve(const double* L, int n, int ld, double* x) {
  for (int j = 0; j < n; ++j) {
    __syncthreads();
    if (threadIdx.x == 0) x[j] /= L[j * ld + j];
    __syncthreads();
    const double xj = x[j];
    for (int i = j + 1 + threadIdx.x; i < n; i += LT) x[i] -= L[i * ld + j] * xj;
  }
  __syncthreads();
}
// x <- L^-T x  (backward substitution)
__device__ void bwd_solve(const double* L, int n, int ld, double* x) {
  for (int j = n - 1; j >= 0; --j) {
    __syncthreads();
    if (threadIdx.x == 0) x[j] /= L[j * ld + j];
    __syncthreads();
    const double xj = x[j];
    for (int i = threadIdx.x; i < j; i += LT) x[i] -= L[j * ld + i] * xj;
  }
  __syncthreads();
}

__global__ void __launch_bounds__(LT, 1) laplace_kernel(const LapParams p) {
  extern __shared__ double sm[];
  long long e = blockIdx.x;
  const int slot = blockIdx.y;
  const long long first = p.first[p.sets[slot]];
  if (e >= p.first[p.sets[slot] + 1] - first) return;
  e += first;
  const long long fr = p.off[first];                    // row of the modes that belong to the set's first row
  const long long r0 = p.off[e];
  const int n = static_cast<int>(p.off[e + 1] - r0);
  const int ld = p.n_max + 1;
  HyperView hv = p.hv;
  const double cls = p.cls[slot];                        // < 0: labels as uploaded
  double* fg = p.f + static_cast<size_t>(p.mode[slot]) * p.n;
  hv.kf = p.kf[slot];
  hv.beta += slot * p.slot_stride; hv.h_coef += slot * p.slot_stride; hv.h_value += slot * p.slot_stride;
  fg += r0 - fr;                                         // the expert's modes
  double* K = sm;                                        // full symmetric
  double* M = K + static_cast<size_t>(p.n_max) * ld;     // B -> L -> L^-1 -> B^-1 (lower)
  double* v = M + static_cast<size_t>(p.n_max) * ld;     // vectors, n_max each
  double *f = v, *yv = v + p.n_max, *pi = v + 2 * p.n_max, *sw = v + 3 * p.n_max, *glp = v + 4 * p.n_max,
         *bv = v + 5 * p.n_max, *av = v + 6 * p.n_max, *nf = v + 7 * p.n_max, *t1 = v + 8 * p.n_max,
         *t2 = v + 9 * p.n_max, *s2 = v + 10 * p.n_max, *wv = v + 11 * p.n_max;
  double* red = v + 12 * p.n_max;                        // [8]
  double* sums = red + 8;                                // [EX_SUMS]
  double* Xs = sums + EX_SUMS;                           // staged rows (if they fit)
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  int xld;
  const double* Xe = ex_stage_rows(p.X + static_cast<size_t>(r0) * hv.d, n, hv.d, p.x_in_smem, Xs, xld);

  for (int i = tid; i < n; i += LT) {
    f[i] = fg[i];
    yv[i] = (cls < 0.0) ? p.y[r0 + i] : (p.y[r0 + i] == cls ? 1.0 : 0.0);
  }
  __syncthreads();
  ex_build_kernel<true>(hv, Xe, xld, n, K, ld);        // K, both triangles
  __syncthreads();

  // ---- Newton iteration for the mode (GPCls:79-111) ------------------------------------------------------------------
  double old_obj = -INFINITY, new_obj = -1.7976931348623157e308;   // Double.NegativeInfinity, Double.MinValue
  double step = 1.0, sumlogL = 0.0;
  bool bad = false;
  while (fabs(old_obj - new_obj) > p.tol && step > p.tol) {
    for (int i = tid; i < n; i += LT) {
      const double s = sigmoid(f[i]);
      pi[i] = s;
      wv[i] = s * (1.0 - s);
      sw[i] = sqrt(wv[i]);
      glp[i] = yv[i] - s;
    }
    __syncthreads();
    for (int a = warp; a < n; a += EX_WARPS)             // B = I + sqrtW K sqrtW   (GPCls:95-97), lower
      for (int b = lane; b <= a; b += 32) M[a * ld + b] = sw[a] * sw[b] * K[a * ld + b] + (a == b ? 1.0 : 0.0);
    __syncthreads();
    sumlogL = ex_cholesky(M, n, ld, t2, red, bad);            // GPCls:98
    for (int i = tid; i < n; i += LT) bv[i] = wv[i] * f[i] + glp[i];           // b = W f + grad log p   (:100)
    __syncthreads();
    for (int i = tid; i < n; i += LT) {                  // rhs = sqrtW (K b)
      double s = 0.0;
      for (int k = 0; k < n; ++k) s += K[i * ld + k] * bv[k];
      t1[i] = sw[i] * s;
    }
    fwd_solve(M, n, ld, t1);                             // L \ rhs
    bwd_solve(M, n, ld, t1);                             // L^T \ .
    for (int i = tid; i < n; i += LT) av[i] = bv[i] - sw[i] * t1[i];           // a   (:101)
    __syncthreads();
    double part = 0.0;
    for (int i = tid; i < n; i += LT) {                  // f_candidate = (1-step) f + step K a   (:102)
      double s = 0.0;
      for (int k = 0; k < n; ++k) s += K[i * ld + k] * av[k];
      const double c = (1.0 - step) * f[i] + step * s;
      nf[i] = c;
      part += -0.5 * av[i] * c + log(sigmoid((yv[i] * 2.0 - 1.0) * c));        // (:103)
    }
    const double cand = ex_block_sum(part, red);
    if (cand > old_obj) {                                // (:104-107)
      for (int i = tid; i < n; i += LT) f[i] = nf[i];
      old_obj = new_obj;
      new_obj = cand;
    } else {
      step *= 0.5;
    }
    __syncthreads();
  }
  if (bad && tid == 0) atomicOr(p.flags + slot, 1);
  for (int i = tid; i < n; i += LT) fg[i] = f[i];   // the mode persists (warm start of the next evaluation)

  // ---- log Z and gradient (GPCls:114-128) --------------------------------------------------------------------------
  double* out = p.out + (static_cast<size_t>(slot) * gridDim.x + blockIdx.x) * (1 + hv.n_hypers);
  if (tid == 0) out[0] = -(new_obj - sumlogL);
  ex_invert_lower(M, n, ld, t1);                         // L^-1 in place
  // diag(C^T C), C = L^-1 (sqrtW K):  cc_i = | L^-1 (sw o K[:,i]) |^2   (GPCls:117,119)
  for (int i = warp; i < n; i += EX_WARPS) {
    double acc = 0.0;
    for (int r = lane; r < n; r += 32) {
      double s = 0.0;
      for (int k = 0; k <= r; ++k) s += M[r * ld + k] * sw[k] * K[k * ld + i];
      acc += s * s;
    }
    for (int o = 16; o > 0; o >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, o);
    if (lane == 0) t2[i] = acc;
  }
  __syncthreads();
  for (int i = tid; i < n; i += LT) {
    const double d3 = -(2.0 * pi[i] - 1.0) * pi[i] * pi[i] * exp(-f[i]);        // (:118) sign as in the reference
    s2[i] = -0.5 * (K[i * ld + i] - t2[i]) * d3;                                // (:119)
  }
  __syncthreads();
  ex_ltl_inplace(M, n, ld, t1);                          // B^-1 = L^-T L^-1 (lower);  R = sqrtW B^-1 sqrtW   (GPCls:116)
  auto Rab = [&](int a, int b) { return sw[a] * sw[b] * ((b <= a) ? M[a * ld + b] : M[b * ld + a]); };
  // GPCls:121-126 per hyper-parameter h:  s1 = 1/2 a' dK a - 1/2 tr(R dK),  b = dK glp,  s3 = b - K R b,
  // gradLogZ_h = s1 + s2 . s3.  With u = s2 - R K s2 (K, R symmetric) this is  sum_ab dK[a,b] W_ab,
  //   W = 1/2 (a a' - R) + 1/2 (u glp' + glp u'),
  // i.e. the same pair-weight form as the regression objective: one sweep for all hyper-parameters.
  for (int a = tid; a < n; a += LT) {                    // t1 = K s2
    double s = 0.0;
    for (int b = 0; b < n; ++b) s += K[a * ld + b] * s2[b];
    t1[a] = s;
  }
  __syncthreads();
  for (int a = tid; a < n; a += LT) {                    // t2 = u = s2 - R t1
    double s = 0.0;
    for (int b = 0; b < n; ++b) s += Rab(a, b) * t1[b];
    t2[a] = s2[a] - s;
  }
  __syncthreads();
  ex_descriptor_gradient(
      hv, Xe, xld, n,
      [&](int a, int b) {
        return 0.5 * (av[a] * av[b] - sw[a] * sw[b] * M[a * ld + b]) + 0.5 * (t2[a] * glp[b] + t2[b] * glp[a]);
      },
      -1.0, out + 1, sums, red);                         // -gradLogZ
}

}  // namespace

size_t laplace_smem_bytes(int n_max) {
  return sizeof(double) * (2 * static_cast<size_t>(n_max) * (n_max + 1) + 12 * static_cast<size_t>(n_max) + 8 + EX_SUMS);
}

cudaError_t launch_laplace(const ObjectivePlan& plan, const ExpertSet& ex, const HyperView& hv, double tol,
                           const ObjectiveSlots& sl, double* rows, double* total, int* flags, cudaStream_t s) {
  LapParams p{};
  p.X = ex.X; p.y = ex.y; p.f = sl.f; p.off = ex.off; p.n_max = ex.n_max; p.x_in_smem = plan.x_in_smem;
  p.hv = hv; p.cls = sl.cls; p.mode = sl.mode; p.kf = sl.kf; p.slot_stride = sl.slot_stride; p.n = sl.f_stride;
  p.sets = sl.sets; p.first = sl.first; p.tol = tol; p.out = rows; p.flags = flags;
  const int n_slots = sl.n_slots;
  const long long E = sl.E_max;
  cudaError_t e = allow_dynamic_smem(reinterpret_cast<const void*>(laplace_kernel));
  if (e != cudaSuccess) return e;
  laplace_kernel<<<dim3(static_cast<unsigned>(E), static_cast<unsigned>(n_slots)), LT, plan.smem, s>>>(p);
  e = cudaGetLastError();
  if (e != cudaSuccess) return e;
  return launch_rows_reduce(total, rows, E, 1 + hv.n_hypers, s, n_slots, p.sets, p.first);
}

}  // namespace sgp
