// Internal declarations shared by the translation units of libsgp.so (not part of the C-ABI).
#pragma once

#include <cuda_runtime.h>
#include <cusolverDn.h>
#include <cublas_v2.h>
#include <nccl.h>

#include <cstdint>
#include <string>
#include <vector>

#include "../../include/sgp.h"

namespace sgp {

// SGP_PREC_AUTO runs the int8 Gram on accumulate calls of at least this many points (smaller ones: fp64 DMMA kernel)
constexpr long long kAutoI8MinPoints = 32768;
// ... and only if mean|x^|^2 + mean|z^|^2 <= this budget (posterior mean vs the all-fp64 mode at 4.3 / 5.8 / 7.2 / 7.9:
// 1.8e-6 / 2.4e-6 / 5.7e-6 / 1.0e-5, tools/i8_budget_edge.py)
constexpr double kI8NormBudget = 6.0;
// direct-distance mode: largest scaled squared norm accepted; measured dG 6.6e-7 at ~1300 and 2.7e-6 at ~7700 on
// clustered data (tests: error_growth)
constexpr float kI8DirectR2Max = 2048.f;
// tensor-core distance mode: largest scaled squared norm |x^|^2 of a point or an active point.  fp16 operands would take
// 16384, but the fp32 contraction returns T = 2 x^.z^ - |x^|^2 - |z^|^2 up to +2.9e-3 for coinciding points at 15500
// (+2.0e-3 at 8800, +3.7e-4 at 2200; H100, tests/test_gpu_entry_points.py), and the int8 Gram's fixed-point encoding
// breaks from kappa = 2^T = 1 + 2.05e-3 on (the element would read back as ~0).  4096 keeps kappa < 1 + 2e-3.
constexpr double kI8TensorR2Max = 4096.0;
constexpr int kMaxTerms = 4;      // non-Eye terms of a flattened kernel
constexpr int kTile = 128;        // edge of one G tile (active-set indices per CTA tile)
constexpr int kSMsH100 = 132;      // H100 SXM; the context reads the real count from the device
constexpr size_t kSmemOptInMax = 227 * 1024;   // largest dynamic shared memory a CTA can opt in to (H100)
constexpr int kMaxHypers = 72;     // hyper-parameters of one objective evaluation: 1 scale + 64 ARD betas + a few more
// int8 Gram: three int8 digit planes of one active tile for one 64-point unit, and the largest plane workspace of one
// launch window (3 bytes per point and padded active row: configs[1] 3.1 GB in one window, configs[3] 7.7 GB in two)
constexpr size_t kI8PlaneBytes = 3 * kTile * 64;
constexpr size_t kI8PlaneCapBytes = size_t(4) << 30;
// global-memory Laplace path: the largest workspace of one launch (one slice per CTA of the persistent grid)
constexpr size_t kLaplaceGlobalCapBytes = size_t(4) << 30;
// ... and its largest expert: the kernel build shared with the on-chip kernels indexes rows of the n x n matrix in int
constexpr int kLaplaceGlobalMaxPoints = 46336;
// BCM LU path (sgp_bcm_nll, sgp_bcm_nll_folds): its largest expert, for the same reason; the n x n matrix has leading
// dimension n, so n^2 <= 2^31 - 1
constexpr int kBcmLuMaxPoints = 46340;
// prediction: the fp64 cross kernel of one window of points takes at most this much device memory (configs[1]'s m = 1000:
// 32768 points per window)
constexpr size_t kPredictKBytes = size_t(256) << 20;

// feature standardisation (scale.cu): rows per row block of the column sums, whose partials are added in block order
constexpr long long kScaleRows = 2048;

// sqrt(log2 e): coordinates scaled by it turn exp(-q) into 2^(-q'), one ex2 (int8 modes, fp32 element of the fp64 Gram)
constexpr double kSqrtLog2e = 0x1.337cc2183b050p+0;

// Flattened kernel description (flatten_kernel in api.cu): k(x, z) = sum_t C_t exp(-q_t(x, z)) + [x == z] eye_sum over
// the non-Eye terms t.  Kernels take it by value, as a parameter or inside their parameter struct.
struct KernelFlat {
  int n_terms = 0;                 // non-Eye terms
  double scale[kMaxTerms] = {0};   // C_t
  double eye_sum = 0.0;            // sum of Eye coefficients = whiteNoiseVar
  double self_kernel = 0.0;        // sum of all scales (every leaf has k(x,x) = 1)

  // C_t.  A select chain: a kernel parameter array indexed at run time would be copied to local memory.
  __host__ __device__ double term_scale(int t) const {
    return t == 0 ? scale[0] : t == 1 ? scale[1] : t == 2 ? scale[2] : scale[3];
  }
  // acc + C_t exp(-q) in fp64, one rounding for the product and the sum
  __device__ double fold_term(double acc, int t, double q) const { return fma(term_scale(t), exp(-q), acc); }
};

// Launch parameters of the fused K_mn + Gram kernel (gram_f64.cu).
struct GramParams {
  const void* X;        // n x d row-major, fp32 or fp64
  const double* y;      // n
  long long n;
  int x_is_f32;
  int d, dpad;          // dpad = d rounded up to a multiple of 4
  int m, m_pad;         // m_pad = m rounded up to a multiple of kTile
  // KernelFlat's n_terms and scale[], not the whole struct: the fp32-element kernel runs at its 128-register cap, and a
  // larger parameter block moves its spills (1M x 16, m = 1000: 3 % slower, H100 SXM at 400 W)
  int n_terms;
  double scale[kMaxTerms];
  const double* Zc;    // [n_terms][m_pad][dpad]  centred, beta-scaled active set (Z - centre) * beta (zero padded)
  const double* beta;   // [kMaxTerms + 1][dpad]   per-term feature scales (zero padded), then the centre c of the
                        //                         staged coordinates (v - c) * beta (stats_scales in api.cu)
  double* Gpart;        // [n_slices][m_pad*m_pad] per-slice partial tiles (lower block triangle)
  double* bpart;        // [n_slices][m_pad]
  int n_slices;
  int n_tiles_1d;       // m_pad / kTile
};

// Direct-distance mode of the int8 digit-plane producer (launch_i8_planes).
struct I8Direct {
  int on = 0;            // 1: exponents from fp32 direct-form distances on the CUDA cores (any norms, up to 4 terms)
  int n_terms = 0, dpad4 = 0;
  float w[4] = {0, 0, 0, 0};   // C_t / sum C
  double csum = 0.0;     // sum of the term scales = the fixed-point scale
};

// Grow-only device buffer owned by a context (no cudaMalloc / cudaFree in steady state); freed by its destructor.
struct DevScratch {
  void* p = nullptr;
  size_t cap = 0;
  DevScratch() = default;
  DevScratch(const DevScratch&) = delete;
  DevScratch& operator=(const DevScratch&) = delete;
  ~DevScratch() { if (p) cudaFree(p); }
  template <class T> T* as() const { return static_cast<T*>(p); }
};

// Experts resident on the device for the per-expert objectives: expert e owns rows off[e] .. off[e+1]-1.
struct ExpertSet {
  double* X = nullptr;        // [n][d] expert-major
  double* y = nullptr;        // [n]
  long long* off = nullptr;   // [E+1]
  double* f = nullptr;        // [n] latent mode of the Laplace approximation (warm start across evaluations)
  long long E = 0, n = 0;
  int d = 0, n_max = 0;       // n_max: largest expert
};

// Latent modes of the Laplace objective for `slots` mode slots (0: none since the last upload).
struct ModeStore {
  DevScratch buf;
  int slots = 0;
};

struct Ctx {
  int device = 0;
  int precision = SGP_PREC_AUTO;
  int last_path = -1;    // path of the last statistics launch (SGP_PREC_F64 / _F64_STRICT / _I8 / _I8_DIRECT)
  std::string err;
  cudaStream_t stream = nullptr;       // compute
  cudaStream_t copy_stream = nullptr;  // H2D staging
  cudaStream_t tail_stream = nullptr;  // second chain of the m x m tail (inv(K_mm) next to the A chain)
  cusolverDnHandle_t solver = nullptr;
  cusolverDnHandle_t solver2 = nullptr;   // bound to tail_stream
  cublasHandle_t blas = nullptr;
  cudaEvent_t tail_fork = nullptr, tail_join = nullptr;
  DevScratch tail_ws, tail_ws2, predict_ws, cross_ws, bcm_ws, sweep_ws, greedy_ws;
  DevScratch kmeans_pts_ws, kmeans_cen_ws, kmeans_new_ws, kmeans_cand_ws;   // sgp_kmeans: point-, centre-, candidate-sized
  DevScratch kmeans_rows_ws;           // sgp_kmeans_device: indices and fp64 copies of the rows the host reads
  DevScratch kmeans_comm_ws;           // sgp_kmeans_sharded: the buffers its collectives sum over the ranks
  DevScratch scale_ws;                 // sgp_column_sums_device, sgp_scale_apply_device: [2][d] column values, then
                                       // the [row blocks][d] partial sums
  bool has_magic_run = false;
  bool tail_fast = false;              // last sgp_magic took the Cholesky path for both matrices
  ncclComm_t comm = nullptr;
  int rank = 0, nranks = 1;
  int num_sms = kSMsH100;

  // active set / kernel (valid after a successful begin; the buffers are grow-only and may be larger than the shape)
  bool begun = false, finished = false, has_magic = false;
  bool range_failed = false;           // the window's finish reported SGP_E_RANGE: its statistics are not a model's
  int m = 0, d = 0, dpad = 0, m_pad = 0;
  KernelFlat kf;
  DevScratch dZ;      // m x d raw active set (fp64)
  DevScratch dZs;     // [n_terms][m_pad][dpad]  Z * beta (K_mm, cross kernel, prediction)
  DevScratch dZc;     // [n_terms][m_pad][dpad]  (Z - centre) * beta (fp64 statistics kernel)
  DevScratch dBeta;   // [kMaxTerms][dpad], then [dpad] the centre of the fp64 statistics kernel
  DevScratch dGb;     // packed [G (m*m) ; b (m) ; status] -- one all-reduce
  DevScratch gpart_ws, bpart_ws;   // per-slice partial tiles of the statistics kernels
  // int8 exact-accumulation path (gram_i8.cu operand preparation, gram_i8_wgmma.cu Gram kernel).  Two modes:
  // tensor-core distances (one non-Eye term, d <= 32) and direct fp32 distances (1..4 non-Eye terms, n_terms * dpad <= 72);
  // the first qualifies only where the second does, and both use the same scales, centre and active-set norm.
  bool i8_ok = false;            // the kernel/shape qualifies for tensor-core distances
  bool i8_direct_ok = false;     // ... for direct distances
  DevScratch dI8Scale;           // [kMaxTerms][dpad] sqrt(log2 e) * beta_tk, then [dpad] centre (active-set mean)
  double i8_z_norm_mean = 0.0;   // mean scaled squared norm of the active set (widest term), for AUTO's budget
  I8Direct i8_direct;            // direct mode's term weights and fixed-point scale (used where i8_direct_ok)
  DevScratch dI8Zt;              // tensor-core mode: active-set operand images
  DevScratch i8_zd_ws;           // direct mode: active-set tiles [tile][term][dpad][128] fp32
  bool i8d_prepared = false;     // ... built in this begin() window (on the first direct-mode launch)
  DevScratch i8_xt_ws, i8_ys_ws; // point operand images / tiles and fp32 y (scratch)
  DevScratch i8_planes_ws;       // digit planes of one launch window (at most kI8PlaneCapBytes)
  DevScratch dI8Flags;           // int [0] the window's int8 status, [1] the active set's (begin), [2] the K_nm sweep's
                                 // (reset to [1] by each host-form call); bit 0: scaled squared norm above
                                 // kI8TensorR2Max; bit 2: above kI8DirectR2Max
  DevScratch dI8NormSum;         // [0]: sum of |x^|^2 over every int8 chunk since begin; [1]: first chunk of this call
  int call_path = SGP_PREC_F64;  // path of the current accumulate call (AUTO decides on its first chunk: stats_path)
  int i8_flag_mask = 0;          // dI8Flags bits the int8 launches since begin can have set (0: no int8 launch)
  long long i8_points = 0;       // points that went through the int8 kernel since begin
  // per-expert objective state
  ExpertSet ex;                  // view of ex_X, ex_y, ex_off, ex_f; E > 0 once an upload has completed
  DevScratch ex_X, ex_y, ex_off;
  ModeStore ex_f;                // the binary objectives' latent modes: one slot of n (ex.f), zeroed by every upload
  ModeStore ex_fc;               // one-vs-rest latent modes [classes][n] (sgp_laplace_nll_classes)
  ModeStore ex_fm;               // param-map latent modes [mode slots][n] (sgp_laplace_nll_slots_any_size)
  ModeStore ex_ffm;              // fold-slot latent modes [mode slots][largest set's rows]
                                 // (sgp_laplace_nll_fold_slots_any_size), indexed from each set's first row
  bool ex_grouped = false;       // ex came from a grouped upload (point i -> expert i % E): its modes can be ungrouped
  // fold upload (sgp_experts_upload_folds): the training sets lie one after another in ex; set k owns the experts
  // fold_first[k] .. fold_first[k+1]-1.  Empty after any other upload.
  std::vector<long long> fold_first;   // [n_sets + 1]
  std::vector<int> fold_nmax;          // [n_sets] largest expert of each set
  std::vector<long long> fold_row0;    // [n_sets + 1] first row of each set
  DevScratch fold_pos_ws;              // upload scratch: the point indices grouped by fold, ascending in each fold
  DevScratch nll_per_ws;         // per-expert objective rows
  DevScratch hyper_ws;           // hyper-parameter descriptors + totals + flags of one evaluation
  bool bcm_general = false;      // the last sgp_bcm_nll took the global-memory LU path
  int laplace_path = -1;         // the last sgp_laplace_nll*: 0 on chip, 1 global memory, -1 none yet
  DevScratch laplace_ws;         // laplace_global_kernel: one workspace slice per CTA
  // tail / predict state
  DevScratch dMagicVec;          // m
  DevScratch dMagicMat;          // m x m
  DevScratch dMagicPacked;       // m_pad x m_pad  triu(M + M^T, 1) + diag(M), built by the first variance call
  bool magic_packed = false;     // dMagicPacked holds the installed magicMatrix
  DevScratch predict_out_ws;     // sgp_predict*: [2][mean | var | p] per window (double buffered)
  DevScratch keval_ws;           // sgp_kernel_eval*: descriptor tables, then (host entry) the staged training vectors
  DevScratch keval_out_ws;       // sgp_kernel_eval: [2][K | dK] per window (double buffered)
  DevScratch dGhRule;            // [nodes | weights] of the gh_nodes-node Gauss-Hermite rule (sgp_predict_probability*)
  int gh_nodes = 0;              // 0: none uploaded yet
  // host->device staging (double buffered)
  DevScratch stage_x[2], stage_y[2];
  cudaEvent_t stage_free[2] = {nullptr, nullptr};   // recorded when the kernel consuming buffer i is done
  cudaEvent_t stage_ready[2] = {nullptr, nullptr};  // recorded when the H2D into buffer i is done
  cudaEvent_t out_ready[2] = {nullptr, nullptr};    // sgp_predict: the window writing output buffer i is done
  cudaEvent_t out_free[2] = {nullptr, nullptr};     // sgp_predict: the device->host copy out of buffer i is done
  // instrumentation
  int64_t launches = 0;
  std::vector<std::pair<cudaEvent_t, cudaEvent_t>> gram_events;   // event POOL (created once, reused)
  size_t gram_events_used = 0;                                    // pairs recorded since the last begin
  cudaEvent_t user_events[8] = {nullptr};
  DevScratch dbgT, dbgW;       // sgp_debug_i8_tile: fp32 T and uint32 words
};

// Opts kernel fn in to dynamic shared memory above 48 KiB.  Launchers call it before every launch of such a kernel and
// pass their own plan's size to the launch itself.  The cap is an attribute of the function on the current device, shared
// by every context of the process on that device (one per Spark task thread), so it is one value per kernel -- the
// largest a CTA can opt in to -- never the size of the call at hand: a context that set its small plan's size between
// another context's set and launch would get that launch refused.  Concurrent sets all write the same value.  Static and
// dynamic shared memory share the opt-in maximum, so the cap is that maximum less the kernel's static shared memory
// (predict_var_kernel declares some; a larger cap is refused).  This is the only place in csrc/ that sets
// cudaFuncAttributeMaxDynamicSharedMemorySize (tests/test_host_concurrent_contexts.py checks it).
inline cudaError_t allow_dynamic_smem(const void* fn) {
  cudaFuncAttributes a;
  const cudaError_t e = cudaFuncGetAttributes(&a, fn);
  if (e != cudaSuccess) return e;
  return cudaFuncSetAttribute(fn, cudaFuncAttributeMaxDynamicSharedMemorySize,
                              static_cast<int>(kSmemOptInMax - a.sharedSizeBytes));
}

// error helpers ---------------------------------------------------------------------------------
int fail(Ctx* c, int code, const std::string& msg);
#define SGP_CUDA(c, expr)                                                                         \
  do {                                                                                            \
    cudaError_t e_ = (expr);                                                                      \
    if (e_ != cudaSuccess)                                                                        \
      return ::sgp::fail((c), SGP_E_CUDA, std::string(#expr) + ": " + cudaGetErrorString(e_));    \
  } while (0)

// kernels (each returns a cudaError_t from the launch) -----------------------------------------
cudaError_t launch_gram_f64(const GramParams& p, bool strict_elements, cudaStream_t s);
cudaError_t launch_gram_reduce(double* G /*m x m*/, double* b, const double* Gpart, const double* bpart,
                               int n_slices, int m, int m_pad, cudaStream_t s);
// same for partial tiles at the mirror position (int8 Gram), with separate slice counts for G and b
cudaError_t launch_gram_reduce_upper(double* G, double* b, const double* Gpart, const double* bpart, int g_slices,
                                     int b_slices, int m, int m_pad, cudaStream_t s);
// out = in * beta; out_centred (optional) = (in - centre) * beta; both zero padded to [rows_out][dpad]
cudaError_t launch_scale_rows(double* out /*[rows][dpad]*/, double* out_centred, const double* in /*rows x d*/,
                              const double* beta, const double* centre, int rows_in, int rows_out, int d, int dpad,
                              cudaStream_t s);
cudaError_t launch_kmm_build(double* Kmm /*m x m*/, const double* Zs, const KernelFlat& kf, int m, int m_pad, int dpad,
                             cudaStream_t s);
cudaError_t launch_cross_kernel(double* K /*n x m*/, const double* X /*n x d*/, const double* Zs,
                                const double* beta, const KernelFlat& kf, long long n, int d, int dpad,
                                int m, int m_pad, cudaStream_t s);
cudaError_t launch_axpby_diag(double* A, const double* K, const double* G, double wn, int m, cudaStream_t s);
cudaError_t launch_set_identity(double* I, int m, cudaStream_t s);
cudaError_t launch_magic_matrix(double* out, const double* invA, const double* invK, double wn, int m,
                                cudaStream_t s);
// Gathers the staged points [p0, p0 + cn) of a training set of n points into E experts.  skip_pos (optional): the sorted
// indices of the n_skip points left out of the set (a validation fold); a kept point's training rank is its index minus
// the left-out points before it.  Without skip_pos every point is kept at its own index.
cudaError_t launch_group_experts(double* Xe, double* ye, const void* dX, int x_is_f32, const double* dy, long long n, int d,
                                 long long E, long long p0, long long cn, const long long* skip_pos, long long n_skip,
                                 cudaStream_t s);
// The inverse of the grouping: out[i] = f[row of point i], point i being expert i % E's (i / E)-th point.
cudaError_t launch_ungroup_experts(double* out, const double* f, long long n, long long E, cudaStream_t s);
// off[e] = base + start of expert e of n points grouped into E experts, e = 0 .. E
cudaError_t launch_expert_offsets(long long* off, long long n, long long E, long long base, cudaStream_t s);
cudaError_t launch_status_to_double(double* dst, const int* flags, int mask, const double* norm_sum, double norm_limit,
                                    cudaStream_t s);
// dst[i] = (flags[i] & mask) ? 1 : 0 for i < n: the per-slot status words of an objective evaluation
cudaError_t launch_flags_to_double(double* dst, const int* flags, int mask, int n, cudaStream_t s);

// Feature standardisation (scale.cu) of n x d device rows (fp32 or fp64), on stream s.  launch_column_sums: out[k] =
// sum_i x_ik, or with centre sum_i (x_ik - centre_k)^2; part holds scale_row_blocks(n) x d partials.  launch_scale_apply:
// Y[i][k] = (x_ik - mean_k) / sd_k.  n >= 1; centre, mean, sd, part, out and Y are device memory.
long long scale_row_blocks(long long n);
cudaError_t launch_column_sums(const void* X, int x_is_f32, long long n, int d, const double* centre, double* part,
                               double* out, cudaStream_t s);
cudaError_t launch_scale_apply(const void* X, int x_is_f32, long long n, int d, const double* mean, const double* sd,
                               double* Y, cudaStream_t s);

// Prediction (predict.cu) over one window of device-resident points.
struct PredictArgs {
  const void* X;         // n x d row-major, fp32 or fp64
  int x_is_f32;
  long long n;           // <= predict_window_points(m_pad)
  int d, dpad, m, m_pad;
  KernelFlat kf;
  const double* Zc;      // [n_terms][m_pad][dpad] (Z - c) * beta
  const double* beta;    // [kMaxTerms][dpad] beta, then [dpad] c
  const double* v;       // m: magic vector
  const double* B;       // m_pad x m_pad packed magic matrix (launch_pack_magic); variance only
  double* ws;            // predict_ws_bytes(window, m_pad); variance only
  double* mean;          // n; nullptr only with prob (the mean then lands in ws)
  double* var;           // n, or nullptr: mean only (or not returned by a probability call)
  const double* rule;    // [n_nodes nodes | n_nodes weights] of the Gauss-Hermite rule; probability only
  int n_nodes;
  double* prob;          // n averaged probabilities, or nullptr (predict_var_reduce_kernel<true>)
};
long long predict_window_points(int m_pad);
size_t predict_ws_bytes(long long window, int m_pad);
// The n-node Gauss-Hermite rule for the weight exp(-x^2) (host code): nodes ascending, exactly symmetric.  false for n
// outside [1, kMaxHermiteNodes] or a null output.
constexpr int kMaxHermiteNodes = 256;
bool gauss_hermite_rule(int n, double* nodes, double* weights);
cudaError_t launch_pack_magic(double* B /*m_pad x m_pad*/, const double* M /*m x m*/, int m, int m_pad, cudaStream_t s);
cudaError_t launch_predict(const PredictArgs& a, cudaStream_t s);

// int8 exact-accumulation path
size_t i8_points_scratch_bytes(long long n, int nchunks);
size_t i8_active_scratch_bytes(int m_pad, int nchunks);
int i8_nchunks(int d);
cudaError_t launch_i8_prep_active(uint8_t* Zt, const double* dZ, int m, int m_pad, int d, const double* dScale,
                                  const double* dCentre, int* dFlags, cudaStream_t s);
cudaError_t launch_i8_prep_points(uint8_t* Xt, float* ys, const void* dX, int x_is_f32, const double* dy, long long n,
                                  int d, const double* dScale, const double* dCentre, int* dFlags, double* dNormSum,
                                  double* dNormSumCall, cudaStream_t s);
// direct-distance mode of the int8 Gram: fp32 coordinate tiles instead of fp16 operand images
cudaError_t launch_i8_prep_active_direct(float* Zd, const double* dZ, int m, int m_pad, int d, int dpad4, int n_terms,
                                         const double* dScale, const double* dCentre, int* flags, float r2max,
                                         cudaStream_t s);
cudaError_t launch_i8_prep_points_direct(float* Xd, float* ys, const void* dX, int x_is_f32, const double* dy, long long n,
                                         int d, int dpad4, int n_terms, const double* dScale, const double* dCentre, int* flags,
                                         float r2max, double* dNormSum, double* dNormSumCall, cudaStream_t s);

// int8 Gram (gram_i8_wgmma.cu).  A launch window over n_units 64-point units is two kernels: the digit-plane producer
// (kernel elements, their fixed-point digit planes in the workspace [n_units][m_pad / kTile][kI8PlaneBytes], and the
// b partials) and the int8 Gram over the workspace (partial tiles of the upper block triangle).  accumulate = false:
// the window stores its partials (first window of a call); true: it adds to them.  C: the fixed-point scale (the term
// scale, or the sum of the term scales in direct mode).  The two kernels split a window into point slices of their own:
// i8_slices for the Gram (its G partials), i8_plane_slices for the producer (its b partials).
int i8_slices(int m_pad, int num_sms, long long n_units);
cudaError_t i8_plane_slices(int m_pad, int num_sms, long long n_units, int d, const I8Direct& direct, int* n_slices);
cudaError_t launch_i8_planes(const uint8_t* Xt, const float* ys, const uint8_t* Zt, long long n_units, int d, int m_pad,
                             int n_slices, const I8Direct& direct, double C, bool accumulate, uint8_t* planes,
                             double* bpart, float* dbg_T, uint32_t* dbg_w, cudaStream_t s);
cudaError_t launch_gram_i8(const uint8_t* planes, long long n_units, int m_pad, int n_slices, double C, bool accumulate,
                           double* Gpart, cudaStream_t s);

// K_nm sweep (kmn_sweep.cu): fp32 cross kernel of a block of points, row-major n x m
cudaError_t launch_kmn_sweep(const uint8_t* Xt, const uint8_t* Zt, long long n, int d, int m, int m_pad, int num_sms, double C,
                             float* K, cudaStream_t s);

// Kernel evaluation (kernel_eval.cu, sgp_kernel_eval*): K[i][j] = k(a_i, b_j) for n rows of A against m rows of B, and
// with dK every derivative dK / d theta_h, h in the order of the hyper-parameter descriptors.
struct KernelEvalArgs {
  const void* A;            // n x d row-major, fp32 or fp64
  int a_is_f32;
  const void* B;            // m x d row-major (TRAINING: the training vectors, of which A is rows row0 ..)
  int b_is_f32;
  long long n;
  int m, d;
  int training;             // 1: the Eye sum (and the Eye coefficients of trainable scalars) go on the diagonal
  long long row0;           // A's row i is row row0 + i of the training vectors (the diagonal is row0 + i == j)
  KernelFlat kf;
  const double* beta;       // [n_terms][d] flattened feature scales (ARD betas; RBF: 1/(sqrt2 sigma))
  double* K;                // n x m
  double* dK;               // [n_hypers][dk_stride] (n x m each), or nullptr: K only
  size_t dk_stride;
  const int* ard_h;         // [n_terms][d] hyper-parameter index of (ARD term t, feature k); -1 for an RBF term
  int rbf_h[kMaxTerms];     // hyper-parameter index of RBF term t's sigma, -1 for an ARD term
  double sigma3[kMaxTerms]; // RBF term t: sigma^3
  int n_scale;              // trainable scalars
  const int* scale_h;       // [n_scale] hyper-parameter index
  const double* scale_coef; // [n_scale][kMaxTerms + 1] d(C_t)/d(theta) per flattened term, then d(eye_sum)/d(theta)
};
cudaError_t launch_kernel_eval(const KernelEvalArgs& a, cudaStream_t s);

// Per-expert objectives (bcm_nll.cu, laplace.cu) ----------------------------------------------------------------------
// Device-side view of the flattened kernel and the hyper-parameter descriptors of one evaluation.
struct HyperView {
  int d;
  KernelFlat kf;
  const double* beta;        // [n_terms][d]  per-term coordinate scales (ARD betas; RBF: 1/(sqrt2 sigma))
  int n_hypers, any_ard;
  const int* h_kind;         // [n_hypers] 0 = SCALE, 1 = ARD_BETA, 2 = RBF_SIGMA
  const int* h_term;         // [n_hypers] flattened term index (ARD_BETA / RBF_SIGMA)
  const int* h_dim;          // [n_hypers] feature index (ARD_BETA)
  const double* h_coef;      // [n_hypers][kMaxTerms+1]  SCALE: d(scale_t)/d(theta_i) per term, last = d(eye_sum)/d(theta_i)
  const double* h_value;     // [n_hypers] current value of the hyper-parameter (beta_k or sigma)
};

// kBcmLu: the BCM objective after its Cholesky broke down.  kLaplace: on chip only (refused past the shared-memory
// limit); kLaplaceAnySize: on chip when the largest expert fits, else the global-memory kernel.
enum class Objective { kBcm, kBcmLu, kLaplace, kLaplaceAnySize };
enum class ObjectiveVariant {
  kReg24, kReg36, kReg47, kReg48,   // BCM: bcm_nll_reg_kernel<RBR, RBC>
  kSmem,                            // BCM: bcm_nll_kernel (shared-memory Cholesky)
  kLu,                              // BCM: global-memory LU path (cuBLAS batched LU / inverse)
  kLaplaceGlobal,                   // laplace_global_kernel (matrices in global memory, persistent grid)
  kLaplace,                         // laplace_kernel
  kRefused                          // Laplace: the expert does not fit on chip
};
// Which kernel evaluates an objective on the uploaded experts, with which launch resources (plan_objective, bcm_nll.cu).
struct ObjectivePlan {
  ObjectiveVariant variant = ObjectiveVariant::kRefused;
  int x_in_smem = 0;   // the kernel stages the expert's rows in shared memory
  size_t smem = 0;     // dynamic shared memory per CTA
  size_t lu_ws = 0;    // kLu: global-memory workspace
  int ya_in_ws = 0;    // kLu: y and alpha live in lu_ws (2 n_max doubles do not fit in shared memory)
  size_t cta_ws = 0;   // kLaplaceGlobal: global-memory workspace of one CTA (the launch takes one per CTA)
};
ObjectivePlan plan_objective(Objective kind, const ExpertSet& ex, int n_terms);
size_t laplace_smem_bytes(int n_max);   // laplace_kernel without the staged rows (laplace.cu)
size_t laplace_global_cta_bytes(int n_max);   // laplace_global_kernel's workspace per CTA (laplace_global.cu)

// The slots of a per-expert objective launch (objective_setup in api.cu).  Every objective entry is a list of slots over
// expert sets of the upload: slot s evaluates the experts first[sets[s]] .. first[sets[s] + 1] - 1 (the whole upload is
// the one set {0, E}) with the flattened kernel kf[s] and the descriptor values slot_stride doubles per slot after hv's.
// The Laplace objective adds the labels (y == cls[s]) (cls[s] < 0: the labels as uploaded) and the modes
// f + mode[s] * f_stride, indexed from the set's first row.  rows: [n_slots][E_max][1 + n_hypers], total:
// [n_slots][1 + n_hypers], flags: [n_slots].
struct ObjectiveSlots {
  int n_slots = 0;
  const int* sets = nullptr;          // device, [n_slots]
  const long long* first = nullptr;   // device, [n_sets + 1]
  long long E_max = 0;                // the largest expert count over the slots' sets
  const KernelFlat* kf = nullptr;     // device, [n_slots]
  long long slot_stride = 0;
  const int* cls = nullptr;           // device, [n_slots] (Laplace)
  const int* mode = nullptr;          // device, [n_slots], distinct (Laplace)
  double* f = nullptr;                // device, [n_mode_slots][f_stride] (Laplace)
  long long f_stride = 0;             // modes per mode slot: the uploaded points, or the largest fold set's rows
};
// Each launcher runs the planned kernel over experts x slots and sums each slot's per-expert rows into total.
cudaError_t launch_bcm_nll(const ObjectivePlan& plan, const ExpertSet& ex, const HyperView& hv, const ObjectiveSlots& sl,
                           double* rows, double* total, int* flags, cudaStream_t s);
// The LU path on one set (ex: the set alone).  ws: plan.lu_ws bytes.  cuBLAS failures are reported through *blas_status.
cudaError_t launch_bcm_nll_general(const ObjectivePlan& plan, cublasHandle_t blas, int* blas_status, void* ws,
                                   const ExpertSet& ex, const HyperView& hv, double* rows, double* total, int* flags,
                                   cudaStream_t s);
cudaError_t launch_laplace(const ObjectivePlan& plan, const ExpertSet& ex, const HyperView& hv, double tol,
                           const ObjectiveSlots& sl, double* rows, double* total, int* flags, cudaStream_t s);
// The global-memory kernel (plan kLaplaceGlobal) on `grid` CTAs, CTA b on the slice ws + b * plan.cta_ws.  The grid
// is laplace_global_grid(E_max * n_slots, laplace_global_ctas_per_sm() * SMs, plan.cta_ws, workspace budget).
int laplace_global_ctas_per_sm();
long long laplace_global_grid(long long items, long long resident, size_t cta_bytes, size_t budget);
cudaError_t launch_laplace_global(const ExpertSet& ex, const HyperView& hv, double tol, double* ws, long long grid,
                                  const ObjectiveSlots& sl, double* rows, double* total, int* flags, cudaStream_t s);

int ctx_scratch(Ctx* c, DevScratch& s, size_t bytes);
// X and y below are host memory, or device memory on the context's device where x_on_device is set (the _device entries)
// csrc/greedy.cu: forward selection with rank-1 updates (ActiveSetProvider.scala:58-139); beta_flat = [n_terms][d]
int run_greedy(Ctx* c, const KernelFlat& kf, const std::vector<double>& beta_flat, const double* X, const double* y,
               bool x_on_device, long long n, int d, long long n_experts, long long first_index, int m_target,
               long long* indices_out);
// csrc/kmeans.cu: Spark 3.1 MLlib KMeans (k-means|| + Lloyd) for KMeansActiveSetProvider (ActiveSetProvider.scala:22-46)
int run_kmeans(Ctx* c, const void* X, int x_is_f32, bool x_on_device, long long n, int d, int k, int max_iter, double tol,
               uint64_t seed, const double* init_centers, double* centers_out, int* k_out, int* labels_out,
               int* iterations_out, double* cost_out);
// the same algorithm on the concatenation of the ranks' rows (this rank: global rows [offset, offset + n) of n_total); its
// collectives go over c's communicator
int run_kmeans_sharded(Ctx* c, const void* X, int x_is_f32, bool x_on_device, long long n, long long offset,
                       long long n_total, int d, int k, int max_iter, double tol, uint64_t seed, const double* init_centers,
                       double* centers_out, int* k_out, int* labels_out, int* iterations_out, double* cost_out);
// in-place sum of count elements of device memory over c's communicator, on c's stream (a no-op for one rank)
int comm_sum(Ctx* c, void* buf, size_t count, ncclDataType_t type);
int run_tail(Ctx* c, double* magic_vector, double* magic_matrix);
// Prediction (tail.cu): predict_prepare sizes the workspace and packs the installed magic matrix (once per pair) for the
// windows that follow; predict_window enqueues one window of at most predict_window_points(m_pad) device-resident points.
// n_nodes > 0 (a probability call) also makes sure dGhRule holds that rule.  dP: the averaged probabilities (dMean may
// then be nullptr).
int predict_prepare(Ctx* c, bool with_var, int n_nodes = 0);
int predict_window(Ctx* c, const void* dX, int x_is_f32, long long n, double* dMean, double* dVar, double* dP = nullptr);

}  // namespace sgp
