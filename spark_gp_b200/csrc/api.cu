// C-ABI entry points (include/sgp.h): context, multi-GPU plumbing, the statistics pipeline.
#include "sgp_internal.h"

#include <dlfcn.h>

#include <algorithm>
#include <cmath>
#include <cstring>
#include <new>
#include <numeric>
#include <utility>

namespace sgp {

static thread_local std::string g_create_err;

// NCCL is resolved lazily with dlopen instead of being a link-time dependency: a host process that also
// loads PyTorch already carries torch's own libnccl.so.2, and two different NCCL builds under one soname
// cannot coexist.  dlopen("libnccl.so.2") returns the copy that is already mapped, else the system one.
struct NcclApi {
  ncclResult_t (*GetUniqueId)(ncclUniqueId*) = nullptr;
  ncclResult_t (*CommInitRank)(ncclComm_t*, int, ncclUniqueId, int) = nullptr;
  ncclResult_t (*AllReduce)(const void*, void*, size_t, ncclDataType_t, ncclRedOp_t, ncclComm_t, cudaStream_t) = nullptr;
  ncclResult_t (*CommDestroy)(ncclComm_t) = nullptr;
  const char* (*GetErrorString)(ncclResult_t) = nullptr;
  bool ok = false;
};
static NcclApi& nccl() {
  static NcclApi api = [] {
    NcclApi a;
    void* h = dlopen("libnccl.so.2", RTLD_LAZY | RTLD_LOCAL);
    if (!h) h = dlopen("libnccl.so", RTLD_LAZY | RTLD_LOCAL);
    if (!h) return a;
    a.GetUniqueId = reinterpret_cast<decltype(a.GetUniqueId)>(dlsym(h, "ncclGetUniqueId"));
    a.CommInitRank = reinterpret_cast<decltype(a.CommInitRank)>(dlsym(h, "ncclCommInitRank"));
    a.AllReduce = reinterpret_cast<decltype(a.AllReduce)>(dlsym(h, "ncclAllReduce"));
    a.CommDestroy = reinterpret_cast<decltype(a.CommDestroy)>(dlsym(h, "ncclCommDestroy"));
    a.GetErrorString = reinterpret_cast<decltype(a.GetErrorString)>(dlsym(h, "ncclGetErrorString"));
    a.ok = a.GetUniqueId && a.CommInitRank && a.AllReduce && a.CommDestroy && a.GetErrorString;
    return a;
  }();
  return api;
}

int fail(Ctx* c, int code, const std::string& msg) {
  if (c) {
    c->err = msg;
  } else {
    g_create_err = msg;
  }
  return code;
}

// Flattens a kernel description: Eye terms drop out of the cross kernel (kernel/Kernel.scala:157) and only sum their
// coefficients into eye_sum; the other terms' feature scales go to beta = [kMaxTerms][beta_stride] (zero padded).
// flat_of (optional) receives the flattened index of every term, -1 for Eye terms.
static int flatten_kernel(Ctx* c, const sgp_kernel_desc* k, int d, int beta_stride, KernelFlat& kf,
                          std::vector<double>& beta, std::vector<int>* flat_of) {
  kf = KernelFlat{};
  beta.assign(static_cast<size_t>(kMaxTerms) * beta_stride, 0.0);
  if (flat_of) flat_of->assign(k->n_terms, -1);
  for (int t = 0; t < k->n_terms; ++t) {
    const sgp_kernel_term& term = k->terms[t];
    if (!(term.scale >= 0.0)) return fail(c, SGP_E_BADARG, "requirement failed: C should be positive");
    kf.self_kernel += term.scale;
    if (term.type == SGP_TERM_EYE) { kf.eye_sum += term.scale; continue; }
    if (kf.n_terms == kMaxTerms) return fail(c, SGP_E_BADARG, "too many non-Eye kernel terms (max 4)");
    double* bt = beta.data() + static_cast<size_t>(kf.n_terms) * beta_stride;
    if (term.type == SGP_TERM_ARD) {
      if (!term.beta) return fail(c, SGP_E_BADARG, "ARD term without beta");
      for (int j = 0; j < d; ++j) bt[j] = term.beta[j];
    } else if (term.type == SGP_TERM_RBF) {
      if (!(term.sigma > 0.0)) return fail(c, SGP_E_BADARG, "RBF sigma must be > 0");
      // exp(-|x-z|^2 / (2 sigma^2)) = exp(-sum_k (x_k - z_k)^2 beta^2), beta = 1/(sqrt(2) sigma)
      for (int j = 0; j < d; ++j) bt[j] = 1.0 / (std::sqrt(2.0) * term.sigma);
    } else {
      return fail(c, SGP_E_BADARG, "unknown kernel term type");
    }
    if (flat_of) (*flat_of)[t] = kf.n_terms;
    kf.scale[kf.n_terms++] = term.scale;
  }
  return SGP_OK;
}

// Streams the host rows X (n rows of `row` bytes) and y through the two staging buffers, so that the copy of one chunk
// (copy_stream) overlaps the kernels of the previous one (compute stream).  The first chunk has `first` points, the
// others `chunk` (first <= chunk); launch(dX, dy, p0, cn) enqueues the consumer of points [p0, p0 + cn) on the compute
// stream.  y may be NULL (points without labels: dy is then NULL).  Returns when every copy is done: the caller may
// reuse X and y.
template <class Launch>
static int stage_rows(Ctx* c, const void* X, const double* y, long long n, size_t row, long long first, long long chunk,
                      Launch&& launch) {
  const size_t xb = row * chunk, yb = y ? static_cast<size_t>(chunk) * 8 : 0;
  if (xb > c->stage_x[0].cap || yb > c->stage_y[0].cap) {
    SGP_CUDA(c, cudaStreamSynchronize(c->stream));
    SGP_CUDA(c, cudaStreamSynchronize(c->copy_stream));
    for (int i = 0; i < 2; ++i) {
      int rc = ctx_scratch(c, c->stage_x[i], xb);
      if (rc == SGP_OK && yb > 0) rc = ctx_scratch(c, c->stage_y[i], yb);
      if (rc != SGP_OK) return rc;
      SGP_CUDA(c, cudaEventRecord(c->stage_free[i], c->stream));
    }
  }
  const char* Xb = static_cast<const char*>(X);
  int buf = 0;
  for (long long p0 = 0, step = first; p0 < n; p0 += step, step = chunk, buf ^= 1) {
    const long long cn = (n - p0 < step) ? (n - p0) : step;
    void* sx = c->stage_x[buf].p;
    double* sy = y ? c->stage_y[buf].as<double>() : nullptr;
    SGP_CUDA(c, cudaStreamWaitEvent(c->copy_stream, c->stage_free[buf], 0));
    SGP_CUDA(c, cudaMemcpyAsync(sx, Xb + static_cast<size_t>(p0) * row, row * cn, cudaMemcpyHostToDevice, c->copy_stream));
    if (y) SGP_CUDA(c, cudaMemcpyAsync(sy, y + p0, static_cast<size_t>(cn) * 8, cudaMemcpyHostToDevice, c->copy_stream));
    SGP_CUDA(c, cudaEventRecord(c->stage_ready[buf], c->copy_stream));
    SGP_CUDA(c, cudaStreamWaitEvent(c->stream, c->stage_ready[buf], 0));
    const int rc = launch(sx, sy, p0, cn);
    if (rc != SGP_OK) return rc;
    SGP_CUDA(c, cudaEventRecord(c->stage_free[buf], c->stream));
  }
  SGP_CUDA(c, cudaStreamSynchronize(c->copy_stream));
  return SGP_OK;
}

// stage_rows for rows that are host memory, or the same chunks read in place where X and y are device memory already
template <class Launch>
static int feed_rows(Ctx* c, bool on_device, const void* X, const double* y, long long n, size_t row, long long chunk,
                     Launch&& launch) {
  if (!on_device) return stage_rows(c, X, y, n, row, chunk, chunk, launch);
  for (long long p0 = 0; p0 < n; p0 += chunk) {
    const long long cn = (n - p0 < chunk) ? (n - p0) : chunk;
    const int rc = launch(static_cast<const char*>(X) + static_cast<size_t>(p0) * row, y ? y + p0 : nullptr, p0, cn);
    if (rc != SGP_OK) return rc;
  }
  return SGP_OK;
}

// The pointer check of the _device entries: p must be device (or managed) memory on the context's device.  Refused
// before any allocation or launch, so that a host pointer never reaches a kernel.
static int device_ptr_ok(Ctx* c, const void* p, const char* entry, const char* what) {
  cudaPointerAttributes a{};
  const cudaError_t e = cudaPointerGetAttributes(&a, p);
  if (e != cudaSuccess) cudaGetLastError();
  if (e != cudaSuccess || (a.type != cudaMemoryTypeDevice && a.type != cudaMemoryTypeManaged) || a.device != c->device)
    return fail(c, SGP_E_BADARG, std::string(entry) + ": " + what + " is not device memory on device " +
                                     std::to_string(c->device));
  return SGP_OK;
}

// Host state of the statistics kernels for the active set Z (m x d) and the flattened beta ([kMaxTerms][dpad]):
// sc = [kMaxTerms][dpad] sqrt(log2 e) * beta_tk (int8 modes only, with_scales), then the [dpad] centre of the int8 modes,
// the active-set mean; ctr64 = [dpad] the centre of the fp64 kernel.  Distances are translation invariant, and centred
// operands keep the rounding of the staged coordinates proportional to the spread of the data instead of to their
// distance from the origin.  The fp64 kernel's centre is the mean rounded to a whole multiple of the active set's
// standard deviation in that dimension (the mean itself where the deviation is 0).  It lies within half a deviation of
// the mean, which removes any offset just as well, and it is exactly 0 for data that are centred already (standardised
// features): those keep the arithmetic they had without a centre.  The fp32 rounding of the active set is common to all
// the kernel values of an active point and does not average out over points; moving centred data by a fraction of a
// deviation re-draws it for no gain in expectation (airfoil, cond(A) ~ 6e7: posterior mean 6.7e-6 -> 1.2e-5 off the
// all-fp64 mode).
// Returns the mean scaled squared norm of the active set under the widest term, which AUTO's magnitude budget adds to the
// points' mean.
static double stats_scales(const double* Z, int m, int d, int dpad, int n_terms, const std::vector<double>& beta,
                           bool with_scales, std::vector<double>& sc, double* ctr64) {
  sc.assign(static_cast<size_t>(kMaxTerms + 1) * dpad, 0.0);
  double* ctr = sc.data() + static_cast<size_t>(kMaxTerms) * dpad;
  for (int j = 0; j < d; ++j) {
    double acc = 0.0;
    for (int i = 0; i < m; ++i) acc += Z[static_cast<size_t>(i) * d + j];
    ctr[j] = acc / m;
    double var = 0.0;
    for (int i = 0; i < m; ++i) {
      const double v = Z[static_cast<size_t>(i) * d + j] - ctr[j];
      var += v * v;
    }
    const double sd = std::sqrt(var / m);
    ctr64[j] = sd > 0.0 ? std::nearbyint(ctr[j] / sd) * sd : ctr[j];
  }
  if (!with_scales) return 0.0;
  for (int t = 0; t < n_terms; ++t)
    for (int j = 0; j < d; ++j) sc[static_cast<size_t>(t) * dpad + j] = kSqrtLog2e * beta[static_cast<size_t>(t) * dpad + j];
  double best = 1e300;
  for (int t = 0; t < n_terms; ++t) {
    const double* st = sc.data() + static_cast<size_t>(t) * dpad;
    double zsum = 0.0;
    for (int i = 0; i < m; ++i)
      for (int j = 0; j < d; ++j) {
        const double v = (Z[static_cast<size_t>(i) * d + j] - ctr[j]) * st[j];
        zsum += v * v;
      }
    best = std::min(best, zsum / m);
  }
  return best;
}

// Active-set tiles of the direct-distance mode, built on its first launch in a begin() window: a window that only runs
// tensor-core or fp64 launches never pays for them.
static int direct_prepare(Ctx* c) {
  if (c->i8d_prepared) return SGP_OK;
  const size_t zd_bytes = static_cast<size_t>(c->m_pad / kTile) * c->kf.n_terms * kTile * c->dpad * sizeof(float);
  const int rc = ctx_scratch(c, c->i8_zd_ws, zd_bytes);
  if (rc != SGP_OK) return rc;
  const double* scale = c->dI8Scale.as<double>();
  SGP_CUDA(c, launch_i8_prep_active_direct(c->i8_zd_ws.as<float>(), c->dZ.as<double>(), c->m, c->m_pad, c->d, c->dpad,
                                           c->kf.n_terms, scale, scale + static_cast<size_t>(kMaxTerms) * c->dpad,
                                           c->dI8Flags.as<int>(), kI8DirectR2Max, c->stream));
  c->launches += 1;
  c->i8d_prepared = true;
  return SGP_OK;
}

// The path of one statistics launch: SGP_PREC_F64 / _F64_STRICT (fp64 DMMA kernel), SGP_PREC_I8 (int8 Gram with
// tensor-core distances: one term, d <= 32) or SGP_PREC_I8_DIRECT (int8 Gram with direct fp32 distances: up to 4 terms,
// n_terms * d <= 72).  AUTO: the int8 kernel inside its measured parity envelope -- accumulate calls (n_call points) of
// >= 32768 points (posterior mean within a few 1e-6 of the all-fp64 kernel from N = 16k up; the limit is the two dropped
// low-order digit products, tools/i8_error_model.py, and does not grow towards small N) and small scaled norms (the gate
// of launch_stats_i8).  Smaller calls stay on the fp64 DMMA kernel (2e-7), which needs < 2 ms at that size.  AUTO
// decides per CALL, on its first chunk, so the chunks of one shard never mix kernels (and only the first chunk pays the
// device->host round trip of the gate).
static int stats_path(Ctx* c, long long n_call, bool first_of_call, int* path) {
  const int i8_mode = c->i8_ok ? SGP_PREC_I8 : c->i8_direct_ok ? SGP_PREC_I8_DIRECT : SGP_PREC_F64;
  *path = c->precision == SGP_PREC_F64_STRICT ? SGP_PREC_F64_STRICT : SGP_PREC_F64;
  if (c->precision == SGP_PREC_I8) {
    if (i8_mode == SGP_PREC_F64)
      return fail(c, SGP_E_BADARG, "SGP_PREC_I8 needs a kernel with 1..4 non-Eye terms and n_terms * d <= 72 "
                                   "(tensor-core distances: exactly one term and d <= 32)");
    *path = i8_mode;
  } else if (c->precision == SGP_PREC_I8_DIRECT) {
    if (!c->i8_direct_ok) return fail(c, SGP_E_BADARG, "SGP_PREC_I8_DIRECT needs a kernel with 1..4 non-Eye terms and n_terms * d <= 72");
    *path = SGP_PREC_I8_DIRECT;
  } else if (c->precision == SGP_PREC_AUTO && n_call >= kAutoI8MinPoints) {
    *path = first_of_call ? i8_mode : c->call_path;
  }
  return SGP_OK;
}

// Records the start of one Gram timing interval (sgp_gram_kernel_time) on the compute stream and returns the event that
// ends it.  The event pool grows on first use only.
static int gram_timer_start(Ctx* c, cudaEvent_t* stop) {
  if (c->gram_events_used == c->gram_events.size()) {
    cudaEvent_t a, b;
    SGP_CUDA(c, cudaEventCreate(&a));
    SGP_CUDA(c, cudaEventCreate(&b));
    c->gram_events.emplace_back(a, b);
  }
  const auto& ev = c->gram_events[c->gram_events_used++];
  *stop = ev.second;
  SGP_CUDA(c, cudaEventRecord(ev.first, c->stream));
  return SGP_OK;
}

// The fp64 DMMA kernel over n device-resident points, then the deterministic slice reduction.
static int launch_stats_f64(Ctx* c, bool strict, const void* dX, int x_is_f32, const double* dy, long long n) {
  const int nt1 = c->m_pad / kTile;
  const int ntiles = nt1 * (nt1 + 1) / 2;
  int n_slices = c->num_sms / ntiles;            // fill the SMs with tiles x point-slices
  if (n_slices < 1) n_slices = 1;
  const long long blocks = (n + 15) / 16;
  if (n_slices > blocks) n_slices = static_cast<int>(blocks);
  int rc = ctx_scratch(c, c->gpart_ws, static_cast<size_t>(n_slices) * c->m_pad * c->m_pad * sizeof(double));
  if (rc == SGP_OK) rc = ctx_scratch(c, c->bpart_ws, static_cast<size_t>(n_slices) * c->m_pad * sizeof(double));
  cudaEvent_t stop = nullptr;
  if (rc == SGP_OK) rc = gram_timer_start(c, &stop);
  if (rc != SGP_OK) return rc;
  GramParams p{};
  p.X = dX; p.y = dy; p.n = n; p.x_is_f32 = x_is_f32;
  p.d = c->d; p.dpad = c->dpad; p.m = c->m; p.m_pad = c->m_pad;
  p.n_terms = c->kf.n_terms;
  std::copy(c->kf.scale, c->kf.scale + kMaxTerms, p.scale);
  p.Zc = c->dZc.as<double>(); p.beta = c->dBeta.as<double>();
  p.Gpart = c->gpart_ws.as<double>(); p.bpart = c->bpart_ws.as<double>();
  p.n_slices = n_slices; p.n_tiles_1d = nt1;
  SGP_CUDA(c, launch_gram_f64(p, strict, c->stream));
  SGP_CUDA(c, cudaEventRecord(stop, c->stream));
  double* G = c->dGb.as<double>();
  SGP_CUDA(c, launch_gram_reduce(G, G + static_cast<size_t>(c->m) * c->m, p.Gpart, p.bpart, n_slices, c->m, c->m_pad,
                                 c->stream));
  c->launches += 2;
  return SGP_OK;
}

// The int8 path (*path: SGP_PREC_I8 or _I8_DIRECT): the point operands, AUTO's magnitude gate (above it *path becomes
// SGP_PREC_F64 and nothing more runs here), the producer and Gram per launch window, the deterministic slice reduction.
static int launch_stats_i8(Ctx* c, int* path, const void* dX, int x_is_f32, const double* dy, long long n,
                           bool first_of_call) {
  const bool direct_mode = *path == SGP_PREC_I8_DIRECT;
  const bool autop = c->precision == SGP_PREC_AUTO, gate = autop && first_of_call;
  const long long n_units = (n + 63) / 64;
  // bytes of one 64-point unit of the point operands: fp16 images (tensor-core distances) or fp32 coordinate tiles
  const size_t x_unit = direct_mode ? static_cast<size_t>(c->kf.n_terms) * 64 * c->dpad * sizeof(float)
                                    : i8_points_scratch_bytes(64, i8_nchunks(c->d));
  int rc = ctx_scratch(c, c->i8_ys_ws, static_cast<size_t>(n_units) * 64 * sizeof(float));
  if (rc == SGP_OK) rc = ctx_scratch(c, c->i8_xt_ws, static_cast<size_t>(n_units) * x_unit);
  if (rc == SGP_OK && direct_mode) rc = direct_prepare(c);
  if (rc != SGP_OK) return rc;
  // the scaled squared norms of EVERY chunk are summed on the device (dI8NormSum[0]: whole begin..finish window,
  // checked against the budget at finish so that an unrepresentative first chunk cannot silently degrade the
  // statistics; dI8NormSum[1]: this call's first chunk, read back here for the kernel choice).  The direct mode sums
  // the WIDEST term's scaled squared norms: they set the size of the kernel values.
  const double* scale = c->dI8Scale.as<double>();
  const double* centre = scale + static_cast<size_t>(kMaxTerms) * c->dpad;
  double* norm_sum = c->dI8NormSum.as<double>();
  double* call_sum = gate ? norm_sum + 1 : nullptr;
  if (gate) SGP_CUDA(c, cudaMemsetAsync(call_sum, 0, sizeof(double), c->stream));
  if (direct_mode)
    SGP_CUDA(c, launch_i8_prep_points_direct(c->i8_xt_ws.as<float>(), c->i8_ys_ws.as<float>(), dX, x_is_f32, dy, n, c->d,
                                             c->dpad, c->kf.n_terms, scale, centre, c->dI8Flags.as<int>(), kI8DirectR2Max,
                                             autop ? norm_sum : nullptr, call_sum, c->stream));
  else
    SGP_CUDA(c, launch_i8_prep_points(c->i8_xt_ws.as<uint8_t>(), c->i8_ys_ws.as<float>(), dX, x_is_f32, dy, n, c->d, scale,
                                      centre, c->dI8Flags.as<int>(), norm_sum, call_sum, c->stream));
  c->launches += 1;
  if (gate) {
    // AUTO's magnitude gate.  The distance contraction accumulates 2 x^.z^ - |x^|^2 - |z^|^2 in fp32 in tensor
    // memory; its rounding (toward zero, measured) scales with those magnitudes: at mean|x^|^2 + mean|z^|^2 ~ 4.4
    // the elements are good to 2.7e-7 rms (parity holds, tests), at ~12 (airfoil: norms up to 40) they are not
    // (posterior mean off by 5e-4).  Large scaled norms also mean tiny kernel values, and the fixed-point digits carry
    // an ABSOLUTE error of 2^-24: on such shards the int8 Gram -- with either distance form -- loses the posterior
    // mean (airfoil-like data: 1.5e-4 to 1.5e-2 against 7e-7 .. 7e-6 of the fp64 kernel).  Above the budget the
    // shard goes to the fp64 DMMA kernel instead.
    double xsum = 0.0;
    SGP_CUDA(c, cudaMemcpyAsync(&xsum, call_sum, sizeof(double), cudaMemcpyDeviceToHost, c->stream));
    SGP_CUDA(c, cudaStreamSynchronize(c->stream));
    if (xsum / static_cast<double>(n) + c->i8_z_norm_mean > kI8NormBudget) {
      *path = SGP_PREC_F64;
      return SGP_OK;
    }
  }
  // the digit planes of a launch window take kI8PlaneBytes per unit and active tile, so a launch covers at most
  // kI8PlaneCapBytes of them; larger launches split into equal windows, all run with the first window's slices: the
  // Gram's (its G partials) and the producer's own (its b partials), a grid that fills the SMs at the variant's occupancy
  const int nt1 = c->m_pad / kTile;
  const long long cap_units = std::max<long long>(1, kI8PlaneCapBytes / (kI8PlaneBytes * nt1));
  const long long n_windows = (n_units + cap_units - 1) / cap_units;
  const long long win_units = (n_units + n_windows - 1) / n_windows;
  const I8Direct direct = direct_mode ? c->i8_direct : I8Direct{};
  const double C = direct_mode ? direct.csum : c->kf.scale[0];
  const uint8_t* zop = direct_mode ? c->i8_zd_ws.as<uint8_t>() : c->dI8Zt.as<uint8_t>();
  const int g_slices = i8_slices(c->m_pad, c->num_sms, win_units);
  int b_slices = 1;
  SGP_CUDA(c, i8_plane_slices(c->m_pad, c->num_sms, win_units, c->d, direct, &b_slices));
  rc = ctx_scratch(c, c->i8_planes_ws, static_cast<size_t>(win_units) * nt1 * kI8PlaneBytes);
  if (rc == SGP_OK) rc = ctx_scratch(c, c->gpart_ws, static_cast<size_t>(g_slices) * c->m_pad * c->m_pad * sizeof(double));
  if (rc == SGP_OK) rc = ctx_scratch(c, c->bpart_ws, static_cast<size_t>(b_slices) * c->m_pad * sizeof(double));
  cudaEvent_t stop = nullptr;
  if (rc == SGP_OK) rc = gram_timer_start(c, &stop);
  if (rc != SGP_OK) return rc;
  uint8_t* planes = c->i8_planes_ws.as<uint8_t>();
  double* Gpart = c->gpart_ws.as<double>();
  double* bpart = c->bpart_ws.as<double>();
  // per window: digit planes + b partials, then the Gram over them; the first window stores the slice partials,
  // later ones add to them, and one deterministic slice reduction follows
  for (long long w = 0; w < n_windows; ++w) {
    const long long u0 = w * win_units;
    const long long nu = std::min(win_units, n_units - u0);
    SGP_CUDA(c, launch_i8_planes(c->i8_xt_ws.as<uint8_t>() + static_cast<size_t>(u0) * x_unit,
                                 c->i8_ys_ws.as<float>() + static_cast<size_t>(u0) * 64, zop, nu, c->d, c->m_pad, b_slices,
                                 direct, C, w > 0, planes, bpart, w == 0 ? c->dbgT.as<float>() : nullptr,
                                 w == 0 ? c->dbgW.as<uint32_t>() : nullptr, c->stream));
    SGP_CUDA(c, launch_gram_i8(planes, nu, c->m_pad, g_slices, C, w > 0, Gpart, c->stream));
    c->launches += 2;
  }
  SGP_CUDA(c, cudaEventRecord(stop, c->stream));
  // partial tiles at the mirror position: upper block triangle
  double* G = c->dGb.as<double>();
  SGP_CUDA(c, launch_gram_reduce_upper(G, G + static_cast<size_t>(c->m) * c->m, Gpart, bpart, g_slices, b_slices, c->m,
                                       c->m_pad, c->stream));
  c->launches += 1;
  return SGP_OK;
}

// The statistics of n device-resident points (n_call: the whole accumulate call's) on the path stats_path picks.
static int launch_stats(Ctx* c, const void* dX, int x_is_f32, const double* dy, long long n, long long n_call,
                        bool first_of_call) {
  if (n <= 0) return SGP_OK;
  const auto int8 = [](int p) { return p == SGP_PREC_I8 || p == SGP_PREC_I8_DIRECT; };
  int path = SGP_PREC_F64;
  int rc = stats_path(c, n_call, first_of_call, &path);
  if (rc == SGP_OK && int8(path)) rc = launch_stats_i8(c, &path, dX, x_is_f32, dy, n, first_of_call);
  if (rc == SGP_OK && !int8(path)) rc = launch_stats_f64(c, path == SGP_PREC_F64_STRICT, dX, x_is_f32, dy, n);
  if (rc != SGP_OK) return rc;
  if (first_of_call) c->call_path = path;
  c->last_path = path;
  if (int8(path)) {
    c->i8_points += n;
    c->i8_flag_mask |= (path == SGP_PREC_I8) ? 1 : 4;
  }
  return SGP_OK;
}

// In-place sum of `count` elements of device memory over the context's communicator, on its stream (a no-op without a
// communicator of more than one rank).  For the sharded K-means: its few collectives are small and synchronous.
int comm_sum(Ctx* c, void* buf, size_t count, ncclDataType_t type) {
  if (!c->comm || c->nranks <= 1 || count == 0) return SGP_OK;
  const ncclResult_t r = nccl().AllReduce(buf, buf, count, type, ncclSum, c->comm, c->stream);
  if (r != ncclSuccess) return fail(c, SGP_E_NCCL, std::string("ncclAllReduce: ") + nccl().GetErrorString(r));
  c->launches += 1;
  return SGP_OK;
}
}  // namespace sgp

using namespace sgp;

extern "C" {

int sgp_version(void) { return 100; }

int sgp_ctx_create(sgp_ctx** out, int device) {
  if (!out) return fail(nullptr, SGP_E_BADARG, "out == NULL");
  *out = nullptr;
  int ndev = 0;
  cudaError_t e = cudaGetDeviceCount(&ndev);
  if (e != cudaSuccess || ndev == 0)
    return fail(nullptr, SGP_E_CUDA, std::string("no CUDA device: ") + cudaGetErrorString(e) +
                                         " (this library has no CPU fallback)");
  if (device < 0 || device >= ndev) return fail(nullptr, SGP_E_BADARG, "device index out of range");
  Ctx* c = new (std::nothrow) Ctx();
  if (!c) return fail(nullptr, SGP_E_NOMEM, "out of host memory");
  c->device = device;
  auto bail = [&](int code, const std::string& m) { std::string mm = m; delete c; return fail(nullptr, code, mm); };
  if ((e = cudaSetDevice(device)) != cudaSuccess) return bail(SGP_E_CUDA, cudaGetErrorString(e));
  cudaDeviceProp prop;
  if ((e = cudaGetDeviceProperties(&prop, device)) != cudaSuccess) return bail(SGP_E_CUDA, cudaGetErrorString(e));
  if (prop.major != 9 || prop.minor != 0)
    return bail(SGP_E_CUDA, "this library is built for sm_90a (H100) only; device is sm_" +
                                std::to_string(prop.major) + std::to_string(prop.minor));
  c->num_sms = prop.multiProcessorCount;
  if ((e = cudaStreamCreateWithFlags(&c->stream, cudaStreamNonBlocking)) != cudaSuccess ||
      (e = cudaStreamCreateWithFlags(&c->copy_stream, cudaStreamNonBlocking)) != cudaSuccess)
    return bail(SGP_E_CUDA, cudaGetErrorString(e));
  for (int i = 0; i < 2; ++i) {
    cudaEventCreateWithFlags(&c->stage_free[i], cudaEventDisableTiming);
    cudaEventCreateWithFlags(&c->stage_ready[i], cudaEventDisableTiming);
    cudaEventCreateWithFlags(&c->out_ready[i], cudaEventDisableTiming);
    cudaEventCreateWithFlags(&c->out_free[i], cudaEventDisableTiming);
  }
  if ((e = cudaStreamCreateWithFlags(&c->tail_stream, cudaStreamNonBlocking)) != cudaSuccess ||
      (e = cudaEventCreateWithFlags(&c->tail_fork, cudaEventDisableTiming)) != cudaSuccess ||
      (e = cudaEventCreateWithFlags(&c->tail_join, cudaEventDisableTiming)) != cudaSuccess)
    return bail(SGP_E_CUDA, cudaGetErrorString(e));
  if (cusolverDnCreate(&c->solver) != CUSOLVER_STATUS_SUCCESS) return bail(SGP_E_CUDA, "cusolverDnCreate failed");
  if (cusolverDnCreate(&c->solver2) != CUSOLVER_STATUS_SUCCESS) return bail(SGP_E_CUDA, "cusolverDnCreate failed");
  if (cublasCreate(&c->blas) != CUBLAS_STATUS_SUCCESS) return bail(SGP_E_CUDA, "cublasCreate failed");
  *out = reinterpret_cast<sgp_ctx*>(c);
  return SGP_OK;
}

int sgp_ctx_destroy(sgp_ctx* h) {
  Ctx* c = reinterpret_cast<Ctx*>(h);
  if (!c) return SGP_OK;
  cudaSetDevice(c->device);
  cudaDeviceSynchronize();
  for (auto& e : c->gram_events) { cudaEventDestroy(e.first); cudaEventDestroy(e.second); }
  for (auto& e : c->user_events) if (e) cudaEventDestroy(e);
  for (int i = 0; i < 2; ++i) {
    if (c->stage_free[i]) cudaEventDestroy(c->stage_free[i]);
    if (c->stage_ready[i]) cudaEventDestroy(c->stage_ready[i]);
    if (c->out_ready[i]) cudaEventDestroy(c->out_ready[i]);
    if (c->out_free[i]) cudaEventDestroy(c->out_free[i]);
  }
  if (c->comm && nccl().ok) nccl().CommDestroy(c->comm);
  if (c->tail_fork) cudaEventDestroy(c->tail_fork);
  if (c->tail_join) cudaEventDestroy(c->tail_join);
  if (c->tail_stream) cudaStreamDestroy(c->tail_stream);
  if (c->solver) cusolverDnDestroy(c->solver);
  if (c->solver2) cusolverDnDestroy(c->solver2);
  if (c->blas) cublasDestroy(c->blas);
  if (c->stream) cudaStreamDestroy(c->stream);
  if (c->copy_stream) cudaStreamDestroy(c->copy_stream);
  delete c;                                         // the device buffers free themselves
  return SGP_OK;
}

const char* sgp_last_error(const sgp_ctx* h) {
  const Ctx* c = reinterpret_cast<const Ctx*>(h);
  return c ? c->err.c_str() : g_create_err.c_str();
}

int sgp_set_precision(sgp_ctx* h, int mode) {
  Ctx* c = reinterpret_cast<Ctx*>(h);
  if (!c) return SGP_E_BADARG;
  if (mode < SGP_PREC_F64 || mode > SGP_PREC_I8_DIRECT) return fail(c, SGP_E_BADARG, "unknown precision mode");
  c->precision = mode;
  return SGP_OK;
}

int sgp_comm_unique_id(void* out128) {
  if (!out128) return SGP_E_BADARG;
  static_assert(sizeof(ncclUniqueId) <= SGP_UNIQUE_ID_BYTES, "ncclUniqueId does not fit");
  if (!nccl().ok) return fail(nullptr, SGP_E_NCCL, "libnccl.so.2 could not be loaded");
  ncclUniqueId id;
  if (nccl().GetUniqueId(&id) != ncclSuccess) return fail(nullptr, SGP_E_NCCL, "ncclGetUniqueId failed");
  std::memset(out128, 0, SGP_UNIQUE_ID_BYTES);
  std::memcpy(out128, &id, sizeof(id));
  return SGP_OK;
}

int sgp_comm_init(sgp_ctx* h, const void* id128, int rank, int nranks) {
  Ctx* c = reinterpret_cast<Ctx*>(h);
  if (!c || !id128 || nranks < 1 || rank < 0 || rank >= nranks) return fail(c, SGP_E_BADARG, "bad comm arguments");
  // a second communicator would orphan the first, and its peers with it: the context keeps the one it has
  if (c->comm) return fail(c, SGP_E_STATE, "sgp_comm_init: the context already has a communicator");
  if (!nccl().ok) return fail(c, SGP_E_NCCL, "libnccl.so.2 could not be loaded");
  SGP_CUDA(c, cudaSetDevice(c->device));
  ncclUniqueId id;
  std::memcpy(&id, id128, sizeof(id));
  ncclComm_t comm = nullptr;
  ncclResult_t r = nccl().CommInitRank(&comm, nranks, id, rank);
  if (r != ncclSuccess) return fail(c, SGP_E_NCCL, std::string("ncclCommInitRank: ") + nccl().GetErrorString(r));
  c->comm = comm;                                   // only a communicator that was made: sgp_ctx_destroy destroys it
  c->rank = rank; c->nranks = nranks;
  return SGP_OK;
}


int sgp_stats_begin(sgp_ctx* h, const sgp_kernel_desc* k, const double* Z, int32_t m, int32_t d) {
  Ctx* c = reinterpret_cast<Ctx*>(h);
  if (!c) return SGP_E_BADARG;
  c->begun = c->finished = c->range_failed = c->has_magic = c->magic_packed = false;   // a failed begin leaves no window
  if (!k || !Z || m <= 0 || d <= 0 || k->n_terms <= 0 || !k->terms)
    return fail(c, SGP_E_BADARG, "sgp_stats_begin: null or empty argument");
  SGP_CUDA(c, cudaSetDevice(c->device));
  KernelFlat kf;
  std::vector<double> beta;
  const int dpad = (d + 3) & ~3;
  int rc = flatten_kernel(c, k, d, dpad, kf, beta, nullptr);
  if (rc != SGP_OK) return rc;
  c->m = m; c->d = d; c->dpad = dpad; c->m_pad = (m + kTile - 1) / kTile * kTile; c->kf = kf;
  // int8 Gram: direct distances for 1..4 non-Eye terms with n_terms * dpad <= 72 (shared memory); tensor-core distances
  // for one term and d <= 32 (two 64-column K chunks)
  c->i8_direct_ok = kf.n_terms >= 1 && kf.n_terms * dpad <= 72;
  c->i8_ok = kf.n_terms == 1 && d <= 32;
  I8Direct& dm = c->i8_direct;     // the direct mode's term weights C_t / sum C; sum C is its fixed-point scale
  dm = I8Direct{1, kf.n_terms, dpad};
  for (int t = 0; t < kf.n_terms; ++t) dm.csum += kf.scale[t];
  for (int t = 0; t < kf.n_terms; ++t) dm.w[t] = static_cast<float>(kf.scale[t] / dm.csum);
  // the device buffers only grow: cudaMalloc/cudaFree are synchronising and cost milliseconds -- more than the whole
  // statistics pass on the GPU
  const size_t mm = static_cast<size_t>(m) * m;
  const size_t z_bytes = static_cast<size_t>(std::max(kf.n_terms, 1)) * c->m_pad * dpad * 8;
  const size_t dim_bytes = static_cast<size_t>(kMaxTerms + 1) * dpad * 8;
  const std::pair<DevScratch*, size_t> bufs[] = {
      {&c->dZ, static_cast<size_t>(m) * d * 8}, {&c->dZs, z_bytes}, {&c->dZc, z_bytes}, {&c->dBeta, dim_bytes},
      {&c->dGb, (mm + m + 1) * 8}, {&c->dMagicVec, static_cast<size_t>(m) * 8}, {&c->dMagicMat, mm * 8},
      {&c->dI8Flags, 3 * sizeof(int)}, {&c->dI8NormSum, 2 * sizeof(double)}, {&c->dI8Scale, dim_bytes},
      {&c->dI8Zt, c->i8_ok ? i8_active_scratch_bytes(c->m_pad, i8_nchunks(d)) : 0}};   // 0: not needed
  for (const auto& [buf, bytes] : bufs)
    if (bytes > 0 && (rc = ctx_scratch(c, *buf, bytes)) != SGP_OK) return rc;
  double* dZ = c->dZ.as<double>();
  double* dBeta = c->dBeta.as<double>();
  double* dScale = c->dI8Scale.as<double>();
  int* dFlags = c->dI8Flags.as<int>();
  SGP_CUDA(c, cudaMemcpyAsync(dZ, Z, static_cast<size_t>(m) * d * 8, cudaMemcpyHostToDevice, c->stream));
  std::vector<double> sc;                          // live until the synchronisation at the end of this function
  beta.resize(static_cast<size_t>(kMaxTerms + 1) * dpad, 0.0);
  c->i8_z_norm_mean = stats_scales(Z, m, d, dpad, kf.n_terms, beta, c->i8_direct_ok, sc,
                                   beta.data() + static_cast<size_t>(kMaxTerms) * dpad);
  SGP_CUDA(c, cudaMemcpyAsync(dBeta, beta.data(), beta.size() * 8, cudaMemcpyHostToDevice, c->stream));
  SGP_CUDA(c, cudaMemsetAsync(c->dGb.p, 0, (mm + m + 1) * 8, c->stream));      // [G ; b ; status] -- one all-reduce
  SGP_CUDA(c, cudaMemcpyAsync(dScale, sc.data(), sc.size() * 8, cudaMemcpyHostToDevice, c->stream));
  for (int t = 0; t < kf.n_terms; ++t) {
    const size_t off = static_cast<size_t>(t) * c->m_pad * dpad;
    SGP_CUDA(c, launch_scale_rows(c->dZs.as<double>() + off, c->dZc.as<double>() + off, dZ,
                                  dBeta + static_cast<size_t>(t) * dpad, dBeta + static_cast<size_t>(kMaxTerms) * dpad, m,
                                  c->m_pad, d, dpad, c->stream));
    c->launches += 1;
  }
  SGP_CUDA(c, cudaMemsetAsync(dFlags, 0, 3 * sizeof(int), c->stream));
  SGP_CUDA(c, cudaMemsetAsync(c->dI8NormSum.p, 0, 2 * sizeof(double), c->stream));
  if (c->i8_ok) {
    // the tensor-core operand images are built here, the direct mode's active-set tiles on its first launch
    // the active set's range status goes to its own word; the window's status starts from it
    SGP_CUDA(c, launch_i8_prep_active(c->dI8Zt.as<uint8_t>(), dZ, m, c->m_pad, d, dScale,
                                      dScale + static_cast<size_t>(kMaxTerms) * dpad, dFlags + 1, c->stream));
    SGP_CUDA(c, cudaMemcpyAsync(dFlags, dFlags + 1, sizeof(int), cudaMemcpyDeviceToDevice, c->stream));
    c->launches += 1;
  }
  c->i8d_prepared = false;
  SGP_CUDA(c, cudaStreamSynchronize(c->stream));   // Z / beta are host temporaries of the caller
  c->gram_events_used = 0;
  c->i8_points = 0;
  c->i8_flag_mask = 0;
  c->begun = true;
  return SGP_OK;
}

int sgp_stats_accumulate_device(sgp_ctx* h, const void* dX, int32_t x_is_f32, const double* dy, int64_t n) {
  Ctx* c = reinterpret_cast<Ctx*>(h);
  if (!c) return SGP_E_BADARG;
  if (!c->begun || c->finished) return fail(c, SGP_E_STATE, "sgp_stats_begin should have been called first");
  if (n < 0 || (n > 0 && (!dX || !dy))) return fail(c, SGP_E_BADARG, "null shard");
  SGP_CUDA(c, cudaSetDevice(c->device));
  if (c->kf.n_terms == 0) return SGP_OK;   // only Eye terms: the cross kernel is identically zero
  return launch_stats(c, dX, x_is_f32, dy, n, n, true);
}

int sgp_stats_accumulate(sgp_ctx* h, const void* X, int32_t x_is_f32, const double* y, int64_t n) {
  Ctx* c = reinterpret_cast<Ctx*>(h);
  if (!c) return SGP_E_BADARG;
  if (!c->begun || c->finished) return fail(c, SGP_E_STATE, "sgp_stats_begin should have been called first");
  if (n < 0 || (n > 0 && (!X || !y))) return fail(c, SGP_E_BADARG, "null shard");
  if (n == 0 || c->kf.n_terms == 0) return SGP_OK;
  SGP_CUDA(c, cudaSetDevice(c->device));
  const size_t esz = x_is_f32 ? 4 : 8;
  const size_t row = static_cast<size_t>(c->d) * esz;
  // chunk so that copy (PCIe) and compute overlap: ~16 MB of X per chunk (the first chunk's copy is the exposed part:
  // 0.3 ms at 55 GB/s), at least 64k points
  long long chunk = static_cast<long long>((16u << 20) / row);
  if (chunk < 65536) chunk = 65536;
  {                                           // equal chunks (multiples of 64 points) instead of a short tail chunk
    const long long nchunks = (n + chunk - 1) / chunk;
    chunk = ((n + nchunks - 1) / nchunks + 63) / 64 * 64;
  }
  if (chunk > n) chunk = n;
  // The first chunk's copy is the only one the kernels cannot hide: make it a quarter of the others
  long long first = chunk;
  if (n > chunk) {
    first = (chunk / 4 + 63) / 64 * 64;
    if (first < 65536) first = 65536;
    if (first > chunk) first = chunk;
    const long long rest = n - first;
    const long long nchunks = (rest + chunk - 1) / chunk;
    chunk = ((rest + nchunks - 1) / nchunks + 63) / 64 * 64;
    if (chunk < first) chunk = first;
  }
  // the caller may reuse / free X, y as soon as we return
  return stage_rows(c, X, y, n, row, first, chunk, [&](const void* dX, const double* dy, long long p0, long long cn) {
    return launch_stats(c, dX, x_is_f32, dy, cn, n, p0 == 0);
  });
}

int sgp_stats_finish(sgp_ctx* h, double* G_out, double* b_out) {
  Ctx* c = reinterpret_cast<Ctx*>(h);
  if (!c) return SGP_E_BADARG;
  if (!c->begun) return fail(c, SGP_E_STATE, "sgp_stats_begin should have been called first");
  SGP_CUDA(c, cudaSetDevice(c->device));
  const size_t mm = static_cast<size_t>(c->m) * c->m;
  double* G = c->dGb.as<double>();
  double status = 0.0;
  if (!c->finished) {
    // The rank-local status of the int8 path (operand range exceeded; AUTO's magnitude budget exceeded over the
    // WHOLE window, not just the first chunk the kernel choice looked at) rides in the last slot of the all-reduced
    // buffer: every rank sees the same sum and takes the same return decision AFTER the collective -- a rank that
    // bailed out before it would leave its peers blocked in ncclAllReduce.
    const int mask = c->i8_flag_mask;
    const bool budget = mask != 0 && c->precision == SGP_PREC_AUTO;
    const double limit = (kI8NormBudget - c->i8_z_norm_mean) * static_cast<double>(c->i8_points) * 1.25;
    SGP_CUDA(c, launch_status_to_double(G + mm + c->m, mask ? c->dI8Flags.as<int>() : nullptr, mask,
                                        budget ? c->dI8NormSum.as<double>() : nullptr, limit, c->stream));
    c->launches += 1;
    if (c->comm && c->nranks > 1) {
      // PGPH:31-35 combOp: one all-reduce of the packed [G;b;status] over NVLink
      ncclResult_t r = nccl().AllReduce(G, G, mm + c->m + 1, ncclDouble, ncclSum, c->comm, c->stream);
      if (r != ncclSuccess) return fail(c, SGP_E_NCCL, std::string("ncclAllReduce: ") + nccl().GetErrorString(r));
      c->launches += 1;
    }
    SGP_CUDA(c, cudaMemcpyAsync(&status, G + mm + c->m, sizeof(double), cudaMemcpyDeviceToHost, c->stream));
  }
  const bool first = !c->finished;
  c->finished = true;
  if (G_out) SGP_CUDA(c, cudaMemcpyAsync(G_out, G, mm * 8, cudaMemcpyDeviceToHost, c->stream));
  if (b_out)
    SGP_CUDA(c, cudaMemcpyAsync(b_out, G + mm, static_cast<size_t>(c->m) * 8, cudaMemcpyDeviceToHost, c->stream));
  SGP_CUDA(c, cudaStreamSynchronize(c->stream));
  if (first) c->range_failed = status != 0.0;      // the window keeps its status: a repeated finish reports it again
  if (c->range_failed)
    return fail(c, SGP_E_RANGE, "the int8 path cannot represent this shard on some rank (scaled squared norms outside the "
                                "tensor-core operand range, scaled squared norms above AUTO's magnitude budget for tensor-core "
                                "distances, or above the fp32 direct-distance limit); rerun the statistics with "
                                "sgp_set_precision(SGP_PREC_I8_DIRECT) or sgp_set_precision(SGP_PREC_F64)");
  return SGP_OK;
}

int sgp_sync(sgp_ctx* h) {
  Ctx* c = reinterpret_cast<Ctx*>(h);
  if (!c) return SGP_E_BADARG;
  SGP_CUDA(c, cudaSetDevice(c->device));
  SGP_CUDA(c, cudaStreamSynchronize(c->copy_stream));
  SGP_CUDA(c, cudaStreamSynchronize(c->stream));
  return SGP_OK;
}

int sgp_magic(sgp_ctx* h, const double* G_in, const double* b_in, double* magic_vector, double* magic_matrix) {
  Ctx* c = reinterpret_cast<Ctx*>(h);
  if (!c) return SGP_E_BADARG;
  if (!c->begun) return fail(c, SGP_E_STATE, "sgp_stats_begin should have been called first");
  if ((G_in == nullptr) != (b_in == nullptr)) return fail(c, SGP_E_BADARG, "G_in and b_in must be given together");
  if (!G_in && !c->finished) return fail(c, SGP_E_STATE, "sgp_stats_finish should have been called first");
  if (!G_in && c->range_failed)
    return fail(c, SGP_E_STATE, "the statistics of this window could not be represented (sgp_stats_finish returned "
                                "SGP_E_RANGE): rerun them, or pass G_in and b_in");
  // the installed pair is gone from here on: only a tail that succeeds installs one again
  c->has_magic = c->magic_packed = false;
  SGP_CUDA(c, cudaSetDevice(c->device));
  const size_t mm = static_cast<size_t>(c->m) * c->m;
  if (G_in) {
    SGP_CUDA(c, cudaMemcpyAsync(c->dGb.p, G_in, mm * 8, cudaMemcpyHostToDevice, c->stream));
    SGP_CUDA(c, cudaMemcpyAsync(c->dGb.as<double>() + mm, b_in, static_cast<size_t>(c->m) * 8, cudaMemcpyHostToDevice, c->stream));
    c->finished = true;
    c->range_failed = false;
  }
  return run_tail(c, magic_vector, magic_matrix);
}

int sgp_set_magic(sgp_ctx* h, const double* v, const double* M) {
  Ctx* c = reinterpret_cast<Ctx*>(h);
  if (!c) return SGP_E_BADARG;
  if (!c->begun) return fail(c, SGP_E_STATE, "sgp_stats_begin should have been called first");
  if (!v || !M) return fail(c, SGP_E_BADARG, "sgp_set_magic: null argument");
  SGP_CUDA(c, cudaSetDevice(c->device));
  const size_t mm = static_cast<size_t>(c->m) * c->m;
  SGP_CUDA(c, cudaMemcpyAsync(c->dMagicVec.p, v, static_cast<size_t>(c->m) * 8, cudaMemcpyHostToDevice, c->stream));
  SGP_CUDA(c, cudaMemcpyAsync(c->dMagicMat.p, M, mm * 8, cudaMemcpyHostToDevice, c->stream));
  SGP_CUDA(c, cudaStreamSynchronize(c->stream));          // the caller may reuse v, M as soon as we return
  c->has_magic = true;
  c->magic_packed = false;
  return SGP_OK;
}

namespace {
// The host rows stream in through the statistics path's double-buffered staging; each window's mean / variance /
// probability go to one of two device output buffers and are copied out (copy stream) once the NEXT window is queued, so
// that the copies in both directions overlap the kernels.  The mean is always computed (the probability reads it); it is
// copied out only where mean_out is given.  p_out: the averaged probabilities with the n_nodes-node rule, or nullptr.
int predict_host(Ctx* c, const double* X, long long n, int n_nodes, double* mean_out, double* var_out, double* p_out) {
  SGP_CUDA(c, cudaSetDevice(c->device));
  // staged chunks of ~32 MB of X (at least 4096 points), never more than one kernel window
  const size_t row = static_cast<size_t>(c->d) * sizeof(double);
  const long long win = predict_window_points(c->m_pad);
  long long chunk = std::max<long long>(4096, static_cast<long long>((size_t(32) << 20) / row));
  chunk = std::min(std::min(chunk, win), n);
  int rc = predict_prepare(c, var_out != nullptr || p_out != nullptr, p_out ? n_nodes : 0);
  if (rc == SGP_OK) rc = ctx_scratch(c, c->predict_out_ws, 6 * static_cast<size_t>(chunk) * sizeof(double));
  if (rc != SGP_OK) return rc;
  double* out = c->predict_out_ws.as<double>();      // [2][mean (chunk) | var (chunk) | p (chunk)]
  auto copy_out = [&](int b, long long p0, long long cn) -> int {
    const double* dm = out + 3 * static_cast<size_t>(chunk) * b;
    SGP_CUDA(c, cudaStreamWaitEvent(c->copy_stream, c->out_ready[b], 0));
    if (mean_out)
      SGP_CUDA(c, cudaMemcpyAsync(mean_out + p0, dm, static_cast<size_t>(cn) * 8, cudaMemcpyDeviceToHost,
                                  c->copy_stream));
    if (var_out)
      SGP_CUDA(c, cudaMemcpyAsync(var_out + p0, dm + chunk, static_cast<size_t>(cn) * 8, cudaMemcpyDeviceToHost,
                                  c->copy_stream));
    if (p_out)
      SGP_CUDA(c, cudaMemcpyAsync(p_out + p0, dm + 2 * chunk, static_cast<size_t>(cn) * 8, cudaMemcpyDeviceToHost,
                                  c->copy_stream));
    SGP_CUDA(c, cudaEventRecord(c->out_free[b], c->copy_stream));
    return SGP_OK;
  };
  long long windows = 0, pending_p0 = 0, pending_n = 0;
  rc = stage_rows(c, X, nullptr, n, row, chunk, chunk,
                  [&](const void* dX, const double*, long long p0, long long cn) -> int {
                    const int b = static_cast<int>(windows & 1);
                    double* dm = out + 3 * static_cast<size_t>(chunk) * b;
                    SGP_CUDA(c, cudaStreamWaitEvent(c->stream, c->out_free[b], 0));
                    int r = predict_window(c, dX, 0, cn, dm, var_out ? dm + chunk : nullptr,
                                           p_out ? dm + 2 * chunk : nullptr);
                    if (r != SGP_OK) return r;
                    SGP_CUDA(c, cudaEventRecord(c->out_ready[b], c->stream));
                    if (windows > 0 && (r = copy_out(b ^ 1, pending_p0, pending_n)) != SGP_OK) return r;
                    ++windows;
                    pending_p0 = p0;
                    pending_n = cn;
                    return SGP_OK;
                  });
  if (rc == SGP_OK) rc = copy_out(static_cast<int>((windows - 1) & 1), pending_p0, pending_n);
  if (rc != SGP_OK) return rc;
  SGP_CUDA(c, cudaStreamSynchronize(c->copy_stream));
  return SGP_OK;
}

// The device entries' shared body: windows of device-resident points, outputs written in place (dMean may be nullptr
// with dP: the mean then lands in the workspace).
int predict_device(Ctx* c, const void* dX, int x_is_f32, long long n, int n_nodes, double* dMean, double* dVar,
                   double* dP) {
  SGP_CUDA(c, cudaSetDevice(c->device));
  int rc = predict_prepare(c, dVar != nullptr || dP != nullptr, dP ? n_nodes : 0);
  if (rc != SGP_OK) return rc;
  const long long win = predict_window_points(c->m_pad);
  const size_t row = static_cast<size_t>(c->d) * (x_is_f32 ? sizeof(float) : sizeof(double));
  for (long long p0 = 0; p0 < n; p0 += win) {
    const long long cn = (n - p0 < win) ? (n - p0) : win;
    rc = predict_window(c, static_cast<const char*>(dX) + static_cast<size_t>(p0) * row, x_is_f32, cn,
                        dMean ? dMean + p0 : nullptr, dVar ? dVar + p0 : nullptr, dP ? dP + p0 : nullptr);
    if (rc != SGP_OK) return rc;
  }
  return SGP_OK;
}

int check_nodes(Ctx* c, int32_t n_nodes) {
  if (n_nodes < 1 || n_nodes > kMaxHermiteNodes)
    return fail(c, SGP_E_BADARG, "n_nodes must be in [1, " + std::to_string(kMaxHermiteNodes) + "]");
  return SGP_OK;
}
}  // namespace

int sgp_predict(sgp_ctx* h, const double* X, int64_t n, double* mean_out, double* var_out) {
  Ctx* c = reinterpret_cast<Ctx*>(h);
  if (!c) return SGP_E_BADARG;
  if (!c->has_magic) return fail(c, SGP_E_STATE, "sgp_magic should have been called first");
  if (n < 0 || (n > 0 && (!X || !mean_out))) return fail(c, SGP_E_BADARG, "null argument");
  if (n == 0) return SGP_OK;
  return predict_host(c, X, n, 0, mean_out, var_out, nullptr);
}

int sgp_predict_device(sgp_ctx* h, const void* dX, int32_t x_is_f32, int64_t n, double* dMean, double* dVar) {
  Ctx* c = reinterpret_cast<Ctx*>(h);
  if (!c) return SGP_E_BADARG;
  if (!c->has_magic) return fail(c, SGP_E_STATE, "sgp_magic should have been called first");
  if (n < 0 || (n > 0 && (!dX || !dMean))) return fail(c, SGP_E_BADARG, "null argument");
  if (n == 0) return SGP_OK;
  return predict_device(c, dX, x_is_f32, n, 0, dMean, dVar, nullptr);
}

int sgp_predict_probability(sgp_ctx* h, const double* X, int64_t n, int32_t n_nodes, double* p_out, double* mean_out,
                            double* var_out) {
  Ctx* c = reinterpret_cast<Ctx*>(h);
  if (!c) return SGP_E_BADARG;
  if (!c->has_magic) return fail(c, SGP_E_STATE, "sgp_magic should have been called first");
  int rc = check_nodes(c, n_nodes);
  if (rc != SGP_OK) return rc;
  if (n < 0 || (n > 0 && (!X || !p_out))) return fail(c, SGP_E_BADARG, "null argument");
  if (n == 0) return SGP_OK;
  return predict_host(c, X, n, n_nodes, mean_out, var_out, p_out);
}

int sgp_predict_probability_device(sgp_ctx* h, const void* dX, int32_t x_is_f32, int64_t n, int32_t n_nodes, double* dP,
                                   double* dMean, double* dVar) {
  Ctx* c = reinterpret_cast<Ctx*>(h);
  if (!c) return SGP_E_BADARG;
  if (!c->has_magic) return fail(c, SGP_E_STATE, "sgp_magic should have been called first");
  int rc = check_nodes(c, n_nodes);
  if (rc != SGP_OK) return rc;
  if (n < 0 || (n > 0 && (!dX || !dP))) return fail(c, SGP_E_BADARG, "null argument");
  if (n == 0) return SGP_OK;
  SGP_CUDA(c, cudaSetDevice(c->device));
  const char* entry = "sgp_predict_probability_device";
  rc = device_ptr_ok(c, dX, entry, "X");
  if (rc == SGP_OK) rc = device_ptr_ok(c, dP, entry, "p_out");
  if (rc == SGP_OK && dMean) rc = device_ptr_ok(c, dMean, entry, "mean_out");
  if (rc == SGP_OK && dVar) rc = device_ptr_ok(c, dVar, entry, "var_out");
  if (rc != SGP_OK) return rc;
  return predict_device(c, dX, x_is_f32, n, n_nodes, dMean, dVar, dP);
}

int sgp_gauss_hermite_rule(int32_t n, double* nodes, double* weights) {
  if (!gauss_hermite_rule(n, nodes, weights))
    return fail(nullptr, SGP_E_BADARG, "sgp_gauss_hermite_rule: n must be in [1, " + std::to_string(kMaxHermiteNodes) +
                                           "] and the outputs non-null");
  return SGP_OK;
}

int64_t sgp_launch_count(const sgp_ctx* h) {
  const Ctx* c = reinterpret_cast<const Ctx*>(h);
  return c ? c->launches : 0;
}

int sgp_gram_kernel_time(sgp_ctx* h, double* total_ms, int64_t* launches) {
  Ctx* c = reinterpret_cast<Ctx*>(h);
  if (!c) return SGP_E_BADARG;
  SGP_CUDA(c, cudaSetDevice(c->device));
  SGP_CUDA(c, cudaStreamSynchronize(c->stream));
  double tot = 0.0;
  for (size_t i = 0; i < c->gram_events_used; ++i) {
    float ms = 0.f;
    SGP_CUDA(c, cudaEventElapsedTime(&ms, c->gram_events[i].first, c->gram_events[i].second));
    tot += ms;
  }
  if (total_ms) *total_ms = tot;
  if (launches) *launches = static_cast<int64_t>(c->gram_events_used);
  return SGP_OK;
}

namespace {
// Drops the context's experts and sizes its expert buffers for E experts of n points in total, with f = zeros
// (GPCls:54).  The caller fills X, y and off, then sets ex.E: the experts count as uploaded only from then on.
int experts_alloc(Ctx* c, long long E, long long n, int d, int n_max) {
  ExpertSet& ex = c->ex;
  ex = ExpertSet{};
  int rc = ctx_scratch(c, c->ex_X, static_cast<size_t>(n) * d * 8);
  if (rc == SGP_OK) rc = ctx_scratch(c, c->ex_y, static_cast<size_t>(n) * 8);
  if (rc == SGP_OK) rc = ctx_scratch(c, c->ex_off, static_cast<size_t>(E + 1) * 8);
  if (rc == SGP_OK) rc = ctx_scratch(c, c->ex_f.buf, static_cast<size_t>(n) * 8);
  if (rc != SGP_OK) return rc;
  ex.X = c->ex_X.as<double>(); ex.y = c->ex_y.as<double>(); ex.off = c->ex_off.as<long long>(); ex.f = c->ex_f.buf.as<double>();
  SGP_CUDA(c, cudaMemsetAsync(ex.f, 0, static_cast<size_t>(n) * 8, c->stream));
  ex.n = n; ex.d = d; ex.n_max = n_max;
  c->ex_grouped = false;
  c->ex_f.slots = 1;                                      // the binary objectives' modes: one slot, zero
  for (ModeStore* m : {&c->ex_fc, &c->ex_fm, &c->ex_ffm}) m->slots = 0;   // the slot stores restart at zero on next use
  c->fold_first.clear();
  c->fold_nmax.clear();
  c->fold_row0.clear();
  return SGP_OK;
}

// Chunks of ~32 MB of rows (at least 64k points) for the grouped uploads' staging
long long group_chunk(long long n, size_t row) {
  long long chunk = static_cast<long long>((32u << 20) / row);
  if (chunk < 65536) chunk = 65536;
  return chunk > n ? n : chunk;
}
}  // namespace

int sgp_experts_upload(sgp_ctx* h, const double* X, const double* y, const int64_t* offsets, int64_t E, int32_t d) {
  Ctx* c = reinterpret_cast<Ctx*>(h);
  if (!c) return SGP_E_BADARG;
  if (!X || !y || !offsets || E <= 0 || d <= 0) return fail(c, SGP_E_BADARG, "sgp_experts_upload: null or empty argument");
  SGP_CUDA(c, cudaSetDevice(c->device));
  const long long n = offsets[E];
  int nmax = 0;
  for (int64_t e = 0; e < E; ++e) {
    const long long ne = offsets[e + 1] - offsets[e];
    if (ne <= 0) return fail(c, SGP_E_BADARG, "empty expert");
    if (ne > nmax) nmax = static_cast<int>(ne);
  }
  // (no upper bound on the expert size -- GaussianProcessParams.scala:36: experts above the on-chip kernel's ~165 points
  //  take the global-memory LU path of sgp_bcm_nll)
  const int rc = experts_alloc(c, E, n, d, nmax);
  if (rc != SGP_OK) return rc;
  SGP_CUDA(c, cudaMemcpyAsync(c->ex.X, X, static_cast<size_t>(n) * d * 8, cudaMemcpyHostToDevice, c->stream));
  SGP_CUDA(c, cudaMemcpyAsync(c->ex.y, y, static_cast<size_t>(n) * 8, cudaMemcpyHostToDevice, c->stream));
  SGP_CUDA(c, cudaMemcpyAsync(c->ex.off, offsets, static_cast<size_t>(E + 1) * 8, cudaMemcpyHostToDevice, c->stream));
  SGP_CUDA(c, cudaStreamSynchronize(c->stream));
  c->ex.E = E;
  return SGP_OK;
}

namespace {
// sgp_experts_upload_grouped and its _device form: X and y are host memory (staged) or device memory (read in place)
// E experts, point i -> expert i % E (after the caller's argument checks)
int upload_strided(Ctx* c, bool on_device, const void* X, int x_is_f32, const double* y, long long n, int d, long long E) {
  int rc = experts_alloc(c, E, n, d, static_cast<int>(n / E + ((n % E) ? 1 : 0)));
  if (rc != SGP_OK) return rc;
  SGP_CUDA(c, launch_expert_offsets(c->ex.off, n, E, 0, c->stream));
  // host input streams through the double-buffered staging area of the statistics path; either way the gather is on the
  // device, chunk by chunk
  const size_t row = static_cast<size_t>(d) * (x_is_f32 ? 4 : 8);
  const long long chunk = group_chunk(n, row);
  rc = feed_rows(c, on_device, X, y, n, row, chunk, [&](const void* dX, const double* dy, long long p0, long long cn) -> int {
    SGP_CUDA(c, launch_group_experts(c->ex.X, c->ex.y, dX, x_is_f32, dy, n, d, E, p0, cn, nullptr, 0, c->stream));
    c->launches += 1;
    return SGP_OK;
  });
  if (rc != SGP_OK) return rc;
  SGP_CUDA(c, cudaStreamSynchronize(c->stream));
  c->ex.E = E;
  c->ex_grouped = true;
  return SGP_OK;
}

int upload_grouped(Ctx* c, bool on_device, const void* X, int x_is_f32, const double* y, long long n, int d,
                   int dataset_size_for_expert, const char* entry) {
  if (!X || !y || n <= 0 || d <= 0 || dataset_size_for_expert <= 0)
    return fail(c, SGP_E_BADARG, std::string(entry) + ": null or empty argument");
  SGP_CUDA(c, cudaSetDevice(c->device));
  if (on_device) {
    int rc = device_ptr_ok(c, X, entry, "X");
    if (rc == SGP_OK) rc = device_ptr_ok(c, y, entry, "y");
    if (rc != SGP_OK) return rc;
  }
  // GPC:27  numberOfExperts = Math.round(points.count() / datasetSizeForExpert)  (round half up on a positive double)
  const long long E = static_cast<long long>(std::floor(static_cast<double>(n) / dataset_size_for_expert + 0.5));
  if (E <= 0) return fail(c, SGP_E_BADARG, "numberOfExperts == 0 (N < datasetSizeForExpert / 2): the reference fails with / by zero");
  return upload_strided(c, on_device, X, x_is_f32, y, n, d, E);
}

// The free-memory rule of the fold uploads: the sets' rows, labels and modes, n_rows (d + 2) doubles, against what the
// device has free plus what the context's expert buffers already hold.
int fold_sets_fit(Ctx* c, long long n_rows, int d, const char* entry) {
  size_t free_b = 0, total_b = 0;
  SGP_CUDA(c, cudaMemGetInfo(&free_b, &total_b));
  const size_t held = c->ex_X.cap + c->ex_y.cap + c->ex_f.buf.cap;
  const size_t need = static_cast<size_t>(n_rows) * (static_cast<size_t>(d) + 2) * 8;
  if (need > free_b + held)
    return fail(c, SGP_E_NOMEM, std::string(entry) + ": the training sets need " + std::to_string(need >> 20) +
                                    " MiB of device memory, " + std::to_string((free_b + held) >> 20) + " MiB available");
  return SGP_OK;
}

// sgp_experts_upload_folds and its _device form; fold_of is host memory in both
int upload_folds(Ctx* c, bool on_device, const void* X, int x_is_f32, const double* y, long long n, int d,
                 const int32_t* fold_of, int n_folds, int dataset_size_for_expert, const char* entry) {
  if (!X || !y || !fold_of || n <= 0 || d <= 0 || dataset_size_for_expert <= 0)
    return fail(c, SGP_E_BADARG, std::string(entry) + ": null or empty argument");
  if (n_folds < 2) return fail(c, SGP_E_BADARG, std::string(entry) + ": n_folds must be >= 2");
  if (on_device) {
    SGP_CUDA(c, cudaSetDevice(c->device));
    int rc = device_ptr_ok(c, X, entry, "X");
    if (rc == SGP_OK) rc = device_ptr_ok(c, y, entry, "y");
    if (rc != SGP_OK) return rc;
  }
  // the points of each fold in index order: set k leaves out pos[fstart[k] .. fstart[k+1]-1]
  std::vector<long long> fstart(static_cast<size_t>(n_folds) + 1, 0);
  for (int64_t i = 0; i < n; ++i) {
    if (fold_of[i] < 0 || fold_of[i] >= n_folds)
      return fail(c, SGP_E_BADARG, std::string(entry) + ": fold index of point " + std::to_string(i) + " outside [0, n_folds)");
    ++fstart[fold_of[i] + 1];
  }
  for (int k = 0; k < n_folds; ++k) fstart[k + 1] += fstart[k];
  std::vector<long long> pos(static_cast<size_t>(n)), next(fstart.begin(), fstart.end() - 1);
  for (int64_t i = 0; i < n; ++i) pos[next[fold_of[i]]++] = i;
  // set k: N_k = n - |fold k| training points in E_k = round(N_k / n_e) experts (GPC:26-31), stored after set k-1
  std::vector<long long> first(static_cast<size_t>(n_folds) + 1, 0), row0(static_cast<size_t>(n_folds) + 1, 0);
  std::vector<int> nmax(n_folds);
  for (int k = 0; k < n_folds; ++k) {
    const long long Nk = n - (fstart[k + 1] - fstart[k]);
    const long long Ek = static_cast<long long>(std::floor(static_cast<double>(Nk) / dataset_size_for_expert + 0.5));
    if (Ek <= 0)
      return fail(c, SGP_E_BADARG, "fold " + std::to_string(k) + ": numberOfExperts == 0 (N < datasetSizeForExpert / 2): "
                                   "the reference fails with / by zero");
    first[k + 1] = first[k] + Ek;
    row0[k + 1] = row0[k] + Nk;
    nmax[k] = static_cast<int>(Nk / Ek + ((Nk % Ek) ? 1 : 0));
  }
  const long long n_rows = row0[n_folds], E = first[n_folds];
  SGP_CUDA(c, cudaSetDevice(c->device));
  int rc = fold_sets_fit(c, n_rows, d, entry);              // (n_folds - 1) n (d + 2) doubles
  if (rc != SGP_OK) return rc;
  rc = experts_alloc(c, E, n_rows, d, *std::max_element(nmax.begin(), nmax.end()));
  if (rc == SGP_OK) rc = ctx_scratch(c, c->fold_pos_ws, static_cast<size_t>(n) * 8);
  if (rc != SGP_OK) return rc;
  const long long* dpos = c->fold_pos_ws.as<long long>();
  SGP_CUDA(c, cudaMemcpyAsync(c->fold_pos_ws.p, pos.data(), pos.size() * 8, cudaMemcpyHostToDevice, c->stream));
  for (int k = 0; k < n_folds; ++k) {
    SGP_CUDA(c, launch_expert_offsets(c->ex.off + first[k], row0[k + 1] - row0[k], first[k + 1] - first[k], row0[k],
                                      c->stream));
    c->launches += 1;
  }
  // X and y are read once (host input: cross PCIe once); each chunk is gathered into every training set that holds its
  // points
  const size_t row = static_cast<size_t>(d) * (x_is_f32 ? 4 : 8);
  const long long chunk = group_chunk(n, row);
  rc = feed_rows(c, on_device, X, y, n, row, chunk, [&](const void* dX, const double* dy, long long p0, long long cn) -> int {
    for (int k = 0; k < n_folds; ++k) {
      SGP_CUDA(c, launch_group_experts(c->ex.X + static_cast<size_t>(row0[k]) * d, c->ex.y + row0[k], dX, x_is_f32, dy,
                                       row0[k + 1] - row0[k], d, first[k + 1] - first[k], p0, cn, dpos + fstart[k],
                                       fstart[k + 1] - fstart[k], c->stream));
      c->launches += 1;
    }
    return SGP_OK;
  });
  if (rc != SGP_OK) return rc;
  SGP_CUDA(c, cudaStreamSynchronize(c->stream));
  c->fold_first = first;
  c->fold_nmax = nmax;
  c->fold_row0 = row0;
  c->ex.E = E;
  return SGP_OK;
}
}  // namespace

int sgp_experts_upload_fold_sets_device(sgp_ctx* h, const void* dX, int32_t x_is_f32, const double* dy,
                                        const int64_t* set_rows, const int64_t* set_experts, int32_t n_sets, int32_t d) {
  Ctx* c = reinterpret_cast<Ctx*>(h);
  if (!c) return SGP_E_BADARG;
  const char* entry = "sgp_experts_upload_fold_sets_device";
  if (!dX || !dy || !set_rows || !set_experts || n_sets < 1 || d < 1)
    return fail(c, SGP_E_BADARG, std::string(entry) + ": null or empty argument");
  // set k: set_rows[k] rows in set_experts[k] experts, stored after set k-1, as upload_folds stores its sets
  std::vector<long long> first(static_cast<size_t>(n_sets) + 1, 0), row0(static_cast<size_t>(n_sets) + 1, 0);
  std::vector<int> nmax(n_sets);
  for (int k = 0; k < n_sets; ++k) {
    const long long Nk = set_rows[k], Ek = set_experts[k];
    if (Nk < 1 || Ek < 1)
      return fail(c, SGP_E_BADARG, std::string(entry) + ": set " + std::to_string(k) + " has no rows or no experts");
    if (Ek > Nk)
      return fail(c, SGP_E_BADARG, std::string(entry) + ": set " + std::to_string(k) +
                                       ": more experts than rows (an empty expert)");
    first[k + 1] = first[k] + Ek;
    row0[k + 1] = row0[k] + Nk;
    nmax[k] = static_cast<int>(Nk / Ek + ((Nk % Ek) ? 1 : 0));
  }
  SGP_CUDA(c, cudaSetDevice(c->device));
  int rc = device_ptr_ok(c, dX, entry, "X");
  if (rc == SGP_OK) rc = device_ptr_ok(c, dy, entry, "y");
  if (rc == SGP_OK) rc = fold_sets_fit(c, row0[n_sets], d, entry);
  if (rc == SGP_OK) rc = experts_alloc(c, first[n_sets], row0[n_sets], d, *std::max_element(nmax.begin(), nmax.end()));
  if (rc != SGP_OK) return rc;
  for (int k = 0; k < n_sets; ++k) {
    SGP_CUDA(c, launch_expert_offsets(c->ex.off + first[k], row0[k + 1] - row0[k], first[k + 1] - first[k], row0[k],
                                      c->stream));
    c->launches += 1;
  }
  // block k is set k's rows in order: the fold upload's gather with no left-out points, in chunks of the same size
  const size_t row = static_cast<size_t>(d) * (x_is_f32 ? 4 : 8);
  const char* X = static_cast<const char*>(dX);
  for (int k = 0; k < n_sets; ++k) {
    const long long Nk = row0[k + 1] - row0[k], chunk = group_chunk(Nk, row);
    for (long long p0 = 0; p0 < Nk; p0 += chunk) {
      const long long cn = std::min(chunk, Nk - p0), at = row0[k] + p0;
      SGP_CUDA(c, launch_group_experts(c->ex.X + static_cast<size_t>(row0[k]) * d, c->ex.y + row0[k],
                                       X + static_cast<size_t>(at) * row, x_is_f32, dy + at, Nk, d,
                                       first[k + 1] - first[k], p0, cn, nullptr, 0, c->stream));
      c->launches += 1;
    }
  }
  SGP_CUDA(c, cudaStreamSynchronize(c->stream));
  c->fold_first = first;
  c->fold_nmax = nmax;
  c->fold_row0 = row0;
  c->ex.E = first[n_sets];
  return SGP_OK;
}

int sgp_experts_upload_grouped(sgp_ctx* h, const void* X, int32_t x_is_f32, const double* y, int64_t n, int32_t d,
                               int32_t dataset_size_for_expert) {
  Ctx* c = reinterpret_cast<Ctx*>(h);
  if (!c) return SGP_E_BADARG;
  return upload_grouped(c, false, X, x_is_f32, y, n, d, dataset_size_for_expert, "sgp_experts_upload_grouped");
}

int sgp_experts_upload_grouped_device(sgp_ctx* h, const void* dX, int32_t x_is_f32, const double* dy, int64_t n, int32_t d,
                                      int32_t dataset_size_for_expert) {
  Ctx* c = reinterpret_cast<Ctx*>(h);
  if (!c) return SGP_E_BADARG;
  return upload_grouped(c, true, dX, x_is_f32, dy, n, d, dataset_size_for_expert, "sgp_experts_upload_grouped_device");
}

int sgp_experts_upload_strided_device(sgp_ctx* h, const void* dX, int32_t x_is_f32, const double* dy, int64_t n, int32_t d,
                                      int64_t n_experts) {
  Ctx* c = reinterpret_cast<Ctx*>(h);
  if (!c) return SGP_E_BADARG;
  const char* entry = "sgp_experts_upload_strided_device";
  if (!dX || !dy || n <= 0 || d <= 0 || n_experts <= 0)
    return fail(c, SGP_E_BADARG, std::string(entry) + ": null or empty argument");
  if (n_experts > n) return fail(c, SGP_E_BADARG, std::string(entry) + ": more experts than points (an empty expert)");
  SGP_CUDA(c, cudaSetDevice(c->device));
  int rc = device_ptr_ok(c, dX, entry, "X");
  if (rc == SGP_OK) rc = device_ptr_ok(c, dy, entry, "y");
  if (rc != SGP_OK) return rc;
  return upload_strided(c, true, dX, x_is_f32, dy, n, d, n_experts);
}

int sgp_experts_upload_folds(sgp_ctx* h, const void* X, int32_t x_is_f32, const double* y, int64_t n, int32_t d,
                             const int32_t* fold_of, int32_t n_folds, int32_t dataset_size_for_expert) {
  Ctx* c = reinterpret_cast<Ctx*>(h);
  if (!c) return SGP_E_BADARG;
  return upload_folds(c, false, X, x_is_f32, y, n, d, fold_of, n_folds, dataset_size_for_expert,
                      "sgp_experts_upload_folds");
}

int sgp_experts_upload_folds_device(sgp_ctx* h, const void* dX, int32_t x_is_f32, const double* dy, int64_t n, int32_t d,
                                    const int32_t* fold_of, int32_t n_folds, int32_t dataset_size_for_expert) {
  Ctx* c = reinterpret_cast<Ctx*>(h);
  if (!c) return SGP_E_BADARG;
  return upload_folds(c, true, dX, x_is_f32, dy, n, d, fold_of, n_folds, dataset_size_for_expert,
                      "sgp_experts_upload_folds_device");
}

namespace {
// The expert sets an objective call's slots index: set k is the experts first[k] .. first[k+1]-1, the largest of nmax[k]
// points.  The fold upload's training sets, or the whole upload as the one set {0, E}.
struct ExpertSets {
  std::vector<long long> first;    // [n_sets + 1]
  std::vector<int> nmax;           // [n_sets]
};
ExpertSets whole_upload(const Ctx* c) { return {{0, c->ex.E}, {c->ex.n_max}}; }
ExpertSets fold_sets(const Ctx* c) { return {c->fold_first, c->fold_nmax}; }

// The slots of one objective call, in list order: slot i evaluates expert set sets[i] at kernels[i] and the descriptors
// hypers + i * nh; the Laplace objective adds the labels (y == cls[i]) (-1: as uploaded) and the modes of mode slot
// modes[i].  A failing slot is named `what` names[i] (what == nullptr: not named).  The constructor makes n slots on
// the whole upload with the labels as uploaded and mode slot 0; the entries fill in what differs.
struct SlotList {
  const sgp_kernel_desc* kernels;
  const sgp_hyper* hypers;
  int nh;
  std::vector<int> sets, cls, modes, names;
  const char* what = nullptr;
  SlotList(const sgp_kernel_desc* k, const sgp_hyper* h, int n_hypers, int n)
      : kernels(k), hypers(h), nh(n_hypers), sets(n, 0), cls(n, -1), modes(n, 0), names(n, 0) {}
};

// Device state of one objective evaluation, in the context's descriptor block.  Set-up slot j is list slot pos[j].
struct ObjectiveSetup {
  HyperView hv;                    // set-up slot 0
  ObjectiveSlots slots;            // the slot table (f and f_stride: the Laplace objective's to fill)
  std::vector<KernelFlat> kf_host; // [n_slots]
  ExpertSets es;                   // the sets the slots index
  std::vector<int> set, pos;       // [n_slots] set-up slot j's expert set and list position
  std::vector<int> names;          // [n_slots] list order
  const char* what = nullptr;
  double* total = nullptr;         // [n_slots][1 + n_hypers] totals, then [n_slots] status words
  int* flags = nullptr;            // [n_slots]
};

// Flattens each slot's kernel (flatten_kernel: Eye terms only add to the diagonal), maps its hyper-parameter descriptors
// onto the flattened terms and uploads everything, with the sets' first experts, the slot list and zeroed totals and
// flags, into the context's descriptor block in one copy.  The slots are set up in the order pos (empty: list order).
// Every slot must have the first one's kernel structure and descriptor kinds.
int objective_setup(Ctx* c, const SlotList& L, ExpertSets es, ObjectiveSetup& o, std::vector<int> pos = {}) {
  if (c->ex.E == 0) return fail(c, SGP_E_STATE, "sgp_experts_upload should have been called first");
  const int nh = L.nh, n_slots = static_cast<int>(L.sets.size());
  if (!L.kernels || nh < 0 || (nh > 0 && !L.hypers)) return fail(c, SGP_E_BADARG, "null argument");
  if (pos.empty()) {
    pos.resize(n_slots);
    std::iota(pos.begin(), pos.end(), 0);
  }
  for (int s = 0; s < n_slots; ++s)
    if (!L.kernels[pos[s]].terms || L.kernels[pos[s]].n_terms <= 0) return fail(c, SGP_E_BADARG, "null argument");
  if (nh > kMaxHypers) return fail(c, SGP_E_BADARG, "too many hyper-parameters");
  const int d = c->ex.d;
  const sgp_kernel_desc* k = L.kernels + pos[0];
  const sgp_hyper* h0 = L.hypers ? L.hypers + static_cast<size_t>(pos[0]) * nh : nullptr;
  std::vector<KernelFlat> kfs(n_slots);
  std::vector<int> flat_of;
  std::vector<double> block;       // [n_slots][beta | coef | value]
  std::vector<int> kind(nh), hterm(nh, 0), hdim(nh, 0);
  size_t nb = 0;                   // beta doubles of one slot
  o = ObjectiveSetup{};
  HyperView& hv = o.hv;
  hv.d = d; hv.n_hypers = nh;
  for (int s = 0; s < n_slots; ++s) {
    const sgp_kernel_desc* ks = L.kernels + pos[s];
    const sgp_hyper* hs = L.hypers ? L.hypers + static_cast<size_t>(pos[s]) * nh : nullptr;
    if (s > 0) {
      bool same = ks->n_terms == k->n_terms;
      for (int t = 0; same && t < k->n_terms; ++t) same = ks->terms[t].type == k->terms[t].type;
      for (int i = 0; same && i < nh; ++i)
        same = hs[i].kind == kind[i] && (hs[i].kind == SGP_HYPER_SCALE || (hs[i].term == h0[i].term && hs[i].dim == hdim[i]));
      if (!same) return fail(c, SGP_E_BADARG, "every class or fold slot needs the same kernel structure and hyper-parameter layout");
    }
    std::vector<double> beta;
    int rc = flatten_kernel(c, ks, d, d, kfs[s], beta, &flat_of);
    if (rc != SGP_OK) return rc;
    std::vector<double> coef(static_cast<size_t>(nh) * (kMaxTerms + 1), 0.0), value(nh, 0.0);
    for (int i = 0; i < nh; ++i) {
      kind[i] = hs[i].kind;
      value[i] = hs[i].value;
      if (hs[i].kind == SGP_HYPER_SCALE) {
        if (!hs[i].coef) return fail(c, SGP_E_BADARG, "SCALE hyper-parameter without coef");
        for (int t = 0; t < ks->n_terms; ++t) {
          const size_t col = (flat_of[t] >= 0) ? static_cast<size_t>(flat_of[t]) : static_cast<size_t>(kMaxTerms);
          coef[static_cast<size_t>(i) * (kMaxTerms + 1) + col] += hs[i].coef[t];
        }
      } else if (hs[i].kind == SGP_HYPER_ARD_BETA || hs[i].kind == SGP_HYPER_RBF_SIGMA) {
        if (hs[i].term < 0 || hs[i].term >= ks->n_terms || flat_of[hs[i].term] < 0)
          return fail(c, SGP_E_BADARG, "hyper-parameter refers to a bad term");
        hterm[i] = flat_of[hs[i].term];
        hdim[i] = hs[i].dim;
        if (hs[i].kind == SGP_HYPER_ARD_BETA) hv.any_ard = 1;
        if (hs[i].kind == SGP_HYPER_ARD_BETA && (hdim[i] < 0 || hdim[i] >= d)) return fail(c, SGP_E_BADARG, "bad ARD dim");
      } else {
        return fail(c, SGP_E_BADARG, "unknown hyper-parameter kind");
      }
    }
    if (s == 0) {
      hv.kf = kfs[0];
      nb = beta.size();
      o.slots.slot_stride = static_cast<long long>(beta.size() + coef.size() + value.size());
    }
    block.insert(block.end(), beta.begin(), beta.end());
    block.insert(block.end(), coef.begin(), coef.end());
    block.insert(block.end(), value.begin(), value.end());
  }
  o.set.resize(n_slots);
  std::vector<int> cls(n_slots), modes(n_slots);
  for (int s = 0; s < n_slots; ++s) {
    const int k_s = o.set[s] = L.sets[pos[s]];
    cls[s] = L.cls[pos[s]];
    modes[s] = L.modes[pos[s]];
    o.slots.E_max = std::max(o.slots.E_max, es.first[k_s + 1] - es.first[k_s]);
  }
  // [KernelFlat n_slots] then doubles [slot blocks | totals | status], long longs [first], then ints [kind | term | dim
  // | flags | sets | classes | modes]
  const int W = 1 + nh;
  const size_t kf_bytes = sizeof(KernelFlat) * n_slots;
  const size_t n_dbl = block.size() + static_cast<size_t>(n_slots) * (W + 1);
  const size_t n_first = es.first.size();
  const size_t n_int = 3 * static_cast<size_t>(nh) + 4 * static_cast<size_t>(n_slots);
  std::vector<char> host(kf_bytes + (n_dbl + n_first) * 8 + n_int * 4, 0);
  std::memcpy(host.data(), kfs.data(), kf_bytes);
  std::memcpy(host.data() + kf_bytes, block.data(), block.size() * 8);
  std::memcpy(host.data() + kf_bytes + n_dbl * 8, es.first.data(), n_first * 8);
  int* hi = reinterpret_cast<int*>(host.data() + kf_bytes + (n_dbl + n_first) * 8);
  std::copy(kind.begin(), kind.end(), hi);
  std::copy(hterm.begin(), hterm.end(), hi + nh);
  std::copy(hdim.begin(), hdim.end(), hi + 2 * nh);
  std::copy(o.set.begin(), o.set.end(), hi + 3 * nh + n_slots);
  std::copy(cls.begin(), cls.end(), hi + 3 * nh + 2 * n_slots);
  std::copy(modes.begin(), modes.end(), hi + 3 * nh + 3 * n_slots);
  int rc = ctx_scratch(c, c->hyper_ws, host.size());
  if (rc != SGP_OK) return rc;
  char* dev = c->hyper_ws.as<char>();
  SGP_CUDA(c, cudaMemcpyAsync(dev, host.data(), host.size(), cudaMemcpyHostToDevice, c->stream));
  SGP_CUDA(c, cudaStreamSynchronize(c->stream));          // host is a local
  rc = ctx_scratch(c, c->nll_per_ws, static_cast<size_t>(n_slots) * o.slots.E_max * W * 8);
  if (rc != SGP_OK) return rc;
  double* dD = reinterpret_cast<double*>(dev + kf_bytes);
  int* dI = reinterpret_cast<int*>(dD + n_dbl + n_first);
  hv.beta = dD; hv.h_coef = dD + nb; hv.h_value = hv.h_coef + static_cast<size_t>(nh) * (kMaxTerms + 1);
  hv.h_kind = dI; hv.h_term = dI + nh; hv.h_dim = dI + 2 * nh;
  o.total = dD + block.size();
  o.flags = dI + 3 * nh;
  o.slots.n_slots = n_slots;
  o.slots.kf = reinterpret_cast<const KernelFlat*>(dev);
  o.slots.first = reinterpret_cast<const long long*>(dD + n_dbl);
  o.slots.sets = o.flags + n_slots;
  o.slots.cls = o.flags + 2 * n_slots;
  o.slots.mode = o.flags + 3 * n_slots;
  o.kf_host = std::move(kfs);
  o.es = std::move(es);
  o.pos = std::move(pos);
  o.names = L.names;
  o.what = L.what;
  return SGP_OK;
}

// Set-up slot s's view of the descriptors: its flattened kernel and its [beta | coef | value] block.
HyperView slot_view(const ObjectiveSetup& o, int s) {
  HyperView hv = o.hv;
  hv.kf = o.kf_host[s];
  const long long shift = s * o.slots.slot_stride;
  hv.beta += shift; hv.h_coef += shift; hv.h_value += shift;
  return hv;
}

// Set-up slots [s0, s1) as one launch: the upload seen with the largest expert over their sets (the kernels lay out
// their shared memory and workspace from it), their slot table, the first one's view and their outputs.
struct SlotRange {
  ExpertSet view;
  ObjectiveSlots slots;
  HyperView hv;
  double* rows;
  double* total;
  int* flags;
};
SlotRange slot_range(const Ctx* c, const ObjectiveSetup& o, int s0, int s1) {
  const size_t W = 1 + o.hv.n_hypers;
  SlotRange r{c->ex, o.slots, slot_view(o, s0), c->nll_per_ws.as<double>() + s0 * o.slots.E_max * W, o.total + s0 * W,
              o.flags + s0};
  r.view.n_max = 0;
  r.slots.E_max = 0;
  for (int s = s0; s < s1; ++s) {
    r.view.n_max = std::max(r.view.n_max, o.es.nmax[o.set[s]]);
    r.slots.E_max = std::max(r.slots.E_max, o.es.first[o.set[s] + 1] - o.es.first[o.set[s]]);
  }
  r.slots.n_slots = s1 - s0;
  r.slots.sets += s0; r.slots.kf += s0; r.slots.cls += s0; r.slots.mode += s0;
  return r;
}

// All-reduces over ranks, copies every slot's (objective, gradient) row to its list position and maps a status word to
// err_code, naming the failing slot of the smallest list position.
int objective_finish(Ctx* c, const ObjectiveSetup& o, int nh, double* val_out, double* grad_out, int mask, int err_code,
                     const char* err_msg) {
  const int W = 1 + nh, S = o.slots.n_slots;
  // the rank-local status flags are all-reduced WITH the totals so that every rank raises (or none does)
  SGP_CUDA(c, launch_flags_to_double(o.total + static_cast<size_t>(S) * W, o.flags, mask, S, c->stream));
  c->launches += 1;
  const size_t len = static_cast<size_t>(S) * (W + 1);
  std::vector<double> tot(len);
  std::vector<int> at = o.pos;                      // the list position of row s
  if (c->comm && c->nranks > 1) {
    if (!std::is_sorted(at.begin(), at.end())) {
      // The row a slot was set up in follows the rank's own experts (the Laplace [on chip | global memory] split), so
      // ranks may disagree on it: move every row and status word to its list position before the sum.
      std::vector<double> set_up(len);
      SGP_CUDA(c, cudaMemcpyAsync(set_up.data(), o.total, len * 8, cudaMemcpyDeviceToHost, c->stream));
      SGP_CUDA(c, cudaStreamSynchronize(c->stream));
      for (int s = 0; s < S; ++s) {
        std::copy(set_up.begin() + static_cast<size_t>(s) * W, set_up.begin() + static_cast<size_t>(s + 1) * W,
                  tot.begin() + static_cast<size_t>(at[s]) * W);
        tot[static_cast<size_t>(S) * W + at[s]] = set_up[static_cast<size_t>(S) * W + s];
      }
      SGP_CUDA(c, cudaMemcpyAsync(o.total, tot.data(), len * 8, cudaMemcpyHostToDevice, c->stream));
      SGP_CUDA(c, cudaStreamSynchronize(c->stream));
      std::iota(at.begin(), at.end(), 0);
    }
    ncclResult_t r = nccl().AllReduce(o.total, o.total, len, ncclDouble, ncclSum, c->comm, c->stream);
    if (r != ncclSuccess) return fail(c, SGP_E_NCCL, std::string("ncclAllReduce: ") + nccl().GetErrorString(r));
    c->launches += 1;
  }
  SGP_CUDA(c, cudaMemcpyAsync(tot.data(), o.total, len * 8, cudaMemcpyDeviceToHost, c->stream));
  SGP_CUDA(c, cudaStreamSynchronize(c->stream));
  int failed = -1;
  for (int s = 0; s < S; ++s)
    if (tot[static_cast<size_t>(S) * W + s] != 0.0 && (failed < 0 || at[s] < at[failed])) failed = s;
  if (failed >= 0)
    return fail(c, err_code, o.what ? std::string(o.what) + " " + std::to_string(o.names[at[failed]]) + ": " + err_msg
                                    : std::string(err_msg));
  for (int s = 0; s < S; ++s) {
    val_out[at[s]] = tot[static_cast<size_t>(s) * W];
    for (int i = 1; i < W; ++i) grad_out[static_cast<size_t>(at[s]) * nh + i - 1] = tot[static_cast<size_t>(s) * W + i];
  }
  return SGP_OK;
}
}  // namespace

const char* const kBcmSingular =
    "an expert's kernel matrix is singular (MatrixSingularException, logDetAndInv.scala:27-28)";

namespace {
// The LU path indexes an expert's n x n matrix in int: refused above kBcmLuMaxPoints, before any allocation or launch.
int bcm_check_size(Ctx* c, int n_max, const char* fn) {
  if (n_max <= kBcmLuMaxPoints) return SGP_OK;
  return fail(c, SGP_E_BADARG, std::string(fn) + ": datasetSizeForExpert above " + std::to_string(kBcmLuMaxPoints) +
                                   " points (the largest expert has " + std::to_string(n_max) +
                                   "; 32-bit indexing of the per-expert kernel matrix)");
}

// c->bcm_ws sized for the LU path's workspace (every expert's K and K^-1 at once).  SGP_E_NOMEM, before allocating, when
// it exceeds the device's free memory plus what bcm_ws already holds.
int bcm_lu_workspace(Ctx* c, const ObjectivePlan& plan) {
  size_t free_b = 0, total_b = 0;
  SGP_CUDA(c, cudaMemGetInfo(&free_b, &total_b));
  const size_t avail = free_b + c->bcm_ws.cap;
  if (plan.lu_ws > avail)
    return fail(c, SGP_E_NOMEM, "the BCM objective's LU path needs " + std::to_string(plan.lu_ws >> 20) +
                                    " MiB of device memory for the experts' kernel matrices and inverses, " +
                                    std::to_string(avail >> 20) + " MiB available (lower datasetSizeForExpert)");
  return ctx_scratch(c, c->bcm_ws, plan.lu_ws);
}

// The BCM objective of a slot list, in one on-chip launch over experts x slots planned on the largest expert over the
// listed sets (on-chip Cholesky per expert: SPD kernel matrices of <= ~165 points, every default configuration).  A slot
// whose Cholesky broke down (not positive definite), or every slot when the experts do not fit on chip, takes the general
// path on its set alone (its experts, its own largest expert), one slot after another: the reference's own arithmetic,
// LU with partial pivoting and log|det| with the sign dropped (logDetAndInv.scala:36-63, GPR:59), on kernel matrices
// staged in global memory.  The choice is rank-local; the one all-reduce per evaluation happens afterwards on every rank.
int bcm_objective(Ctx* c, const char* fn, const SlotList& L, ExpertSets es, double* nll_out, double* grad_out) {
  SGP_CUDA(c, cudaSetDevice(c->device));
  if (c->ex.E > 0) {                          // (without experts, objective_setup refuses)
    int n_max = 0;
    for (int k : L.sets) n_max = std::max(n_max, es.nmax[k]);
    const int rc = bcm_check_size(c, n_max, fn);
    if (rc != SGP_OK) return rc;
  }
  ObjectiveSetup o;
  int rc = objective_setup(c, L, std::move(es), o);
  if (rc != SGP_OK) return rc;
  const int n = o.slots.n_slots;
  const SlotRange all = slot_range(c, o, 0, n);
  const ObjectivePlan plan = plan_objective(Objective::kBcm, all.view, o.hv.kf.n_terms);
  std::vector<int> flags(n, 1);               // bit 0: the slot goes to the LU path
  if (plan.variant != ObjectiveVariant::kLu) {
    SGP_CUDA(c, launch_bcm_nll(plan, all.view, all.hv, all.slots, all.rows, all.total, all.flags, c->stream));
    c->launches += 2;
    SGP_CUDA(c, cudaMemcpyAsync(flags.data(), o.flags, sizeof(int) * n, cudaMemcpyDeviceToHost, c->stream));
    SGP_CUDA(c, cudaStreamSynchronize(c->stream));
  }
  c->bcm_general = false;
  for (int s = 0; s < n; ++s) {
    if (!(flags[s] & 1)) continue;
    c->bcm_general = true;
    const SlotRange one = slot_range(c, o, s, s + 1);
    ExpertSet set = one.view;
    set.off += o.es.first[o.set[s]];
    set.E = one.slots.E_max;
    const ObjectivePlan lu = plan_objective(Objective::kBcmLu, set, one.hv.kf.n_terms);
    rc = bcm_lu_workspace(c, lu);
    if (rc != SGP_OK) return rc;
    SGP_CUDA(c, cudaMemsetAsync(one.flags, 0, sizeof(int), c->stream));
    int blas_status = 0;
    SGP_CUDA(c, launch_bcm_nll_general(lu, c->blas, &blas_status, c->bcm_ws.p, set, one.hv, one.rows, one.total,
                                       one.flags, c->stream));
    if (blas_status != 0) return fail(c, SGP_E_CUDA, "cuBLAS batched LU failed, status " + std::to_string(blas_status));
    c->launches += 5;
  }
  return objective_finish(c, o, L.nh, nll_out, grad_out, 2, SGP_E_SINGULAR, kBcmSingular);
}
}  // namespace

int sgp_bcm_nll(sgp_ctx* h, const sgp_kernel_desc* k, const sgp_hyper* hypers, int32_t nh, double* nll_out,
                double* grad_out) {
  Ctx* c = reinterpret_cast<Ctx*>(h);
  if (!c) return SGP_E_BADARG;
  if (!nll_out || (nh > 0 && !grad_out)) return fail(c, SGP_E_BADARG, "sgp_bcm_nll: null output");
  return bcm_objective(c, "sgp_bcm_nll", SlotList(k, hypers, nh, 1), whole_upload(c), nll_out, grad_out);
}

int sgp_bcm_nll_folds(sgp_ctx* h, const int32_t* sets, int32_t n_eval, const sgp_kernel_desc* kernels,
                      const sgp_hyper* hypers, int32_t nh, double* nll_out, double* grad_out) {
  Ctx* c = reinterpret_cast<Ctx*>(h);
  if (!c) return SGP_E_BADARG;
  if (!nll_out || (nh > 0 && !grad_out) || !sets) return fail(c, SGP_E_BADARG, "sgp_bcm_nll_folds: null argument");
  if (c->ex.E == 0 || c->fold_first.empty())
    return fail(c, SGP_E_STATE, "sgp_experts_upload_folds should have been called first");
  const int n_sets = static_cast<int>(c->fold_first.size()) - 1;
  if (n_eval < 1 || n_eval > 65535) return fail(c, SGP_E_BADARG, "sgp_bcm_nll_folds: need 1 <= n_eval <= 65535");
  for (int s = 0; s < n_eval; ++s)
    if (sets[s] < 0 || sets[s] >= n_sets)
      return fail(c, SGP_E_BADARG, "sgp_bcm_nll_folds: set index " + std::to_string(sets[s]) + " outside [0, n_folds)");
  SlotList L(kernels, hypers, nh, n_eval);
  L.sets.assign(sets, sets + n_eval);
  L.names = L.sets;
  L.what = "fold set";
  return bcm_objective(c, "sgp_bcm_nll_folds", L, fold_sets(c), nll_out, grad_out);
}

int sgp_bcm_nll_slots(sgp_ctx* h, int32_t n_eval, const sgp_kernel_desc* kernels, const sgp_hyper* hypers, int32_t nh,
                      double* nll_out, double* grad_out) {
  Ctx* c = reinterpret_cast<Ctx*>(h);
  if (!c) return SGP_E_BADARG;
  if (!nll_out || (nh > 0 && !grad_out)) return fail(c, SGP_E_BADARG, "sgp_bcm_nll_slots: null argument");
  if (c->ex.E == 0 || !c->ex_grouped)
    return fail(c, SGP_E_STATE, "sgp_experts_upload_grouped should have been called first (sgp_bcm_nll_slots evaluates "
                                "one grouped training set; a fold upload or sgp_experts_upload has none)");
  if (n_eval < 1 || n_eval > 65535) return fail(c, SGP_E_BADARG, "sgp_bcm_nll_slots: need 1 <= n_eval <= 65535");
  SlotList L(kernels, hypers, nh, n_eval);    // every slot on the whole upload, named by its index
  std::iota(L.names.begin(), L.names.end(), 0);
  L.what = "slot";
  return bcm_objective(c, "sgp_bcm_nll_slots", L, whole_upload(c), nll_out, grad_out);
}

const char* const kLaplaceRefused =
    "datasetSizeForExpert too large for the on-chip Laplace kernel (max ~115 points per expert)";
const char* const kLaplaceNotPd = "an expert's B = I + sqrt(W) K sqrt(W) is not positive definite (increase sigma2)";
const char* const kLaplaceNoIteration =
    "tol >= 1: no Newton iteration runs (the loop needs step = 1 > tol), so L stays zero and L \\ sqrtW throws "
    "MatrixSingularException (GaussianProcessClassifier.scala:91,116)";

namespace {
// A mode store of n_store slots of `stride` modes each, (re)allocated and zeroed when store.slots, the count it was set
// up for, differs (0 after every upload).  SGP_E_NOMEM, before allocating, past the device's free memory; a failed
// allocation leaves no store behind.
int mode_store(Ctx* c, ModeStore& store, int n_store, long long stride) {
  if (store.slots == n_store) return SGP_OK;
  const size_t bytes = static_cast<size_t>(n_store) * stride * 8;
  size_t free_b = 0, total_b = 0;
  SGP_CUDA(c, cudaMemGetInfo(&free_b, &total_b));
  if (bytes > free_b + store.buf.cap)
    return fail(c, SGP_E_NOMEM, "the Laplace modes of " + std::to_string(n_store) + " slots need " +
                                    std::to_string(bytes >> 20) + " MiB of device memory, " +
                                    std::to_string((free_b + store.buf.cap) >> 20) + " MiB available");
  store.slots = 0;
  const int rc = ctx_scratch(c, store.buf, bytes);
  if (rc != SGP_OK) return rc;
  SGP_CUDA(c, cudaMemsetAsync(store.buf.p, 0, bytes, c->stream));
  store.slots = n_store;
  return SGP_OK;
}

// The Laplace objective of a slot list with the modes of `store` (n_store mode slots of `stride` modes).  Each slot runs
// the kernel its own set plans (sgp_laplace_nll_any_size's rule on the set's largest expert): the slots are set up in
// the order [on chip | global memory], each family a contiguous range planned for `kind` and launched on its own.  On
// one set this is one family, planned on the whole upload.
int laplace_objective(Ctx* c, Objective kind, const SlotList& L, ExpertSets es, ModeStore& store, int n_store,
                      long long stride, double tol, double* neg_log_z_out, double* grad_out) {
  SGP_CUDA(c, cudaSetDevice(c->device));
  const int n = static_cast<int>(L.sets.size());
  ExpertSet probe = c->ex;
  std::vector<char> on_chip(n);
  for (int s = 0; s < n; ++s) {
    probe.n_max = es.nmax[L.sets[s]];
    on_chip[s] = plan_objective(Objective::kLaplaceAnySize, probe, 1).variant == ObjectiveVariant::kLaplace;
  }
  std::vector<int> pos;
  for (int s = 0; s < n; ++s) if (on_chip[s]) pos.push_back(s);
  const int n_chip = static_cast<int>(pos.size());
  for (int s = 0; s < n; ++s) if (!on_chip[s]) pos.push_back(s);
  ObjectiveSetup o;
  int rc = objective_setup(c, L, std::move(es), o, std::move(pos));
  if (rc != SGP_OK) return rc;
  struct Family { SlotRange r; ObjectivePlan plan; };
  std::vector<Family> fams;
  for (const auto& [s0, s1] : {std::pair<int, int>{0, n_chip}, std::pair<int, int>{n_chip, n}}) {
    if (s0 == s1) continue;
    Family fam{slot_range(c, o, s0, s1), {}};
    fam.plan = plan_objective(kind, fam.r.view, o.hv.kf.n_terms);
    if (fam.plan.variant == ObjectiveVariant::kRefused) return fail(c, SGP_E_BADARG, kLaplaceRefused);
    fams.push_back(fam);
  }
  rc = mode_store(c, store, n_store, stride);   // first use after an upload, or another slot count
  if (rc != SGP_OK) return rc;
  // the global-memory family: one workspace slice per CTA; the grid is bounded by the work items, the resident CTAs and
  // the workspace that fits under kLaplaceGlobalCapBytes and the device's free memory (what this context holds included)
  long long grid = 0;
  for (const Family& fam : fams) {
    if (fam.plan.variant != ObjectiveVariant::kLaplaceGlobal) continue;
    size_t free_b = 0, total_b = 0;
    SGP_CUDA(c, cudaMemGetInfo(&free_b, &total_b));
    const size_t avail = free_b + c->laplace_ws.cap;
    if (fam.plan.cta_ws > avail)
      return fail(c, SGP_E_NOMEM, "the global-memory Laplace kernel needs " + std::to_string(fam.plan.cta_ws >> 20) +
                                      " MiB of device memory for one expert of " + std::to_string(fam.r.view.n_max) +
                                      " points, " + std::to_string(avail >> 20) + " MiB available");
    if (fam.r.view.n_max > kLaplaceGlobalMaxPoints)
      return fail(c, SGP_E_BADARG, "datasetSizeForExpert above " + std::to_string(kLaplaceGlobalMaxPoints) +
                                       " points (32-bit indexing of the per-expert kernel build)");
    const long long resident = static_cast<long long>(laplace_global_ctas_per_sm()) * c->num_sms;
    grid = laplace_global_grid(fam.r.slots.E_max * fam.r.slots.n_slots, resident, fam.plan.cta_ws,
                               std::min(kLaplaceGlobalCapBytes, avail));
    rc = ctx_scratch(c, c->laplace_ws, static_cast<size_t>(grid) * fam.plan.cta_ws);
    if (rc != SGP_OK) return rc;
  }
  c->laplace_path = 0;
  for (Family& fam : fams) {
    SlotRange& r = fam.r;
    r.slots.f = store.buf.as<double>();
    r.slots.f_stride = stride;
    if (fam.plan.variant == ObjectiveVariant::kLaplace) {
      SGP_CUDA(c, launch_laplace(fam.plan, r.view, r.hv, tol, r.slots, r.rows, r.total, r.flags, c->stream));
    } else {
      SGP_CUDA(c, launch_laplace_global(r.view, r.hv, tol, c->laplace_ws.as<double>(), grid, r.slots, r.rows, r.total,
                                        r.flags, c->stream));
      c->laplace_path = 1;
    }
    c->launches += 2;
  }
  return objective_finish(c, o, L.nh, neg_log_z_out, grad_out, 1, SGP_E_NOT_PD, kLaplaceNotPd);
}

// sgp_laplace_nll and _any_size: one slot on the whole upload, the labels as uploaded, the binary modes ex.f
int laplace_nll(Ctx* c, Objective kind, const sgp_kernel_desc* k, const sgp_hyper* hypers, int32_t nh, double tol,
                double* neg_log_z_out, double* grad_out) {
  if (!neg_log_z_out || (nh > 0 && !grad_out) || !(tol > 0.0)) return fail(c, SGP_E_BADARG, "sgp_laplace_nll: bad argument");
  if (tol >= 1.0) return fail(c, SGP_E_SINGULAR, kLaplaceNoIteration);
  return laplace_objective(c, kind, SlotList(k, hypers, nh, 1), whole_upload(c), c->ex_f, 1, c->ex.n, tol, neg_log_z_out,
                           grad_out);
}

// true when the n entries of v are distinct and in [0, bound)
bool distinct_in_range(const int32_t* v, int n, int bound) {
  std::vector<int> sorted(v, v + n);
  std::sort(sorted.begin(), sorted.end());
  return sorted.front() >= 0 && sorted.back() < bound && std::adjacent_find(sorted.begin(), sorted.end()) == sorted.end();
}

int laplace_nll_classes(Ctx* c, Objective kind, int32_t n_classes, const int32_t* classes, int32_t n_eval,
                        const sgp_kernel_desc* kernels, const sgp_hyper* hypers, int32_t nh, double tol,
                        double* neg_log_z_out, double* grad_out) {
  if (!neg_log_z_out || (nh > 0 && !grad_out) || !(tol > 0.0) || !classes)
    return fail(c, SGP_E_BADARG, "sgp_laplace_nll_classes: bad argument");
  if (n_classes < 1 || n_eval < 1 || n_eval > n_classes || n_eval > 65535)
    return fail(c, SGP_E_BADARG, "sgp_laplace_nll_classes: need 1 <= n_eval <= n_classes and n_eval <= 65535");
  if (!distinct_in_range(classes, n_eval, n_classes))
    return fail(c, SGP_E_BADARG, "sgp_laplace_nll_classes: class indices must be distinct and in [0, n_classes)");
  if (tol >= 1.0) return fail(c, SGP_E_SINGULAR, kLaplaceNoIteration);
  SlotList L(kernels, hypers, nh, n_eval);    // class c keeps its modes in mode slot c
  L.cls.assign(classes, classes + n_eval);
  L.modes = L.names = L.cls;
  L.what = "class";
  return laplace_objective(c, kind, L, whole_upload(c), c->ex_fc, n_classes, c->ex.n, tol, neg_log_z_out, grad_out);
}
}  // namespace

int sgp_laplace_nll(sgp_ctx* h, const sgp_kernel_desc* k, const sgp_hyper* hypers, int32_t nh, double tol,
                    double* neg_log_z_out, double* grad_out) {
  Ctx* c = reinterpret_cast<Ctx*>(h);
  if (!c) return SGP_E_BADARG;
  return laplace_nll(c, Objective::kLaplace, k, hypers, nh, tol, neg_log_z_out, grad_out);
}

int sgp_laplace_nll_any_size(sgp_ctx* h, const sgp_kernel_desc* k, const sgp_hyper* hypers, int32_t nh, double tol,
                             double* neg_log_z_out, double* grad_out) {
  Ctx* c = reinterpret_cast<Ctx*>(h);
  if (!c) return SGP_E_BADARG;
  return laplace_nll(c, Objective::kLaplaceAnySize, k, hypers, nh, tol, neg_log_z_out, grad_out);
}

int sgp_laplace_nll_classes(sgp_ctx* h, int32_t n_classes, const int32_t* classes, int32_t n_eval,
                            const sgp_kernel_desc* kernels, const sgp_hyper* hypers, int32_t nh, double tol,
                            double* neg_log_z_out, double* grad_out) {
  Ctx* c = reinterpret_cast<Ctx*>(h);
  if (!c) return SGP_E_BADARG;
  return laplace_nll_classes(c, Objective::kLaplace, n_classes, classes, n_eval, kernels, hypers, nh, tol, neg_log_z_out,
                             grad_out);
}

int sgp_laplace_nll_classes_any_size(sgp_ctx* h, int32_t n_classes, const int32_t* classes, int32_t n_eval,
                                     const sgp_kernel_desc* kernels, const sgp_hyper* hypers, int32_t nh, double tol,
                                     double* neg_log_z_out, double* grad_out) {
  Ctx* c = reinterpret_cast<Ctx*>(h);
  if (!c) return SGP_E_BADARG;
  return laplace_nll_classes(c, Objective::kLaplaceAnySize, n_classes, classes, n_eval, kernels, hypers, nh, tol,
                             neg_log_z_out, grad_out);
}

int sgp_laplace_nll_slots_any_size(sgp_ctx* h, int32_t n_mode_slots, const int32_t* mode_slots, const int32_t* classes,
                                   int32_t n_eval, const sgp_kernel_desc* kernels, const sgp_hyper* hypers, int32_t nh,
                                   double tol, double* neg_log_z_out, double* grad_out) {
  Ctx* c = reinterpret_cast<Ctx*>(h);
  if (!c) return SGP_E_BADARG;
  if (!neg_log_z_out || (nh > 0 && !grad_out) || !(tol > 0.0) || !mode_slots || !classes)
    return fail(c, SGP_E_BADARG, "sgp_laplace_nll_slots_any_size: bad argument");
  if (n_mode_slots < 1 || n_eval < 1 || n_eval > n_mode_slots || n_eval > 65535)
    return fail(c, SGP_E_BADARG, "sgp_laplace_nll_slots_any_size: need 1 <= n_eval <= n_mode_slots and n_eval <= 65535");
  if (!distinct_in_range(mode_slots, n_eval, n_mode_slots))
    return fail(c, SGP_E_BADARG, "sgp_laplace_nll_slots_any_size: mode slots must be distinct and in [0, n_mode_slots)");
  if (*std::min_element(classes, classes + n_eval) < 0)
    return fail(c, SGP_E_BADARG, "sgp_laplace_nll_slots_any_size: class indices must be >= 0");
  if (tol >= 1.0) return fail(c, SGP_E_SINGULAR, kLaplaceNoIteration);
  SlotList L(kernels, hypers, nh, n_eval);
  L.cls.assign(classes, classes + n_eval);
  L.modes.assign(mode_slots, mode_slots + n_eval);
  L.names = L.modes;
  L.what = "mode slot";
  return laplace_objective(c, Objective::kLaplaceAnySize, L, whole_upload(c), c->ex_fm, n_mode_slots, c->ex.n, tol,
                           neg_log_z_out, grad_out);
}

namespace {
// rows of the largest training set of the fold upload: the stride of the fold-slot mode store
long long fold_rows_max(const Ctx* c) {
  long long m = 0;
  for (size_t k = 0; k + 1 < c->fold_row0.size(); ++k) m = std::max(m, c->fold_row0[k + 1] - c->fold_row0[k]);
  return m;
}
}  // namespace

int sgp_laplace_nll_fold_slots_any_size(sgp_ctx* h, int32_t n_mode_slots, const int32_t* mode_slots,
                                        const int32_t* sets, const int32_t* classes, int32_t n_eval,
                                        const sgp_kernel_desc* kernels, const sgp_hyper* hypers, int32_t nh, double tol,
                                        double* neg_log_z_out, double* grad_out) {
  Ctx* c = reinterpret_cast<Ctx*>(h);
  if (!c) return SGP_E_BADARG;
  const std::string fn = "sgp_laplace_nll_fold_slots_any_size";
  if (!neg_log_z_out || (nh > 0 && !grad_out) || !(tol > 0.0) || !mode_slots || !sets || !classes)
    return fail(c, SGP_E_BADARG, fn + ": bad argument");
  if (c->ex.E == 0 || c->fold_first.empty())
    return fail(c, SGP_E_STATE, "sgp_experts_upload_folds should have been called first");
  if (n_mode_slots < 1 || n_eval < 1 || n_eval > n_mode_slots || n_eval > 65535)
    return fail(c, SGP_E_BADARG, fn + ": need 1 <= n_eval <= n_mode_slots and n_eval <= 65535");
  if (!distinct_in_range(mode_slots, n_eval, n_mode_slots))
    return fail(c, SGP_E_BADARG, fn + ": mode slots must be distinct and in [0, n_mode_slots)");
  if (*std::min_element(classes, classes + n_eval) < 0) return fail(c, SGP_E_BADARG, fn + ": class indices must be >= 0");
  const int n_sets = static_cast<int>(c->fold_first.size()) - 1;
  int n_max = 0;
  for (int s = 0; s < n_eval; ++s) {
    if (sets[s] < 0 || sets[s] >= n_sets)
      return fail(c, SGP_E_BADARG, fn + ": set index " + std::to_string(sets[s]) + " outside [0, n_folds)");
    n_max = std::max(n_max, c->fold_nmax[sets[s]]);
  }
  if (n_max > kLaplaceGlobalMaxPoints)
    return fail(c, SGP_E_BADARG, "datasetSizeForExpert above " + std::to_string(kLaplaceGlobalMaxPoints) +
                                     " points (32-bit indexing of the per-expert kernel build)");
  if (tol >= 1.0) return fail(c, SGP_E_SINGULAR, kLaplaceNoIteration);
  if (!kernels || nh < 0 || (nh > 0 && !hypers)) return fail(c, SGP_E_BADARG, fn + ": null argument");
  SlotList L(kernels, hypers, nh, n_eval);
  L.sets.assign(sets, sets + n_eval);
  L.cls.assign(classes, classes + n_eval);
  L.modes.assign(mode_slots, mode_slots + n_eval);
  L.names = L.modes;
  L.what = "mode slot";
  return laplace_objective(c, Objective::kLaplaceAnySize, L, fold_sets(c), c->ex_ffm, n_mode_slots, fold_rows_max(c),
                           tol, neg_log_z_out, grad_out);
}

namespace {
constexpr int kModesFold = -1;   // the fold-slot store (sgp_experts_get_f_fold_*), next to sgp.h's SGP_MODES_*

// The modes a getter reads: rows modes of `experts` experts from f.
struct Modes {
  const double* f;
  long long rows, experts;
};

// The modes of store SGP_MODES_BINARY (index ignored), _CLASS or _SLOT (class or mode slot `index`), or kModesFold (mode
// slot `index` on fold set `set`), after the getters' refusals in their order; fn names the getter.
int find_modes(Ctx* c, int store, int index, int set, const void* out, const char* fn, Modes& m) {
  const bool fold = store == kModesFold;
  if (c->ex.E == 0 || (fold && c->fold_first.empty()) || !out)
    return fail(c, SGP_E_STATE, fold ? "sgp_experts_upload_folds should have been called first"
                                     : "sgp_experts_upload should have been called first");
  m = {c->ex.f, c->ex.n, c->ex.E};
  if (store == SGP_MODES_BINARY) return SGP_OK;
  const ModeStore& s = fold ? c->ex_ffm : store == SGP_MODES_CLASS ? c->ex_fc : c->ex_fm;
  if (s.slots == 0)
    return fail(c, SGP_E_STATE, fold ? "no fold slot modes: sgp_laplace_nll_fold_slots_any_size has not run since the upload"
                                : store == SGP_MODES_CLASS ? "no class modes: sgp_laplace_nll_classes has not run since the upload"
                                : "no slot modes: sgp_laplace_nll_slots_any_size has not run since the upload");
  long long stride = c->ex.n;
  if (fold) {
    if (set < 0 || set >= static_cast<int>(c->fold_first.size()) - 1)
      return fail(c, SGP_E_BADARG, std::string(fn) + ": set index outside [0, n_folds)");
    stride = fold_rows_max(c);
    m.rows = c->fold_row0[set + 1] - c->fold_row0[set];
    m.experts = c->fold_first[set + 1] - c->fold_first[set];
  }
  if (index < 0 || index >= s.slots)
    return fail(c, SGP_E_BADARG, std::string(fn) + (store == SGP_MODES_CLASS ? ": class index out of range"
                                                                           : ": mode slot outside [0, n_mode_slots)"));
  m.f = s.buf.as<double>() + static_cast<size_t>(index) * stride;
  return SGP_OK;
}

// the host getters: the modes in the experts' packed order
int copy_modes(Ctx* c, int store, int index, int set, double* f_out, const char* fn) {
  Modes m;
  const int rc = find_modes(c, store, index, set, f_out, fn, m);
  if (rc != SGP_OK) return rc;
  SGP_CUDA(c, cudaSetDevice(c->device));
  SGP_CUDA(c, cudaMemcpyAsync(f_out, m.f, static_cast<size_t>(m.rows) * 8, cudaMemcpyDeviceToHost, c->stream));
  SGP_CUDA(c, cudaStreamSynchronize(c->stream));
  return SGP_OK;
}

// the _rows_device getters: the modes ungrouped into row order (a grouped upload, or a fold set, which is grouped as one)
int ungroup_modes(Ctx* c, const Modes& m, double* dF_out, const char* fn) {
  SGP_CUDA(c, cudaSetDevice(c->device));
  const int rc = device_ptr_ok(c, dF_out, fn, "f_out");
  if (rc != SGP_OK) return rc;
  SGP_CUDA(c, launch_ungroup_experts(dF_out, m.f, m.rows, m.experts, c->stream));
  c->launches += 1;
  SGP_CUDA(c, cudaStreamSynchronize(c->stream));
  return SGP_OK;
}
}  // namespace

int sgp_experts_get_f_fold_slot(sgp_ctx* h, int32_t set, int32_t mode_slot, double* f_out) {
  Ctx* c = reinterpret_cast<Ctx*>(h);
  if (!c) return SGP_E_BADARG;
  return copy_modes(c, kModesFold, mode_slot, set, f_out, "sgp_experts_get_f_fold_slot");
}

int sgp_experts_get_f_fold_rows_device(sgp_ctx* h, int32_t set, int32_t mode_slot, double* dF_out) {
  Ctx* c = reinterpret_cast<Ctx*>(h);
  if (!c) return SGP_E_BADARG;
  const char* fn = "sgp_experts_get_f_fold_rows_device";
  Modes m;
  const int rc = find_modes(c, kModesFold, mode_slot, set, dF_out, fn, m);
  return rc != SGP_OK ? rc : ungroup_modes(c, m, dF_out, fn);
}

int sgp_experts_get_f_slot(sgp_ctx* h, int32_t mode_slot, double* f_out) {
  Ctx* c = reinterpret_cast<Ctx*>(h);
  if (!c) return SGP_E_BADARG;
  return copy_modes(c, SGP_MODES_SLOT, mode_slot, 0, f_out, "sgp_experts_get_f_slot");
}

int sgp_experts_get_f_class(sgp_ctx* h, int32_t cls, double* f_out) {
  Ctx* c = reinterpret_cast<Ctx*>(h);
  if (!c) return SGP_E_BADARG;
  return copy_modes(c, SGP_MODES_CLASS, cls, 0, f_out, "sgp_experts_get_f_class");
}

int sgp_experts_get_f(sgp_ctx* h, double* f_out) {
  Ctx* c = reinterpret_cast<Ctx*>(h);
  if (!c) return SGP_E_BADARG;
  return copy_modes(c, SGP_MODES_BINARY, 0, 0, f_out, "sgp_experts_get_f");
}

int sgp_experts_get_f_rows_device(sgp_ctx* h, int32_t store, int32_t index, double* dF_out) {
  Ctx* c = reinterpret_cast<Ctx*>(h);
  if (!c) return SGP_E_BADARG;
  const char* fn = "sgp_experts_get_f_rows_device";
  if (store != SGP_MODES_BINARY && store != SGP_MODES_CLASS && store != SGP_MODES_SLOT)
    return fail(c, SGP_E_BADARG, std::string(fn) + ": unknown mode store");
  Modes m;
  const int rc = find_modes(c, store, index, 0, dF_out, fn, m);
  if (rc != SGP_OK) return rc;
  if (!c->ex_grouped)
    return fail(c, SGP_E_STATE, "sgp_experts_get_f_rows_device: the experts were not uploaded by sgp_experts_upload_grouped "
                                "or its _device form, so their rows have no row order");
  return ungroup_modes(c, m, dF_out, fn);
}

int sgp_last_path(const sgp_ctx* h) {
  const Ctx* c = reinterpret_cast<const Ctx*>(h);
  return c ? c->last_path : -1;
}

int sgp_last_bcm_path(const sgp_ctx* h) {
  const Ctx* c = reinterpret_cast<const Ctx*>(h);
  return c ? (c->bcm_general ? 1 : 0) : -1;
}

int sgp_last_laplace_path(const sgp_ctx* h) {
  const Ctx* c = reinterpret_cast<const Ctx*>(h);
  return c ? c->laplace_path : -1;
}

int sgp_last_tail_path(const sgp_ctx* h) {
  const Ctx* c = reinterpret_cast<const Ctx*>(h);
  if (!c || !c->has_magic_run) return -1;
  return c->tail_fast ? 1 : 0;
}

int sgp_debug_i8_tile(sgp_ctx* h, float* T_out, uint32_t* w_out) {
  Ctx* c = reinterpret_cast<Ctx*>(h);
  if (!c) return SGP_E_BADARG;
  SGP_CUDA(c, cudaSetDevice(c->device));
  if (!c->dbgW.p) {   // arm: the next I8 launches dump the first distance tile of CTA (0,0)
    int rc = ctx_scratch(c, c->dbgT, 128 * 64 * 4);
    if (rc == SGP_OK) rc = ctx_scratch(c, c->dbgW, 128 * 64 * 4);
    if (rc != SGP_OK) return rc;
    SGP_CUDA(c, cudaMemset(c->dbgT.p, 0, 128 * 64 * 4));
    SGP_CUDA(c, cudaMemset(c->dbgW.p, 0, 128 * 64 * 4));
  }
  SGP_CUDA(c, cudaStreamSynchronize(c->stream));
  if (T_out) SGP_CUDA(c, cudaMemcpy(T_out, c->dbgT.p, 128 * 64 * 4, cudaMemcpyDeviceToHost));
  if (w_out) SGP_CUDA(c, cudaMemcpy(w_out, c->dbgW.p, 128 * 64 * 4, cudaMemcpyDeviceToHost));
  return SGP_OK;
}

int sgp_event_record(sgp_ctx* h, int slot) {
  Ctx* c = reinterpret_cast<Ctx*>(h);
  if (!c) return SGP_E_BADARG;
  if (slot < 0 || slot >= 8) return fail(c, SGP_E_BADARG, "event slot out of range");
  SGP_CUDA(c, cudaSetDevice(c->device));
  if (!c->user_events[slot]) SGP_CUDA(c, cudaEventCreate(&c->user_events[slot]));
  SGP_CUDA(c, cudaEventRecord(c->user_events[slot], c->stream));
  return SGP_OK;
}

int sgp_event_elapsed_ms(sgp_ctx* h, int a, int b, double* ms) {
  Ctx* c = reinterpret_cast<Ctx*>(h);
  if (!c) return SGP_E_BADARG;
  if (a < 0 || a >= 8 || b < 0 || b >= 8 || !ms || !c->user_events[a] || !c->user_events[b])
    return fail(c, SGP_E_BADARG, "bad event slots");
  SGP_CUDA(c, cudaSetDevice(c->device));
  SGP_CUDA(c, cudaEventSynchronize(c->user_events[b]));
  float f = 0.f;
  SGP_CUDA(c, cudaEventElapsedTime(&f, c->user_events[a], c->user_events[b]));
  *ms = f;
  return SGP_OK;
}

// One sweep launch over n device-resident points (prep of the fp16 operand images + the sweep kernel).  The sweep's
// points are not statistics points: their range bits go to the sweep's own status word (dI8Flags[2]) and their norms
// to no budget, so a sweep inside a begin..finish window leaves the window's status alone.
static int sweep_device(Ctx* c, const void* dX, int x_is_f32, long long n, float* dK) {
  int rc = ctx_scratch(c, c->i8_xt_ws, i8_points_scratch_bytes(n, i8_nchunks(c->d)));
  if (rc == SGP_OK) rc = ctx_scratch(c, c->i8_ys_ws, static_cast<size_t>((n + 63) / 64) * 64 * sizeof(float));
  if (rc != SGP_OK) return rc;
  const double* scale = c->dI8Scale.as<double>();
  SGP_CUDA(c, launch_i8_prep_points(c->i8_xt_ws.as<uint8_t>(), c->i8_ys_ws.as<float>(), dX, x_is_f32, nullptr, n, c->d,
                                    scale, scale + static_cast<size_t>(kMaxTerms) * c->dpad, c->dI8Flags.as<int>() + 2,
                                    nullptr, nullptr, c->stream));
  SGP_CUDA(c, launch_kmn_sweep(c->i8_xt_ws.as<uint8_t>(), c->dI8Zt.as<uint8_t>(), n, c->d, c->m, c->m_pad, c->num_sms,
                               c->kf.scale[0], dK, c->stream));
  c->launches += 2;
  return SGP_OK;
}

int sgp_kmn_sweep_device(sgp_ctx* h, const void* dX, int32_t x_is_f32, int64_t n, float* dK_out) {
  Ctx* c = reinterpret_cast<Ctx*>(h);
  if (!c) return SGP_E_BADARG;
  if (!c->begun) return fail(c, SGP_E_STATE, "setTrainingVectors method should have been called first");
  if (n <= 0 || !dX || !dK_out) return fail(c, SGP_E_BADARG, "null argument");
  if (!c->i8_ok) return fail(c, SGP_E_BADARG, "sgp_kmn_sweep needs a kernel with exactly one non-Eye term and d <= 32");
  SGP_CUDA(c, cudaSetDevice(c->device));
  return sweep_device(c, dX, x_is_f32, n, dK_out);
}

int sgp_kmn_sweep(sgp_ctx* h, const void* X, int32_t x_is_f32, int64_t n, float* K_out) {
  Ctx* c = reinterpret_cast<Ctx*>(h);
  if (!c) return SGP_E_BADARG;
  if (!c->begun) return fail(c, SGP_E_STATE, "setTrainingVectors method should have been called first");
  if (n <= 0 || !X || !K_out) return fail(c, SGP_E_BADARG, "null argument");
  if (!c->i8_ok) return fail(c, SGP_E_BADARG, "sgp_kmn_sweep needs a kernel with exactly one non-Eye term and d <= 32");
  SGP_CUDA(c, cudaSetDevice(c->device));
  const size_t esz = x_is_f32 ? 4 : 8;
  const long long chunk = 65536;
  const long long cn0 = n < chunk ? n : chunk;
  int rc = ctx_scratch(c, c->sweep_ws, static_cast<size_t>(cn0) * c->d * esz + static_cast<size_t>(cn0) * c->m * sizeof(float));
  if (rc != SGP_OK) return rc;
  float* dK = static_cast<float*>(c->sweep_ws.p);
  void* dX = dK + static_cast<size_t>(cn0) * c->m;
  // this call's status: the active set's range bit from begin, then the bits of this call's points
  SGP_CUDA(c, cudaMemcpyAsync(c->dI8Flags.as<int>() + 2, c->dI8Flags.as<int>() + 1, sizeof(int), cudaMemcpyDeviceToDevice, c->stream));
  for (long long p0 = 0; p0 < n; p0 += chunk) {
    const long long cn = (n - p0 < chunk) ? (n - p0) : chunk;
    SGP_CUDA(c, cudaMemcpyAsync(dX, static_cast<const char*>(X) + static_cast<size_t>(p0) * c->d * esz,
                                static_cast<size_t>(cn) * c->d * esz, cudaMemcpyHostToDevice, c->stream));
    rc = sweep_device(c, dX, x_is_f32, cn, dK);
    if (rc != SGP_OK) return rc;
    SGP_CUDA(c, cudaMemcpyAsync(K_out + static_cast<size_t>(p0) * c->m, dK, static_cast<size_t>(cn) * c->m * sizeof(float),
                                cudaMemcpyDeviceToHost, c->stream));
    SGP_CUDA(c, cudaStreamSynchronize(c->stream));
  }
  int flags = 0;
  SGP_CUDA(c, cudaMemcpyAsync(&flags, c->dI8Flags.as<int>() + 2, sizeof(int), cudaMemcpyDeviceToHost, c->stream));
  SGP_CUDA(c, cudaStreamSynchronize(c->stream));
  if (flags & 1)
    return fail(c, SGP_E_RANGE, "scaled squared norms exceed the operand range of the tensor-core distance contraction (4096); "
                                "use sgp_cross_kernel");
  return SGP_OK;
}

namespace {
int greedy_active_set(Ctx* c, bool on_device, const sgp_kernel_desc* k, const double* X, const double* y, int64_t n,
                      int32_t d, int64_t n_experts, int64_t first_index, int32_t m_target, int64_t* indices_out,
                      const char* entry) {
  if (!k || !X || !y || !indices_out || n <= 0 || d <= 0 || m_target <= 0 || k->n_terms <= 0 || !k->terms)
    return fail(c, SGP_E_BADARG, std::string(entry) + ": null or empty argument");
  if (n_experts <= 0) return fail(c, SGP_E_BADARG, "numberOfExperts == 0 (N < datasetSizeForExpert / 2)");
  if (first_index < 0 || first_index >= n) return fail(c, SGP_E_BADARG, "first_index out of range");
  if (n > 2147483647LL) return fail(c, SGP_E_BADARG, std::string(entry) + ": n too large for one device");
  SGP_CUDA(c, cudaSetDevice(c->device));
  if (on_device) {
    int rc = device_ptr_ok(c, X, entry, "X");
    if (rc == SGP_OK) rc = device_ptr_ok(c, y, entry, "y");
    if (rc != SGP_OK) return rc;
  }
  KernelFlat kf;
  std::vector<double> beta;
  const int rc = flatten_kernel(c, k, d, d, kf, beta, nullptr);
  if (rc != SGP_OK) return rc;
  static_assert(sizeof(long long) == sizeof(int64_t), "index type");
  return run_greedy(c, kf, beta, X, y, on_device, n, d, n_experts, first_index, m_target,
                    reinterpret_cast<long long*>(indices_out));
}

// sgp_kmeans_sharded and its _device form: every refusal is taken on every rank together (the layout table and the
// local argument verdicts are all-reduced before anything else)
int kmeans_sharded(Ctx* c, bool on_device, const void* X, int32_t x_is_f32, int64_t n, int64_t offset, int64_t n_total,
                   int32_t d, int32_t k, int32_t max_iter, double tol, int64_t seed, const double* init_centers,
                   double* centers_out, int32_t* k_out, int32_t* labels_out, int32_t* iterations_out, double* cost_out,
                   const char* entry) {
  if (!centers_out || !k_out || !iterations_out || !cost_out)
    return fail(c, SGP_E_BADARG, std::string(entry) + ": null argument");
  if (k < 2) return fail(c, SGP_E_BADARG, "requirement failed: k must be > 1");
  if (max_iter < 0) return fail(c, SGP_E_BADARG, "requirement failed: maxIter must be >= 0");
  if (!(tol >= 0.0)) return fail(c, SGP_E_BADARG, "requirement failed: tol must be >= 0");
  if (d < 1) return fail(c, SGP_E_BADARG, std::string(entry) + ": no features");
  SGP_CUDA(c, cudaSetDevice(c->device));
  int local_bad = (n < 0 || n > 2147483647LL || offset < 0 || (n > 0 && !X)) ? 1 : 0;
  if (!local_bad && n > 0 && on_device && device_ptr_ok(c, X, entry, "X") != SGP_OK) local_bad = 2;
  if (init_centers)
    for (size_t i = 0; i < static_cast<size_t>(k) * d; ++i)
      if (!std::isfinite(init_centers[i]))
        return fail(c, SGP_E_BADARG, std::string(entry) + ": initial centres contain NaN or infinity");
  // the layout table [rank][n, offset, verdict], summed over the ranks: every rank checks every rank's entry
  const int R = c->comm ? c->nranks : 1, me = c->comm ? c->rank : 0;
  std::vector<long long> table(static_cast<size_t>(R) * 3, 0);
  table[static_cast<size_t>(me) * 3] = n;
  table[static_cast<size_t>(me) * 3 + 1] = offset;
  table[static_cast<size_t>(me) * 3 + 2] = local_bad;
  int rc = ctx_scratch(c, c->kmeans_comm_ws, table.size() * 8);
  if (rc != SGP_OK) return rc;
  SGP_CUDA(c, cudaMemcpyAsync(c->kmeans_comm_ws.p, table.data(), table.size() * 8, cudaMemcpyHostToDevice, c->stream));
  rc = comm_sum(c, c->kmeans_comm_ws.p, table.size(), ncclInt64);
  if (rc != SGP_OK) return rc;
  SGP_CUDA(c, cudaMemcpyAsync(table.data(), c->kmeans_comm_ws.p, table.size() * 8, cudaMemcpyDeviceToHost, c->stream));
  SGP_CUDA(c, cudaStreamSynchronize(c->stream));
  long long next = 0;
  for (int r = 0; r < R; ++r) {
    const long long* t = &table[static_cast<size_t>(r) * 3];
    if (t[2] == 2) return fail(c, SGP_E_BADARG, std::string(entry) + ": X of rank " + std::to_string(r) +
                                                    " is not device memory on its context's device");
    if (t[2] != 0 || t[1] != next)
      return fail(c, SGP_E_BADARG, std::string(entry) + ": rank " + std::to_string(r) + " holds rows [" +
                                       std::to_string(t[1]) + ", +" + std::to_string(t[0]) + "); the ranks' rows must " +
                                       "follow each other in rank order from 0");
    next += t[0];
  }
  if (next != n_total || n_total < 1)
    return fail(c, SGP_E_BADARG, std::string(entry) + ": the ranks hold " + std::to_string(next) + " rows, n_total is " +
                                     std::to_string(n_total));
  return run_kmeans_sharded(c, X, x_is_f32, on_device, n, offset, n_total, d, k, max_iter, tol,
                            static_cast<uint64_t>(seed), init_centers, centers_out, k_out, labels_out, iterations_out,
                            cost_out);
}

int kmeans(Ctx* c, bool on_device, const void* X, int32_t x_is_f32, int64_t n, int32_t d, int32_t k, int32_t max_iter,
           double tol, int64_t seed, const double* init_centers, double* centers_out, int32_t* k_out, int32_t* labels_out,
           int32_t* iterations_out, double* cost_out, const char* entry) {
  if (!X || !centers_out || !k_out || !iterations_out || !cost_out)
    return fail(c, SGP_E_BADARG, std::string(entry) + ": null argument");
  if (k < 2) return fail(c, SGP_E_BADARG, "requirement failed: k must be > 1");
  if (max_iter < 0) return fail(c, SGP_E_BADARG, "requirement failed: maxIter must be >= 0");
  if (!(tol >= 0.0)) return fail(c, SGP_E_BADARG, "requirement failed: tol must be >= 0");
  if (n < 1 || d < 1) return fail(c, SGP_E_BADARG, std::string(entry) + ": no points or no features");
  if (n > 2147483647LL) return fail(c, SGP_E_BADARG, std::string(entry) + ": n too large for one device");
  if (init_centers)
    for (size_t i = 0; i < static_cast<size_t>(k) * d; ++i)
      if (!std::isfinite(init_centers[i]))
        return fail(c, SGP_E_BADARG, std::string(entry) + ": initial centres contain NaN or infinity");
  SGP_CUDA(c, cudaSetDevice(c->device));
  if (on_device) {
    const int rc = device_ptr_ok(c, X, entry, "X");
    if (rc != SGP_OK) return rc;
  }
  static_assert(sizeof(int) == sizeof(int32_t), "label type");
  return run_kmeans(c, X, x_is_f32, on_device, n, d, k, max_iter, tol, static_cast<uint64_t>(seed), init_centers,
                    centers_out, k_out, labels_out, iterations_out, cost_out);
}
}  // namespace

int sgp_greedy_active_set(sgp_ctx* h, const sgp_kernel_desc* k, const double* X, const double* y, int64_t n, int32_t d,
                          int64_t n_experts, int64_t first_index, int32_t m_target, int64_t* indices_out) {
  Ctx* c = reinterpret_cast<Ctx*>(h);
  if (!c) return SGP_E_BADARG;
  return greedy_active_set(c, false, k, X, y, n, d, n_experts, first_index, m_target, indices_out, "sgp_greedy_active_set");
}

int sgp_greedy_active_set_device(sgp_ctx* h, const sgp_kernel_desc* k, const double* dX, const double* dy, int64_t n,
                                 int32_t d, int64_t n_experts, int64_t first_index, int32_t m_target, int64_t* indices_out) {
  Ctx* c = reinterpret_cast<Ctx*>(h);
  if (!c) return SGP_E_BADARG;
  return greedy_active_set(c, true, k, dX, dy, n, d, n_experts, first_index, m_target, indices_out,
                           "sgp_greedy_active_set_device");
}

int sgp_kmeans(sgp_ctx* h, const void* X, int32_t x_is_f32, int64_t n, int32_t d, int32_t k, int32_t max_iter, double tol,
               int64_t seed, const double* init_centers, double* centers_out, int32_t* k_out, int32_t* labels_out,
               int32_t* iterations_out, double* cost_out) {
  Ctx* c = reinterpret_cast<Ctx*>(h);
  if (!c) return SGP_E_BADARG;
  return kmeans(c, false, X, x_is_f32, n, d, k, max_iter, tol, seed, init_centers, centers_out, k_out, labels_out,
                iterations_out, cost_out, "sgp_kmeans");
}

int sgp_kmeans_device(sgp_ctx* h, const void* dX, int32_t x_is_f32, int64_t n, int32_t d, int32_t k, int32_t max_iter,
                      double tol, int64_t seed, const double* init_centers, double* centers_out, int32_t* k_out,
                      int32_t* labels_out, int32_t* iterations_out, double* cost_out) {
  Ctx* c = reinterpret_cast<Ctx*>(h);
  if (!c) return SGP_E_BADARG;
  return kmeans(c, true, dX, x_is_f32, n, d, k, max_iter, tol, seed, init_centers, centers_out, k_out, labels_out,
                iterations_out, cost_out, "sgp_kmeans_device");
}

int sgp_kmeans_sharded(sgp_ctx* h, const void* X, int32_t x_is_f32, int64_t n, int64_t offset, int64_t n_total, int32_t d,
                       int32_t k, int32_t max_iter, double tol, int64_t seed, const double* init_centers,
                       double* centers_out, int32_t* k_out, int32_t* labels_out, int32_t* iterations_out,
                       double* cost_out) {
  Ctx* c = reinterpret_cast<Ctx*>(h);
  if (!c) return SGP_E_BADARG;
  return kmeans_sharded(c, false, X, x_is_f32, n, offset, n_total, d, k, max_iter, tol, seed, init_centers, centers_out,
                        k_out, labels_out, iterations_out, cost_out, "sgp_kmeans_sharded");
}

int sgp_kmeans_sharded_device(sgp_ctx* h, const void* dX, int32_t x_is_f32, int64_t n, int64_t offset, int64_t n_total,
                              int32_t d, int32_t k, int32_t max_iter, double tol, int64_t seed,
                              const double* init_centers, double* centers_out, int32_t* k_out, int32_t* labels_out,
                              int32_t* iterations_out, double* cost_out) {
  Ctx* c = reinterpret_cast<Ctx*>(h);
  if (!c) return SGP_E_BADARG;
  return kmeans_sharded(c, true, dX, x_is_f32, n, offset, n_total, d, k, max_iter, tol, seed, init_centers, centers_out,
                        k_out, labels_out, iterations_out, cost_out, "sgp_kmeans_sharded_device");
}

int sgp_cross_kernel(sgp_ctx* h, const double* X, int64_t n, double* K_out) {
  Ctx* c = reinterpret_cast<Ctx*>(h);
  if (!c) return SGP_E_BADARG;
  if (!c->begun) return fail(c, SGP_E_STATE, "setTrainingVectors method should have been called first");
  if (n <= 0 || !X || !K_out) return fail(c, SGP_E_BADARG, "null argument");
  if (n > 65535 * 8) return fail(c, SGP_E_BADARG, "sgp_cross_kernel: n too large for one call");
  SGP_CUDA(c, cudaSetDevice(c->device));
  int rc = ctx_scratch(c, c->cross_ws, (static_cast<size_t>(n) * c->d + static_cast<size_t>(n) * c->m) * 8);
  if (rc != SGP_OK) return rc;
  double* dX = static_cast<double*>(c->cross_ws.p);
  double* dK = dX + static_cast<size_t>(n) * c->d;
  SGP_CUDA(c, cudaMemcpyAsync(dX, X, static_cast<size_t>(n) * c->d * 8, cudaMemcpyHostToDevice, c->stream));
  if (c->kf.n_terms > 0) {
    SGP_CUDA(c, launch_cross_kernel(dK, dX, c->dZs.as<double>(), c->dBeta.as<double>(), c->kf, n, c->d, c->dpad, c->m,
                                    c->m_pad, c->stream));
    c->launches += 1;
  } else {
    SGP_CUDA(c, cudaMemsetAsync(dK, 0, static_cast<size_t>(n) * c->m * 8, c->stream));
  }
  SGP_CUDA(c, cudaMemcpyAsync(K_out, dK, static_cast<size_t>(n) * c->m * 8, cudaMemcpyDeviceToHost, c->stream));
  SGP_CUDA(c, cudaStreamSynchronize(c->stream));
  return SGP_OK;
}

namespace {
// One sgp_kernel_eval* call after its checks: the launch arguments (pointers into the descriptor tables still unset) and
// the tables themselves, [beta (n_terms x d) | scale coefficients (n_scale x (kMaxTerms + 1))] doubles then
// [ARD indices (n_terms x d) | scale indices (n_scale)] ints.
struct KernelEvalSetup {
  KernelEvalArgs a{};
  std::vector<char> tables;
  size_t n_dbl = 0;
  int nh = 0;            // matrices of dK written (0 without dK_out)
};

// Every refusal of both entries, before any allocation or launch.  The descriptors must be those of the kernel: one
// ARD_BETA per feature of every ARD term and one RBF_SIGMA per RBF term, each carrying the term's own value, plus any
// number of SCALE descriptors (trainable scalars), in any order.
int kernel_eval_setup(Ctx* c, const char* entry, const sgp_kernel_desc* k, const sgp_hyper* hypers, int32_t nh,
                      const void* A, int64_t n, const double* B, int32_t m, int32_t d, int32_t mode, const double* K_out,
                      const double* dK_out, KernelEvalSetup& o) {
  const std::string fn(entry);
  if (!k || k->n_terms <= 0 || !k->terms) return fail(c, SGP_E_BADARG, fn + ": a kernel with no terms");
  if (n < 1 || m < 1 || d < 1) return fail(c, SGP_E_BADARG, fn + ": n, m and d must be >= 1");
  if (!A || !K_out) return fail(c, SGP_E_BADARG, fn + ": null argument");
  if (mode != SGP_KEVAL_CROSS && mode != SGP_KEVAL_TRAINING) return fail(c, SGP_E_BADARG, fn + ": unknown mode");
  if (mode == SGP_KEVAL_CROSS && !B) return fail(c, SGP_E_BADARG, fn + ": CROSS needs the training vectors B");
  if (mode == SGP_KEVAL_TRAINING && (B || m != n))
    return fail(c, SGP_E_BADARG, fn + ": TRAINING takes no B and m == n");
  if (nh < 0 || (nh > 0 && !hypers)) return fail(c, SGP_E_BADARG, fn + ": null hyper-parameter descriptors");
  const int n_mat = 1 + (dK_out ? nh : 0);
  if (static_cast<unsigned __int128>(n_mat) * static_cast<unsigned __int128>(n) * static_cast<unsigned __int128>(m) * 8 >
      static_cast<unsigned __int128>(INT64_MAX))
    return fail(c, SGP_E_BADARG, fn + ": the output exceeds 64-bit sizes");
  KernelFlat kf;
  std::vector<double> beta;
  std::vector<int> flat_of;
  int rc = flatten_kernel(c, k, d, d, kf, beta, &flat_of);
  if (rc != SGP_OK) return rc;
  const int T = kf.n_terms;
  std::vector<int> ard_h(static_cast<size_t>(T) * d, -1), scale_h;
  std::vector<double> scale_coef;
  KernelEvalArgs& a = o.a;
  for (int t = 0; t < kMaxTerms; ++t) { a.rbf_h[t] = -1; a.sigma3[t] = 1.0; }
  const std::string mismatch = fn + ": the hyper-parameter descriptors do not match the kernel";
  for (int i = 0; i < nh; ++i) {
    const sgp_hyper& hp = hypers[i];
    if (hp.kind == SGP_HYPER_SCALE) {
      if (!hp.coef) return fail(c, SGP_E_BADARG, fn + ": SCALE hyper-parameter without coef");
      scale_h.push_back(i);
      scale_coef.resize(scale_coef.size() + kMaxTerms + 1, 0.0);
      double* cf = scale_coef.data() + scale_coef.size() - (kMaxTerms + 1);
      for (int t = 0; t < k->n_terms; ++t) cf[flat_of[t] >= 0 ? flat_of[t] : kMaxTerms] += hp.coef[t];
      continue;
    }
    if (hp.term < 0 || hp.term >= k->n_terms) return fail(c, SGP_E_BADARG, mismatch);
    const sgp_kernel_term& term = k->terms[hp.term];
    const int t = flat_of[hp.term];
    if (hp.kind == SGP_HYPER_ARD_BETA && term.type == SGP_TERM_ARD) {
      if (hp.dim < 0 || hp.dim >= d || ard_h[static_cast<size_t>(t) * d + hp.dim] >= 0 || hp.value != term.beta[hp.dim])
        return fail(c, SGP_E_BADARG, mismatch);
      ard_h[static_cast<size_t>(t) * d + hp.dim] = i;
    } else if (hp.kind == SGP_HYPER_RBF_SIGMA && term.type == SGP_TERM_RBF) {
      if (a.rbf_h[t] >= 0 || hp.value != term.sigma) return fail(c, SGP_E_BADARG, mismatch);
      a.rbf_h[t] = i;
      a.sigma3[t] = term.sigma * term.sigma * term.sigma;
    } else {
      return fail(c, SGP_E_BADARG, mismatch);
    }
  }
  for (int t = 0; t < k->n_terms; ++t) {
    const int ft = flat_of[t];
    if (ft < 0) continue;
    bool covered = true;
    if (k->terms[t].type == SGP_TERM_RBF) covered = a.rbf_h[ft] >= 0;
    for (int j = 0; covered && k->terms[t].type == SGP_TERM_ARD && j < d; ++j)
      covered = ard_h[static_cast<size_t>(ft) * d + j] >= 0;
    if (!covered) return fail(c, SGP_E_BADARG, mismatch);
  }
  const int ns = static_cast<int>(scale_h.size());
  o.n_dbl = static_cast<size_t>(T) * d + scale_coef.size();
  o.tables.assign(o.n_dbl * 8 + (ard_h.size() + scale_h.size()) * 4 + 8, 0);
  std::memcpy(o.tables.data(), beta.data(), static_cast<size_t>(T) * d * 8);
  std::memcpy(o.tables.data() + static_cast<size_t>(T) * d * 8, scale_coef.data(), scale_coef.size() * 8);
  std::memcpy(o.tables.data() + o.n_dbl * 8, ard_h.data(), ard_h.size() * 4);
  std::memcpy(o.tables.data() + o.n_dbl * 8 + ard_h.size() * 4, scale_h.data(), scale_h.size() * 4);
  a.n = n; a.m = m; a.d = d;
  a.training = mode == SGP_KEVAL_TRAINING;
  a.kf = kf;
  a.n_scale = dK_out ? ns : 0;
  o.nh = dK_out ? nh : 0;
  return SGP_OK;
}

// Points the launch arguments at the tables uploaded to dev.
void kernel_eval_bind(KernelEvalSetup& o, const char* dev) {
  const double* dd = reinterpret_cast<const double*>(dev);
  const int* di = reinterpret_cast<const int*>(dev + o.n_dbl * 8);
  const size_t td = static_cast<size_t>(o.a.kf.n_terms) * o.a.d;
  o.a.beta = dd;
  o.a.scale_coef = dd + td;
  o.a.ard_h = di;
  o.a.scale_h = di + td;
}

// Allocations of one call that do not fit in the device's free memory (counting what regrowing a buffer frees):
// SGP_E_NOMEM before any of them is made.
int kernel_eval_fits(Ctx* c, const char* entry, std::initializer_list<std::pair<const DevScratch*, size_t>> bufs) {
  size_t free_b = 0, total_b = 0;
  SGP_CUDA(c, cudaMemGetInfo(&free_b, &total_b));
  size_t need = 0;
  for (const auto& [buf, bytes] : bufs)
    if (bytes > buf->cap) need += bytes - buf->cap;
  if (need > free_b)
    return fail(c, SGP_E_NOMEM, std::string(entry) + ": " + std::to_string(need >> 20) + " MiB of device memory needed, " +
                                    std::to_string(free_b >> 20) + " MiB free");
  return SGP_OK;
}

int upload_tables(Ctx* c, const KernelEvalSetup& o) {
  SGP_CUDA(c, cudaMemcpyAsync(c->keval_ws.p, o.tables.data(), o.tables.size(), cudaMemcpyHostToDevice, c->stream));
  SGP_CUDA(c, cudaStreamSynchronize(c->stream));   // o.tables is the caller's local
  return SGP_OK;
}

size_t align256(size_t b) { return (b + 255) / 256 * 256; }
}  // namespace

int sgp_kernel_eval(sgp_ctx* h, const sgp_kernel_desc* kernel, const sgp_hyper* hypers, int32_t n_hypers, const void* A,
                    int32_t a_is_f32, int64_t n, const double* B, int32_t m, int32_t d, int32_t mode, double* K_out,
                    double* dK_out) {
  Ctx* c = reinterpret_cast<Ctx*>(h);
  if (!c) return SGP_E_BADARG;
  KernelEvalSetup o;
  int rc = kernel_eval_setup(c, "sgp_kernel_eval", kernel, hypers, n_hypers, A, n, B, m, d, mode, K_out, dK_out, o);
  if (rc != SGP_OK) return rc;
  SGP_CUDA(c, cudaSetDevice(c->device));
  const bool training = mode == SGP_KEVAL_TRAINING;
  const size_t esz = a_is_f32 ? 4 : 8;
  const size_t row = static_cast<size_t>(d) * esz;
  // windows of rows whose K and dK together stay within kPredictKBytes (at least one row)
  const size_t row_out = static_cast<size_t>(1 + o.nh) * m * 8;
  const long long win = std::min<long long>(n, std::max<long long>(1, static_cast<long long>(kPredictKBytes / row_out)));
  const size_t win_out = static_cast<size_t>(win) * row_out;
  // the training vectors go to the device once, after the tables: B as fp64 (CROSS), or A as given (TRAINING, where the
  // windows then read their rows from that copy instead of staging them)
  const size_t tab = align256(o.tables.size());
  const size_t b_bytes = training ? static_cast<size_t>(n) * row : static_cast<size_t>(m) * d * 8;
  const size_t stage = training ? 0 : static_cast<size_t>(win) * row;
  rc = kernel_eval_fits(c, "sgp_kernel_eval", {{&c->keval_ws, tab + b_bytes}, {&c->keval_out_ws, 2 * win_out},
                                               {&c->stage_x[0], stage}, {&c->stage_x[1], stage}});
  if (rc == SGP_OK) rc = ctx_scratch(c, c->keval_ws, tab + b_bytes);
  if (rc == SGP_OK) rc = ctx_scratch(c, c->keval_out_ws, 2 * win_out);
  if (rc != SGP_OK) return rc;
  char* dev = c->keval_ws.as<char>();
  kernel_eval_bind(o, dev);
  SGP_CUDA(c, cudaMemcpyAsync(dev + tab, training ? A : B, b_bytes, cudaMemcpyHostToDevice, c->stream));
  if ((rc = upload_tables(c, o)) != SGP_OK) return rc;
  o.a.B = dev + tab;
  o.a.b_is_f32 = training ? a_is_f32 : 0;
  o.a.a_is_f32 = a_is_f32;
  // each window's K and dK go to one of two output buffers [K | dK_0 | dK_1 ..] of win rows each, and are copied out
  // (copy stream) once the next window is queued, as sgp_predict does
  double* out = c->keval_out_ws.as<double>();
  const size_t mat = static_cast<size_t>(win) * m;
  const size_t full = static_cast<size_t>(n) * m;
  auto copy_out = [&](int b, long long p0, long long cn) -> int {
    const double* src = out + static_cast<size_t>(1 + o.nh) * mat * b;
    const size_t bytes = static_cast<size_t>(cn) * m * 8, off = static_cast<size_t>(p0) * m;
    SGP_CUDA(c, cudaStreamWaitEvent(c->copy_stream, c->out_ready[b], 0));
    SGP_CUDA(c, cudaMemcpyAsync(K_out + off, src, bytes, cudaMemcpyDeviceToHost, c->copy_stream));
    for (int hh = 0; hh < o.nh; ++hh)
      SGP_CUDA(c, cudaMemcpyAsync(dK_out + hh * full + off, src + (1 + hh) * mat, bytes, cudaMemcpyDeviceToHost,
                                  c->copy_stream));
    SGP_CUDA(c, cudaEventRecord(c->out_free[b], c->copy_stream));
    return SGP_OK;
  };
  long long windows = 0, pending_p0 = 0, pending_n = 0;
  rc = feed_rows(c, training, training ? o.a.B : A, nullptr, n, row, win,
                 [&](const void* dA, const double*, long long p0, long long cn) -> int {
                   const int b = static_cast<int>(windows & 1);
                   double* dst = out + static_cast<size_t>(1 + o.nh) * mat * b;
                   KernelEvalArgs a = o.a;
                   a.A = dA; a.n = cn; a.row0 = p0;
                   a.K = dst;
                   a.dK = o.nh > 0 ? dst + mat : nullptr;
                   a.dk_stride = mat;
                   SGP_CUDA(c, cudaStreamWaitEvent(c->stream, c->out_free[b], 0));
                   SGP_CUDA(c, launch_kernel_eval(a, c->stream));
                   c->launches += 1;
                   SGP_CUDA(c, cudaEventRecord(c->out_ready[b], c->stream));
                   int r = SGP_OK;
                   if (windows > 0 && (r = copy_out(b ^ 1, pending_p0, pending_n)) != SGP_OK) return r;
                   ++windows;
                   pending_p0 = p0;
                   pending_n = cn;
                   return SGP_OK;
                 });
  if (rc == SGP_OK) rc = copy_out(static_cast<int>((windows - 1) & 1), pending_p0, pending_n);
  if (rc != SGP_OK) return rc;
  SGP_CUDA(c, cudaStreamSynchronize(c->copy_stream));
  return SGP_OK;
}

int sgp_kernel_eval_device(sgp_ctx* h, const sgp_kernel_desc* kernel, const sgp_hyper* hypers, int32_t n_hypers,
                           const void* dA, int32_t a_is_f32, int64_t n, const double* dB, int32_t m, int32_t d, int32_t mode,
                           double* dK_out, double* ddK_out) {
  Ctx* c = reinterpret_cast<Ctx*>(h);
  if (!c) return SGP_E_BADARG;
  const char* entry = "sgp_kernel_eval_device";
  KernelEvalSetup o;
  int rc = kernel_eval_setup(c, entry, kernel, hypers, n_hypers, dA, n, dB, m, d, mode, dK_out, ddK_out, o);
  if (rc != SGP_OK) return rc;
  SGP_CUDA(c, cudaSetDevice(c->device));
  rc = device_ptr_ok(c, dA, entry, "A");
  if (rc == SGP_OK && dB) rc = device_ptr_ok(c, dB, entry, "B");
  if (rc == SGP_OK) rc = device_ptr_ok(c, dK_out, entry, "K_out");
  if (rc == SGP_OK && ddK_out) rc = device_ptr_ok(c, ddK_out, entry, "dK_out");
  if (rc == SGP_OK) rc = kernel_eval_fits(c, entry, {{&c->keval_ws, o.tables.size()}});
  if (rc == SGP_OK) rc = ctx_scratch(c, c->keval_ws, o.tables.size());
  if (rc == SGP_OK) rc = upload_tables(c, o);
  if (rc != SGP_OK) return rc;
  kernel_eval_bind(o, c->keval_ws.as<char>());
  KernelEvalArgs& a = o.a;
  a.A = dA; a.a_is_f32 = a_is_f32;
  a.B = dB ? static_cast<const void*>(dB) : dA;
  a.b_is_f32 = dB ? 0 : a_is_f32;
  a.row0 = 0;
  a.K = dK_out;
  a.dK = o.nh > 0 ? ddK_out : nullptr;
  a.dk_stride = static_cast<size_t>(n) * m;
  SGP_CUDA(c, launch_kernel_eval(a, c->stream));
  c->launches += 1;
  return SGP_OK;
}

namespace {
// The refusals both scale entries share, taken before any allocation or launch: the dtype flag, the shape, and X on
// the context's device wherever rows exist.
int scale_args(Ctx* c, const char* entry, const void* dX, int32_t x_is_f32, int64_t n, int32_t d) {
  if (x_is_f32 != 0 && x_is_f32 != 1)
    return fail(c, SGP_E_BADARG, std::string(entry) + ": x_is_f32 must be 0 (fp64) or 1 (fp32), not " +
                                     std::to_string(x_is_f32));
  if (n < 0 || d < 1) return fail(c, SGP_E_BADARG, std::string(entry) + ": no features or a negative row count");
  if (n > 0 && (n > INT64_MAX / d || scale_row_blocks(n) > 2147483647LL))
    return fail(c, SGP_E_BADARG, std::string(entry) + ": too many rows");
  if (n > 0 && !dX) return fail(c, SGP_E_BADARG, std::string(entry) + ": null X");
  SGP_CUDA(c, cudaSetDevice(c->device));
  return n > 0 ? device_ptr_ok(c, dX, entry, "X") : SGP_OK;
}
}  // namespace

int sgp_column_sums_device(sgp_ctx* h, const void* dX, int32_t x_is_f32, int64_t n, int32_t d, const double* center,
                           double* out) {
  Ctx* c = reinterpret_cast<Ctx*>(h);
  if (!c) return SGP_E_BADARG;
  const char* entry = "sgp_column_sums_device";
  int rc = scale_args(c, entry, dX, x_is_f32, n, d);
  if (rc != SGP_OK) return rc;
  if (!out) return fail(c, SGP_E_BADARG, std::string(entry) + ": null out");
  if (n == 0) {
    std::fill(out, out + d, 0.0);
    return SGP_OK;
  }
  const size_t cols = static_cast<size_t>(d);
  rc = ctx_scratch(c, c->scale_ws, (2 + static_cast<size_t>(scale_row_blocks(n))) * cols * sizeof(double));
  if (rc != SGP_OK) return rc;
  double* ws = c->scale_ws.as<double>();
  if (center) SGP_CUDA(c, cudaMemcpyAsync(ws, center, cols * sizeof(double), cudaMemcpyHostToDevice, c->stream));
  SGP_CUDA(c, launch_column_sums(dX, x_is_f32, n, d, center ? ws : nullptr, ws + 2 * cols, ws + cols, c->stream));
  c->launches += 2;
  SGP_CUDA(c, cudaMemcpyAsync(out, ws + cols, cols * sizeof(double), cudaMemcpyDeviceToHost, c->stream));
  SGP_CUDA(c, cudaStreamSynchronize(c->stream));
  return SGP_OK;
}

int sgp_scale_apply_device(sgp_ctx* h, const void* dX, int32_t x_is_f32, int64_t n, int32_t d, const double* mean,
                           const double* sd, double* dY) {
  Ctx* c = reinterpret_cast<Ctx*>(h);
  if (!c) return SGP_E_BADARG;
  const char* entry = "sgp_scale_apply_device";
  int rc = scale_args(c, entry, dX, x_is_f32, n, d);
  if (rc != SGP_OK || n == 0) return rc;
  if (!mean || !sd || !dY) return fail(c, SGP_E_BADARG, std::string(entry) + ": null mean, sd or Y");
  rc = device_ptr_ok(c, dY, entry, "Y");
  if (rc == SGP_OK) rc = ctx_scratch(c, c->scale_ws, 2 * static_cast<size_t>(d) * sizeof(double));
  if (rc != SGP_OK) return rc;
  double* ws = c->scale_ws.as<double>();
  SGP_CUDA(c, cudaMemcpyAsync(ws, mean, static_cast<size_t>(d) * sizeof(double), cudaMemcpyHostToDevice, c->stream));
  SGP_CUDA(c, cudaMemcpyAsync(ws + d, sd, static_cast<size_t>(d) * sizeof(double), cudaMemcpyHostToDevice, c->stream));
  SGP_CUDA(c, launch_scale_apply(dX, x_is_f32, n, d, ws, ws + d, dY, c->stream));
  c->launches += 1;
  return SGP_OK;
}

}  // extern "C"
