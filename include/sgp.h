/* sgp.h -- C-ABI of the H100-native projected-process (sparse GP) hot path.
 *
 * Drop-in boundary for ONE path of akopich/spark-gp (reference paths relative to
 * /root/reference/src/main/scala/org/apache/spark/ml/):
 *
 *   commons/ProjectedGaussianProcessHelper.scala:20-36   getMatrixKmnKnmAndVectorKmny
 *       G = sum_e K_mn^(e) K_mn^(e)^T  (m x m),  b = sum_e K_mn^(e) y_e  (m)
 *   commons/ProjectedGaussianProcessHelper.scala:49-65   getMagicVector / assertSymPositiveDefinite
 *   commons/GaussianProcessCommons.scala:118-126         GaussianProjectedProcessRawPredictor.predict
 *
 * The reference has NO FFI of its own (pure Scala on Breeze); these entry points are what a JNI shim
 * replacing the body of `getMatrixKmnKnmAndVectorKmny` / `getMagicVector` would bind (INTEGRATION.md
 * shows the Scala + JNI stub).  Plain pointers and sizes only; the caller owns every host array; the
 * context owns device memory, streams, cuSOLVER/cuBLAS handles and the NCCL communicator.  Every call
 * returns an int status (never throws, never aborts); sgp_last_error() gives the text.
 *
 * Threading: a context is bound to one CUDA device and may be used from any ONE thread at a time
 * (Spark executor task threads: one context per task/partition, or lock around it).  No global
 * mutable state.
 */
#ifndef SGP_H_
#define SGP_H_

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

typedef struct sgp_ctx sgp_ctx;

/* status codes; the host shim maps them back to the reference's exceptions */
enum {
  SGP_OK = 0,
  SGP_E_BADARG = 1,   /* IllegalArgumentException / require(...)                                  */
  SGP_E_CUDA = 2,     /* CUDA / cuSOLVER / cuBLAS runtime failure                                 */
  SGP_E_NOT_PD = 3,   /* NotPositiveDefiniteException   (PGPH:9-11, 62-65)                        */
  SGP_E_NCCL = 4,
  SGP_E_STATE = 5,    /* call order violated (e.g. accumulate before begin) ~ TrainingVectorsNotInitializedException */
  SGP_E_SINGULAR = 6, /* MatrixSingularException (commons/util/logDetAndInv.scala:27-28), LU info > 0 */
  SGP_E_NOMEM = 7,
  SGP_E_RANGE = 8     /* int8 modes only: scaled squared norms above 4096 (the tensor-core operand range) / above the
                         magnitude budget (SGP_PREC_I8), or scaled squared norms above 2048 (SGP_PREC_I8_DIRECT); rerun in SGP_PREC_F64.
                         sgp_kmeans*: a nearest-centre squared distance beyond the fp32 range after the prescale */
};

/* Flattened kernel DSL (the files under commons/kernel/).  A kernel is a sum of terms  sum_t scale_t * k_t:
 *   SGP_TERM_ARD : k(a,b) = exp(-sum_k beta_k^2 (a_k-b_k)^2)      kernel/ARDRBFKernel.scala:43-46
 *   SGP_TERM_RBF : k(a,b) = exp(-||a-b||^2 / (2 sigma^2))         kernel/RBFKernel.scala:66-76
 *   SGP_TERM_EYE : identity kernel: contributes ZERO to any cross kernel (kernel/Kernel.scala:157),
 *                  `scale` to the training-kernel diagonal (:151), to selfKernel (:161) and to
 *                  whiteNoiseVar (:159).
 * `scale` is the product of all ScalarTimesKernel factors above the leaf (kernel/ScalarTimesKernel.scala:20-28). */
enum { SGP_TERM_ARD = 0, SGP_TERM_RBF = 1, SGP_TERM_EYE = 2 };

typedef struct {
  int32_t type;        /* SGP_TERM_*                                   */
  int32_t reserved;
  double scale;        /* C >= 0                                       */
  double sigma;        /* RBF only                                     */
  const double* beta;  /* ARD only: d inverse length-scales            */
} sgp_kernel_term;

typedef struct {
  int32_t n_terms;
  int32_t reserved;
  const sgp_kernel_term* terms;
} sgp_kernel_desc;

/* Arithmetic modes of the statistics kernel.  All modes accumulate G and b in fp64. */
enum {
  SGP_PREC_F64 = 0,        /* fp32 kernel elements (direct-form distances in fp32, exp as ex2.approx within 2 ulp;
                              elements below 2^-126 C flushed to 0; the term scale C applied in fp64), fp64 DMMA Gram.
                              Points and active set are centred in fp64 before the fp32 rounding (on the active-set
                              mean, rounded to a whole multiple of its standard deviation), so the error does not grow
                              with the data's distance from the origin: G, b <= 1e-6 and mean / variance <= 1e-5 also
                              for data 1e3 length scales out (see DESIGN.md). */
  SGP_PREC_F64_STRICT = 1, /* elements in fp64 as well, same centring (verification mode, ~1e-13 on G,b)   */
  SGP_PREC_I8 = 2,         /* wgmma path: distance contraction on fp16 hi/lo splits (fp32 accumulators), kernel elements
                              as 23-bit fixed point in three balanced int8 digits, Gram = six int8 products with
                              EXACT int32 accumulation, folded into fp64.  Kernels with one non-Eye term, d <= 32; other
                              qualifying shapes are served by SGP_PREC_I8_DIRECT (sgp_last_path tells which ran).       */
  SGP_PREC_AUTO = 3,       /* default.  An accumulate call of >= 32768 points whose scaled squared norms are small (mean over
                              points + mean over the active set <= 6: the kernel values are not tiny) runs the int8 Gram --
                              SGP_PREC_I8 when the kernel / shape qualifies, else SGP_PREC_I8_DIRECT when THAT qualifies;
                              everything else runs SGP_PREC_F64.  The budget is decided on the first chunk of a call and
                              re-checked over the whole begin..finish window (SGP_E_RANGE at finish -> rerun in F64).
                              On large-norm data the fixed-point elements (absolute error 2^-24) are not parity-grade
                              whatever the distance form (DESIGN.md, 'precision': airfoil-like data 1.5e-4 .. 1.5e-2 on
                              the posterior mean), hence the budget applies to both int8 modes.                         */
  SGP_PREC_I8_DIRECT = 4   /* same exact int8 Gram as SGP_PREC_I8, but the exponents come from fp32 DIRECT-FORM distances on
                              the CUDA cores (no cancellation; coordinates are centred on the active-set mean in fp64
                              first) and the kernel may be a sum of up to 4 non-Eye terms (kernel/SumOfKernels.scala:57-58)
                              with n_terms * roundup(d, 4) <= 72.  Scaled squared norms up to 2048 (statistics <= 1e-6);
                              requesting it explicitly asserts that the data are benign (see SGP_PREC_AUTO).            */
};

/* ---- context ------------------------------------------------------------------------------ */
int sgp_ctx_create(sgp_ctx** out, int device);
int sgp_ctx_destroy(sgp_ctx* ctx);
const char* sgp_last_error(const sgp_ctx* ctx);   /* valid until the next call on ctx; ctx==NULL -> creation error */
int sgp_set_precision(sgp_ctx* ctx, int mode);
int sgp_version(void);

/* ---- multi-GPU (one process / context per GPU; replaces PGPH:23 broadcast + PGPH:25-35 treeAggregate) */
#define SGP_UNIQUE_ID_BYTES 128
int sgp_comm_unique_id(void* out128);                                   /* rank 0, then ship the bytes to all ranks */
/* Attaches one communicator of nranks ranks to ctx.  SGP_E_BADARG for a null id, nranks < 1, rank < 0 or rank >= nranks;
 * SGP_E_STATE when ctx already has a communicator (the first one stays attached); SGP_E_NCCL when ncclCommInitRank
 * fails, leaving ctx without a communicator.  A refused call leaves ctx usable.
 * With a communicator of nranks > 1, sgp_stats_finish, sgp_bcm_nll, _folds, _slots and sgp_laplace_nll, _any_size,
 * _classes, _classes_any_size, _slots_any_size, _fold_slots_any_size each make exactly one ncclAllReduce, and a status
 * decided on one rank (SGP_E_RANGE, SGP_E_SINGULAR, SGP_E_NOT_PD) is returned on every rank.  sgp_kmeans_sharded[_device]
 * makes collectives of its own (see there).  The other entries are rank-local.  The caller's obligation: every rank makes the same sequence of these calls, with the same kernel
 * structure, n_eval and descriptor layout.  Refusals that depend on the rank's own data return BEFORE the collective and
 * leave the peers blocked in it: the on-chip Laplace limit (117 points in the largest expert), the global-memory Laplace
 * kernel's limit (SGP_E_BADARG above its per-expert point bound), the 46340-point limit of
 * the BCM LU path, SGP_E_NOMEM of the LU workspace / Laplace workspace / mode stores, and a rank without experts
 * (SGP_E_STATE).  The caller must prevent them, e.g. by giving every rank experts that fit the same kernel family. */
int sgp_comm_init(sgp_ctx* ctx, const void* id128, int rank, int nranks);

/* ---- the hot path:  PGPH:20-36 ------------------------------------------------------------- */
/* Active set Z: m x d row-major fp64 (activeSet: Array[Vector]).  Resets G, b to zero.  Every begin closes the previous
 * window first: after a failed begin, the calls that need one (accumulate, finish, magic, set_magic, predict,
 * cross_kernel, kmn_sweep) return SGP_E_STATE until a begin succeeds. */
int sgp_stats_begin(sgp_ctx* ctx, const sgp_kernel_desc* kernel, const double* Z, int32_t m, int32_t d);

/* One shard / partition / expert group of points in HOST memory: X is n x d row-major (fp64, or fp32
 * when x_is_f32 != 0), y is n fp64 labels.  Copies host->device in pipelined chunks and launches the
 * fused K_mn + Gram kernel per chunk.  May be called any number of times between begin and finish. */
int sgp_stats_accumulate(sgp_ctx* ctx, const void* X, int32_t x_is_f32, const double* y, int64_t n);

/* Same, points already resident in device memory (the bench's `value` leg). */
int sgp_stats_accumulate_device(sgp_ctx* ctx, const void* dX, int32_t x_is_f32, const double* dy, int64_t n);

/* Sum over ranks (one ncclAllReduce of the packed [G;b], if a communicator exists), then copy out.
 * G_out: m x m fp64 (symmetric, so row-/column-major are the same bytes), b_out: m.  Either may be NULL
 * (statistics stay on the device for sgp_magic).  The first finish closes the window and decides its status; a repeated
 * finish only copies out again and returns the same status.  A window whose finish returned SGP_E_RANGE keeps that
 * status until the next begin: G_out / b_out are still copied out, but sgp_magic without G_in returns SGP_E_STATE. */
int sgp_stats_finish(sgp_ctx* ctx, double* G_out, double* b_out);

/* Block until the context's stream is idle (timing hygiene for callers using the _device entry). */
int sgp_sync(sgp_ctx* ctx);

/* ---- the m x m tail:  PGPH:49-65 ------------------------------------------------------------ */
/* Uses the kernel + active set of the last sgp_stats_begin and the device-resident G, b (after finish),
 * or host G_in/b_in when non-NULL.  K_mm = trainingKernel (Eye terms on the diagonal),
 * A = whiteNoiseVar*K_mm + G; SGP_E_NOT_PD if any eigenvalue of A < 0; magicVector = A \ b;
 * magicMatrix = whiteNoiseVar*inv(A) - inv(K_mm).  Outputs may be NULL (kept on device for predict).
 * A successful Cholesky factorization of A proves "no eigenvalue < 0" and supplies the solves (SPD: same result as
 * the reference's LU to rounding); only if it breaks down does the call run the reference's literal dsyevd + LU sequence.
 * SGP_E_STATE without G_in before finish, or after a finish that returned SGP_E_RANGE.  Once its arguments and the
 * window's state are accepted, the call uninstalls the pair of any earlier sgp_magic / sgp_set_magic: if it then fails
 * (SGP_E_NOT_PD, SGP_E_SINGULAR, ...), sgp_predict and sgp_predict_device return SGP_E_STATE until a pair is installed
 * again.  With G_in on a window that is still open, the window is closed and its accumulated statistics are replaced. */
int sgp_magic(sgp_ctx* ctx, const double* G_in, const double* b_in,
              double* magic_vector /* m */, double* magic_matrix /* m x m */);

/* ---- the hyper-parameter objective (SURVEY 8 f1):  GPR:55-68 summed over experts as GPC:73-78 ----------------- */
/* Experts of this rank, packed expert-major: expert e owns rows offsets[e] .. offsets[e+1]-1 of X (row-major, d
 * columns, fp64) and of y.  Kept on the device until replaced (the L-BFGS-B loop evaluates the objective many times). */
int sgp_experts_upload(sgp_ctx* ctx, const double* X, const double* y, const int64_t* offsets, int64_t n_experts, int32_t d);

/* Same result as sgp_experts_upload, but the grouping itself (commons/GaussianProcessCommons.scala:26-31: E =
 * Math.round(N / datasetSizeForExpert), point i in zipWithIndex order -> expert i % E) runs on the device: the caller
 * passes the points as they are (row-major, fp32 or fp64) and the library gathers them into the expert-major layout while
 * the copy streams in -- the reference's zipWithIndex / groupByKey shuffle, here a strided gather.  Latent modes start at 0. */
int sgp_experts_upload_grouped(sgp_ctx* ctx, const void* X, int32_t x_is_f32, const double* y, int64_t n, int32_t d,
                               int32_t dataset_size_for_expert);
/* sgp_experts_upload_grouped on points already in device memory: the same refusals, allocation, offsets and gather, read
 * in place instead of staged, so the experts are the same bits as the host upload's (the gather is a permutation and an
 * exact fp32 -> fp64 conversion).  The library's stream does not wait for other streams: dX and dy must be written
 * before the call.  They are read before it returns.  The same holds for every _device entry below. dX and dy must be device (or managed) memory on the
 * context's device: anything else is refused with SGP_E_BADARG (checked with cudaPointerGetAttributes) before any
 * allocation or launch. */
int sgp_experts_upload_grouped_device(sgp_ctx* ctx, const void* dX, int32_t x_is_f32, const double* dy, int64_t n,
                                      int32_t d, int32_t dataset_size_for_expert);

/* The grouped upload with the number of experts given instead of derived from datasetSizeForExpert: point i of dX -> expert
 * i % n_experts, the same offsets, gather and bits as sgp_experts_upload_grouped_device with that E.  A rank of a
 * data-parallel fit uploads with it the rows of its own block of the global experts [e0, e0 + n_experts): taken in global
 * row order, row e + j E_total of expert e is local row (e - e0) + j n_experts, so each expert is the single-GPU upload's,
 * row for row.  SGP_E_BADARG for null pointers, n < 1, d < 1, n_experts < 1, n_experts > n (an empty expert), and for
 * pointers that are not device memory on the context's device, before any allocation or launch.  The modes of such an
 * upload can be ungrouped (sgp_experts_get_f_rows_device). */
int sgp_experts_upload_strided_device(sgp_ctx* ctx, const void* dX, int32_t x_is_f32, const double* dy, int64_t n,
                                      int32_t d, int64_t n_experts);

/* One hyper-parameter, in the order of Kernel.getHyperparameters (depth first, trainable scalar prepended). */
enum { SGP_HYPER_SCALE = 0, SGP_HYPER_ARD_BETA = 1, SGP_HYPER_RBF_SIGMA = 2 };
typedef struct {
  int32_t kind;        /* SGP_HYPER_*                                                                            */
  int32_t term;        /* ARD_BETA / RBF_SIGMA: index into sgp_kernel_desc.terms                                  */
  int32_t dim;         /* ARD_BETA: feature index                                                                 */
  int32_t reserved;
  double value;        /* ARD_BETA: beta_k ; RBF_SIGMA: sigma                                                     */
  const double* coef;  /* SCALE: kernel->n_terms entries, d(terms[t].scale)/d(this scalar)  (TrainableScalarTimesKernel,
                          kernel/ScalarTimesKernel.scala:93-97: the derivative is the inner kernel matrix)        */
} sgp_hyper;

/* nll = sum_e [ 1/2 y_e^T K_e^-1 y_e + 1/2 log|det K_e| ]  and its gradient (n_hypers entries), summed over the
 * uploaded experts and over ranks (ncclAllReduce of 1 + n_hypers doubles + a status word if a communicator exists).
 * Experts of any size (GaussianProcessParams.scala:36 sets no bound).  Fast path: on-chip Cholesky per expert (<= ~165
 * points, SPD).  When an expert is larger, or a Cholesky pivot is not positive, the evaluation runs the reference's own
 * arithmetic instead -- LU with partial pivoting, log|det| with the sign dropped (logDetAndInv.scala:36-63, GPR:59) --
 * and only an exactly singular matrix fails, with SGP_E_SINGULAR (Breeze's MatrixSingularException).
 * The LU path holds every expert's matrix and inverse at once, about 16 E n_max^2 bytes (E experts, n_max the largest):
 * SGP_E_NOMEM, before any launch, when that exceeds the device's free memory.  SGP_E_BADARG, before any allocation or
 * launch, above 46340 points per expert (32-bit indexing of the per-expert matrix, as for the Laplace limit below). */
int sgp_bcm_nll(sgp_ctx* ctx, const sgp_kernel_desc* kernel, const sgp_hyper* hypers, int32_t n_hypers,
                double* nll_out, double* grad_out);

/* ---- cross-validation (Spark's CrossValidator over the regression estimator) ------------------------------------ */
/* Uploads the n_folds training sets of a k-fold split at once.  fold_of[i] in [0, n_folds) is the fold of point i
 * (n_folds >= 2).  Set k is fold k's training split: the points with fold_of[i] != k, in index order (Spark keeps the
 * row order).  It is grouped as sgp_experts_upload_grouped groups a shard: E_k = Math.round(N_k / dataset_size_for_expert),
 * the j-th training point goes to expert j % E_k.  The sets are stored one after another: X and y cross PCIe once, and
 * each staged chunk is gathered on the device into every set that holds its points.  Needs (n_folds - 1) n (d + 2) * 8
 * bytes of device memory (rows, labels and latent modes of every set): SGP_E_NOMEM past what the device has free.
 * SGP_E_BADARG for n_folds < 2, a fold index outside [0, n_folds), or a set with E_k == 0 (the reference's / by zero).
 * As every upload, it resets the latent modes and the one-vs-rest modes.  The other objectives (sgp_bcm_nll,
 * sgp_laplace_nll* but sgp_laplace_nll_fold_slots_any_size) see a fold upload as one expert set: the union of every
 * set's experts. */
int sgp_experts_upload_folds(sgp_ctx* ctx, const void* X, int32_t x_is_f32, const double* y, int64_t n, int32_t d,
                             const int32_t* fold_of, int32_t n_folds, int32_t dataset_size_for_expert);
/* sgp_experts_upload_folds on points already in device memory: every set is the same bits as the host upload's.  fold_of
 * (the split, not the data) stays in host memory. dX and dy must be device (or managed) memory on the
 * context's device: anything else is refused with SGP_E_BADARG (checked with cudaPointerGetAttributes) before any
 * allocation or launch. */
int sgp_experts_upload_folds_device(sgp_ctx* ctx, const void* dX, int32_t x_is_f32, const double* dy, int64_t n,
                                    int32_t d, const int32_t* fold_of, int32_t n_folds, int32_t dataset_size_for_expert);
/* The training sets of a data-parallel model selection, stored as sgp_experts_upload_folds stores its sets.  dX / dy
 * hold n_sets blocks one after another: block k has set_rows[k] rows, the rows of training set k that this rank's
 * experts own, in the set's row order.  Row i of block k goes to local expert i % set_experts[k] of set k.
 * Per set, one expert-offset launch and one gather of the block, by the fold upload's kernels and arithmetic.  It fills
 * the state sgp_experts_upload_folds fills (the sets, their experts and largest experts, the reset latent and one-vs-rest
 * modes), so sgp_bcm_nll_folds, sgp_laplace_nll_fold_slots_any_size, sgp_experts_get_f_fold_slot and
 * sgp_experts_get_f_fold_rows_device read it unchanged; like the fold upload, its modes are read per set.
 * Contract: with block k the plain fold set X[fold_of != k] and set_experts[k] = Math.round(N_k / dataset_size_for_expert),
 * every fold-slot value, gradient and mode equals the one after sgp_experts_upload_folds_device, bit for bit.
 * SGP_E_BADARG for null pointers, n_sets < 1, d < 1, set_rows[k] < 1, set_experts[k] < 1, set_experts[k] > set_rows[k]
 * (an empty expert), and for pointers that are not device memory on the context's device; SGP_E_NOMEM under the fold
 * upload's free-memory rule (the sets' rows, labels and modes, sum set_rows (d + 2) * 8 bytes).  Every refusal comes
 * before any allocation or launch. */
int sgp_experts_upload_fold_sets_device(sgp_ctx* ctx, const void* dX, int32_t x_is_f32, const double* dy,
                                        const int64_t* set_rows, const int64_t* set_experts, int32_t n_sets, int32_t d);

/* The BCM objective of sgp_bcm_nll on several training sets of the last sgp_experts_upload_folds, in one launch over
 * experts x slots.  Slot s evaluates set sets[s] at its own kernels[s] and hypers[s * n_hypers ...] (the same kernel
 * structure and descriptor layout in every slot).  A set may be listed more than once, for several parameter maps on
 * one fold.  Outputs per slot: nll_out[s], grad_out[s * n_hypers ...].
 * Contract: slot s's value and gradient equal, bit for bit, what sgp_bcm_nll returns on
 * sgp_experts_upload_grouped(X[fold_of != k], y[fold_of != k], dataset_size_for_expert) with k = sets[s] and the same
 * kernel, whenever that single-set call runs the same kernel family (register, shared-memory or LU).  The call plans its
 * kernel once, on the largest expert over the listed sets; the register kernel's padded shapes add exact zeros only, so
 * within the register family the shape does not matter.
 * A slot whose on-chip Cholesky breaks down is evaluated again on the LU path, on its own set alone.  Experts too large for
 * the on-chip kernels put every slot on the LU path, one slot after another: 5 launches per slot instead of 2 per call.
 * sgp_last_bcm_path is 1 if any slot ran LU.  With a communicator: one ncclAllReduce of the n_eval rows and n_eval status
 * words.  Errors: SGP_E_STATE without a fold upload; SGP_E_BADARG for a set index outside [0, n_folds), a structure that
 * differs between slots, or n_eval outside [1, 65535], or more than 46340 points in the largest expert of a listed set
 * (before any allocation or launch); SGP_E_NOMEM when a slot's LU workspace exceeds the device's free memory, as for
 * sgp_bcm_nll; SGP_E_SINGULAR naming the first slot's set whose matrix is exactly singular. */
int sgp_bcm_nll_folds(sgp_ctx* ctx, const int32_t* sets, int32_t n_eval, const sgp_kernel_desc* kernels,
                      const sgp_hyper* hypers, int32_t n_hypers, double* nll_out /* n_eval */,
                      double* grad_out /* n_eval x n_hypers */);

/* The BCM objective of sgp_bcm_nll at several kernels on the last grouped upload (sgp_experts_upload_grouped or its
 * _device form), in one launch over experts x slots: several param maps on one training set.  Slot s evaluates every
 * uploaded expert at kernels[s] and hypers[s * n_hypers ...] (the same kernel structure and descriptor layout in every
 * slot).  Outputs per slot: nll_out[s], grad_out[s * n_hypers ...].
 * Contract: slot s's value and gradient equal, bit for bit, what sgp_bcm_nll returns on the same upload with the same
 * kernel, whatever else is in the call.  The call plans its kernel on the upload's largest expert, as sgp_bcm_nll does.
 * A slot whose on-chip Cholesky breaks down is evaluated again on the LU path, alone; experts too large for the on-chip
 * kernels put every slot on the LU path, one slot after another (the rules of sgp_bcm_nll_folds, whose code this entry
 * runs with every slot on one set).  sgp_last_bcm_path is 1 if any slot ran LU.  With a communicator: one ncclAllReduce
 * of the n_eval rows and n_eval status words.
 * Errors: SGP_E_STATE without a grouped upload -- a fold upload or an sgp_experts_upload is refused, since neither has
 * one training set to hand every slot; SGP_E_BADARG for n_eval outside [1, 65535], a structure or descriptor layout that
 * differs between slots, or more than 46340 points in the largest expert (before any allocation or launch); SGP_E_NOMEM
 * when a slot's LU workspace exceeds the device's free memory, as for sgp_bcm_nll; SGP_E_SINGULAR naming the first slot
 * whose matrix is exactly singular. */
int sgp_bcm_nll_slots(sgp_ctx* ctx, int32_t n_eval, const sgp_kernel_desc* kernels, const sgp_hyper* hypers,
                      int32_t n_hypers, double* nll_out /* n_eval */, double* grad_out /* n_eval x n_hypers */);

/* Binary classification (labels 0/1 in the uploaded y): per-expert Laplace approximation,
 * classification/GaussianProcessClassifier.scala:74-129 -- Newton iteration for the mode with the reference's step
 * halving, tolerance `tol` and warm start (the latent f of every uploaded point lives on the device, starts at zero
 * and persists across calls), then -log Z and its gradient, summed over experts and ranks.
 * The on-chip form: every expert's matrices live in shared memory, so an upload whose largest expert has more than 117
 * points is refused with SGP_E_BADARG.  sgp_laplace_nll_any_size takes any size.
 * tol must be > 0 (SGP_E_BADARG otherwise).  tol >= 1 returns SGP_E_SINGULAR before any launch, with the modes left as
 * they were: the loop runs while step > tol and step starts at 1, so no Newton iteration runs, the reference's L stays
 * zero and `L \ sqrtW` throws MatrixSingularException. */
int sgp_laplace_nll(sgp_ctx* ctx, const sgp_kernel_desc* kernel, const sgp_hyper* hypers, int32_t n_hypers, double tol,
                    double* neg_log_z_out, double* grad_out);
/* sgp_laplace_nll for experts of any size (GaussianProcessParams.scala:36 puts no bound on datasetSizeForExpert): same
 * arguments, outputs, modes, warm start and all-reduce.  When the largest uploaded expert fits on chip (<= 117 points)
 * it makes exactly sgp_laplace_nll's launch, so the results are the same bits.  Otherwise a global-memory kernel runs:
 * a persistent grid over the experts, each CTA with a workspace slice of 8 ld (2 ld + 44) bytes, ld = the largest
 * expert rounded up to 32 (the grid is bounded by the experts, the resident CTAs and 4 GiB of workspace), the Cholesky
 * of B and the cubic post-loop steps blocked on fp64 tensor cores.  Its bits do not depend on the grid or on the other
 * experts of the upload.  SGP_E_NOMEM, before the launch, when one slice exceeds the device's free memory;
 * SGP_E_BADARG above 46336 points per expert; SGP_E_SINGULAR for tol >= 1, as sgp_laplace_nll.  sgp_last_laplace_path
 * tells which kernel ran. */
int sgp_laplace_nll_any_size(sgp_ctx* ctx, const sgp_kernel_desc* kernel, const sgp_hyper* hypers, int32_t n_hypers,
                             double tol, double* neg_log_z_out, double* grad_out);
/* The latent modes f (same packed expert-major order as the uploaded points): the `y := f` of GPCls:62-65. */
int sgp_experts_get_f(sgp_ctx* ctx, double* f_out);

/* One-vs-rest (Spark's OneVsRest over the binary classifier): the uploaded y holds class indices 0 .. n_classes-1, and
 * class c's binary problem has the labels (y == c).  Evaluates the Laplace objective of sgp_laplace_nll for the n_eval
 * distinct classes listed in `classes`, each at its own hyper-parameters (kernels[i] and hypers[i * n_hypers ...]: the
 * same kernel structure and descriptor layout for every class), in one launch over experts x classes.  Every class keeps
 * its own latent modes on the device, [n_classes][n], allocated on first use and zero after every sgp_experts_upload* and
 * whenever n_classes changes; the modes of classes not listed are left as they are.  Outputs per listed class, in the
 * order of `classes`: neg_log_z_out[i], grad_out[i * n_hypers ...].  Class c's value, gradient and modes equal, bit for
 * bit, what sgp_laplace_nll returns on an upload of the labels (y == c) with the same modes, whichever other classes are
 * in the call.  With a communicator: one ncclAllReduce of the n_eval rows and n_eval status words.
 * Errors: SGP_E_BADARG for bad or repeated class indices, a structure that differs between classes, and experts above the
 * on-chip limit (as sgp_laplace_nll: the on-chip form); SGP_E_NOT_PD naming the first listed class whose B broke down;
 * SGP_E_SINGULAR for tol >= 1 (no Newton iteration runs, as sgp_laplace_nll), before any launch, every class's modes
 * left as they were. */
int sgp_laplace_nll_classes(sgp_ctx* ctx, int32_t n_classes, const int32_t* classes, int32_t n_eval,
                            const sgp_kernel_desc* kernels, const sgp_hyper* hypers, int32_t n_hypers, double tol,
                            double* neg_log_z_out /* n_eval */, double* grad_out /* n_eval x n_hypers */);
/* sgp_laplace_nll_classes for experts of any size, as sgp_laplace_nll_any_size: on chip (the same launch and bits as
 * sgp_laplace_nll_classes) when the largest expert fits, else the global-memory kernel over experts x listed classes.
 * On either path class c's value, gradient and modes equal, bit for bit, what sgp_laplace_nll_any_size returns on an
 * upload of the labels (y == c) with the same modes.  SGP_E_SINGULAR for tol >= 1, as sgp_laplace_nll_classes. */
int sgp_laplace_nll_classes_any_size(sgp_ctx* ctx, int32_t n_classes, const int32_t* classes, int32_t n_eval,
                                     const sgp_kernel_desc* kernels, const sgp_hyper* hypers, int32_t n_hypers, double tol,
                                     double* neg_log_z_out /* n_eval */, double* grad_out /* n_eval x n_hypers */);
/* Class cls's latent modes (packed expert-major order, n entries).  SGP_E_STATE before the first sgp_laplace_nll_classes
 * after an upload; SGP_E_BADARG for cls outside [0, n_classes). */
int sgp_experts_get_f_class(sgp_ctx* ctx, int32_t cls, double* f_out);

/* Model selection over param maps (TrainValidationSplit over the binary classifier or one-vs-rest): the Laplace
 * objective of n_eval slots in one launch over experts x slots, where slots may share a class and each keeps latent modes
 * of its own.  Listed slot i evaluates the labels (y == classes[i]) at kernels[i] and hypers[i * n_hypers ...] (the same
 * kernel structure and descriptor layout for every slot), and reads and writes the modes of mode slot mode_slots[i].
 * Classes may repeat (the binary classifier passes class 1 over its 0/1 labels: y == 1 is y itself); mode slots are
 * distinct and in [0, n_mode_slots).  The modes live in a store [n_mode_slots][n] of their own, apart from
 * sgp_laplace_nll_classes's, so neither entry moves the other's modes: allocated on first use, zero after every
 * sgp_experts_upload* and whenever n_mode_slots changes; the modes of mode slots not listed are left as they are.
 * Outputs per listed slot, in list order: neg_log_z_out[i], grad_out[i * n_hypers ...].  Slot i's value, gradient and
 * modes equal, bit for bit, what sgp_laplace_nll_any_size returns on an upload of the labels (y == classes[i]) with the
 * same modes, whichever other slots are in the call, on the on-chip and on the global-memory kernel alike (the kernel is
 * chosen as sgp_laplace_nll_any_size chooses it).  With a communicator: one ncclAllReduce of the n_eval rows and n_eval
 * status words.  Errors: SGP_E_STATE without an upload; SGP_E_BADARG for a repeated or out-of-range mode slot, a negative
 * class, n_eval > n_mode_slots, n_eval outside [1, 65535], or a structure that differs between slots; SGP_E_SINGULAR for
 * tol >= 1, before any launch, every mode left as it was; SGP_E_NOT_PD naming the mode slot of the first listed slot
 * whose B broke down; SGP_E_NOMEM, before any launch, when the store or one global-memory workspace slice exceeds the
 * device's free memory. */
int sgp_laplace_nll_slots_any_size(sgp_ctx* ctx, int32_t n_mode_slots, const int32_t* mode_slots,
                                   const int32_t* classes, int32_t n_eval, const sgp_kernel_desc* kernels,
                                   const sgp_hyper* hypers, int32_t n_hypers, double tol,
                                   double* neg_log_z_out /* n_eval */, double* grad_out /* n_eval x n_hypers */);
/* Mode slot mode_slot's latent modes (packed expert-major order, n entries).  SGP_E_STATE before the first
 * sgp_laplace_nll_slots_any_size after an upload; SGP_E_BADARG for mode_slot outside [0, n_mode_slots). */
int sgp_experts_get_f_slot(sgp_ctx* ctx, int32_t mode_slot, double* f_out);

/* One stored mode vector in ROW order, written to device memory: dF_out[i] = the mode of point i, which the grouped
 * upload put at position i / E of expert i % E (the first n % E experts one longer).  store: SGP_MODES_BINARY (the modes
 * of sgp_experts_get_f; index ignored), SGP_MODES_CLASS (class `index`, as sgp_experts_get_f_class) or SGP_MODES_SLOT
 * (mode slot `index`, as sgp_experts_get_f_slot).  The same refusals as those three getters, with their codes; besides,
 * SGP_E_BADARG for an unknown store and SGP_E_STATE when the experts did not come from sgp_experts_upload_grouped or its
 * _device form (other uploads have no row order to restore).  dF_out (n doubles) must be device memory on the context's
 * device (SGP_E_BADARG otherwise, before the launch).  Returns when the modes are written. */
enum { SGP_MODES_BINARY = 0, SGP_MODES_CLASS = 1, SGP_MODES_SLOT = 2 };
int sgp_experts_get_f_rows_device(sgp_ctx* ctx, int32_t store, int32_t index, double* dF_out);

/* Cross-validation over one-vs-rest (Spark's CrossValidator over OneVsRest): the Laplace objective of n_eval slots over
 * the training sets of the last sgp_experts_upload_folds, in one launch per kernel family.  Listed slot i evaluates, with
 * no other inputs, the training set sets[i], the labels (y == classes[i]), kernels[i] with hypers[i * n_hypers ...] (the
 * same kernel structure and descriptor layout for every slot), and the latent modes of mode slot mode_slots[i], which it
 * warm-starts from and writes back.  Sets and classes may repeat; mode slots are distinct and in [0, n_mode_slots).  The
 * binary classifier is class 1 over 0/1 labels.
 * Contract: slot i's value, gradient and modes equal, bit for bit, what sgp_laplace_nll_any_size returns after
 * sgp_experts_upload_grouped(X[fold_of != k], y[fold_of != k] == c, dataset_size_for_expert), k = sets[i] and
 * c = classes[i], with the same modes, on either kernel and whichever other slots share the call.  The kernel is chosen
 * per set, by sgp_laplace_nll_any_size's rule on the set's largest expert (on chip up to 117 points, else global memory),
 * so a call whose sets straddle that edge makes two launches, one per family; each slot's results land in its list
 * position.  sgp_last_laplace_path is 1 if the global-memory kernel ran.
 * The modes live in a store of their own, [n_mode_slots][rows of the largest set], indexed from each set's first row
 * (apart from the stores of sgp_laplace_nll_classes and sgp_laplace_nll_slots_any_size: no entry moves another's modes):
 * allocated on first use, zero after every sgp_experts_upload* and whenever n_mode_slots changes; the modes of mode slots
 * not listed are left as they are.  With a communicator: one ncclAllReduce of the n_eval rows and n_eval status words.
 * Errors, all before any allocation or launch: SGP_E_STATE without a fold upload; SGP_E_BADARG for a set outside
 * [0, n_folds), a repeated or out-of-range mode slot, a negative class, n_eval outside [1, 65535] or above n_mode_slots,
 * a structure that differs between slots, or a listed set's expert above 46336 points; SGP_E_SINGULAR for tol >= 1,
 * every mode left as it was; SGP_E_NOMEM when the store or one global-memory workspace slice exceeds the device's free
 * memory.  SGP_E_NOT_PD names the mode slot of the first listed slot whose B broke down. */
int sgp_laplace_nll_fold_slots_any_size(sgp_ctx* ctx, int32_t n_mode_slots, const int32_t* mode_slots,
                                        const int32_t* sets, const int32_t* classes, int32_t n_eval,
                                        const sgp_kernel_desc* kernels, const sgp_hyper* hypers, int32_t n_hypers,
                                        double tol, double* neg_log_z_out /* n_eval */,
                                        double* grad_out /* n_eval x n_hypers */);
/* Mode slot mode_slot's latent modes on fold set `set` (its N_k rows, in the set's packed expert-major order).
 * SGP_E_STATE without a fold upload or before the first sgp_laplace_nll_fold_slots_any_size after it; SGP_E_BADARG for a
 * set outside [0, n_folds) or a mode slot outside [0, n_mode_slots). */
int sgp_experts_get_f_fold_slot(sgp_ctx* ctx, int32_t set, int32_t mode_slot, double* f_out);
/* The same modes in the set's training-row order (the order of X[fold_of != set]), written to device memory dF_out (N_k
 * doubles on the context's device: SGP_E_BADARG otherwise, before the launch).  The refusals of
 * sgp_experts_get_f_fold_slot.  Returns when the modes are written.  (sgp_experts_get_f_rows_device refuses a fold
 * upload.) */
int sgp_experts_get_f_fold_rows_device(sgp_ctx* ctx, int32_t set, int32_t mode_slot, double* dF_out);

/* Installs a caller-supplied (vector v, m x m matrix M, row-major) in place of the pair sgp_magic computes, so that
 * sgp_predict returns  mean_t = k(x_t, Z) . v  and  var_t = selfKernel + k(x_t, Z) M k(x_t, Z)^T  for them.  M need not be
 * bit-symmetric: the variance is the quadratic form of M itself.  This is the per-point part of
 * GreedilyOptimizingActiveSetProvider.getNext (commons/ActiveSetProvider.scala:109-113: p_i, q_i, mu_i are exactly such
 * forms with M = inv(K_mm), inv(sigma2 K_mm + G) and v = magicVector).  Needs sgp_stats_begin. */
int sgp_set_magic(sgp_ctx* ctx, const double* v, const double* M);

/* ---- prediction:  GPC:121-125 for a block of test vectors ----------------------------------- */
/* mean_t = k(x_t, Z) . magicVector ;  var_t = selfKernel + k(x_t,Z) magicMatrix k(x_t,Z)^T, all in fp64 (kernel
 * elements on the CUDA cores, the quadratic form on fp64 tensor cores over the packed triangle of M + M^T).
 * X: n x d row-major fp64 host.  var_out may be NULL (mean only: the cross kernel never reaches device memory).
 * SGP_E_STATE before sgp_magic / sgp_set_magic; n = 0 is a no-op.  A point's outputs do not depend on the call it
 * arrives in: host and device entry, fp32 input and its fp64 upcast, one call or a split, with or without var_out (the
 * mean) give the same bits.  Neither entry changes the statistics of an open begin..finish window. */
int sgp_predict(sgp_ctx* ctx, const double* X, int64_t n, double* mean_out, double* var_out);
/* Same, points already resident in device memory: dX is n x d row-major (fp64, or fp32 when x_is_f32 != 0), dMean and
 * dVar (may be NULL) are device pointers.  Asynchronous on the context's stream: synchronise with sgp_sync before reading
 * the outputs. */
int sgp_predict_device(sgp_ctx* ctx, const void* dX, int32_t x_is_f32, int64_t n, double* dMean, double* dVar);

/* ---- averaged predictive probability (GPML eq. 3.25) with commons/util/Integrator.scala's quadrature ---------------- */
/* The n-node Gauss-Hermite rule for the weight exp(-x^2): sum_i weights[i] f(nodes[i]) ~ int f(x) exp(-x^2) dx.  Nodes
 * ascending, exactly antisymmetric (nodes[i] == -nodes[n-1-i]); weights exactly symmetric.  Host code, no context, no
 * GPU.  SGP_E_BADARG for n outside [1, 256] or a NULL output. */
int sgp_gauss_hermite_rule(int32_t n, double* nodes, double* weights);
/* p_t = (1/sqrt(pi)) sum_i w_i sigmoid(mean_t + sqrt(2 var_t) x_i), sigmoid(z) = 1/(1 + exp(-z)), with the n_nodes-node
 * rule (x_i, w_i) of sgp_gauss_hermite_rule and (mean_t, var_t) bit for bit what sgp_predict returns (var_t includes the
 * white-noise part of selfKernel): Integrator.expectedOfFunctionOfNormal(mean_t, var_t, sigmoid), the probability of
 * class 1 averaged over the latent posterior.  One deviation: var_t < 0 (rounding, or a caller's sgp_set_magic pair) is
 * taken as 0, so that p_t = sigmoid(mean_t) times the rule's weight sum / sqrt(pi), where the Integrator would return
 * NaN; a NaN mean or variance gives NaN.  The quadrature is fused into the variance pass: the call makes the launches of
 * an sgp_predict with var_out.  mean_out and var_out may be NULL.  Refuses what sgp_predict refuses, with the same codes,
 * and n_nodes outside [1, 256] (SGP_E_BADARG).  A point's outputs do not depend on the call it arrives in, as for
 * sgp_predict. */
int sgp_predict_probability(sgp_ctx* ctx, const double* X, int64_t n, int32_t n_nodes, double* p_out, double* mean_out,
                            double* var_out);
/* Same, points and outputs in device memory (dX fp64, or fp32 when x_is_f32 != 0; dMean and dVar may be NULL); every
 * pointer must be device memory on the context's device (SGP_E_BADARG otherwise, before any launch).  Asynchronous on
 * the context's stream: synchronise with sgp_sync before reading the outputs. */
int sgp_predict_probability_device(sgp_ctx* ctx, const void* dX, int32_t x_is_f32, int64_t n, int32_t n_nodes,
                                   double* dP, double* dMean, double* dVar);

/* ---- introspection (tests / bench) ---------------------------------------------------------- */
/* Number of kernels this library launched on ctx since creation. */
int64_t sgp_launch_count(const sgp_ctx* ctx);
/* Device time (ms, CUDA events on the context's stream) of the Gram kernel launches since the last
 * sgp_stats_begin, and how many there were. */
int sgp_gram_kernel_time(sgp_ctx* ctx, double* total_ms, int64_t* launches);
/* Device-side stopwatch on the context's compute stream (CUDA events; torch.cuda.Event cannot see this
 * stream).  slot in [0, 8): sgp_event_record enqueues an event; sgp_event_elapsed_ms waits for both. */
int sgp_event_record(sgp_ctx* ctx, int slot);
int sgp_event_elapsed_ms(sgp_ctx* ctx, int slot_start, int slot_stop, double* ms);
/* Which kernel the last statistics launch used: SGP_PREC_F64, SGP_PREC_F64_STRICT, SGP_PREC_I8 or SGP_PREC_I8_DIRECT
 * (-1: none yet). */
int sgp_last_path(const sgp_ctx* ctx);
/* Which path the last sgp_magic took: 1 = Cholesky for both A and K_mm (success of dpotrf IS the reference's positive-
 * definiteness check PGPH:62-65), 0 = the reference's literal sequence (dsyevd eigenvalue check, LU solves) because a
 * Cholesky factorization broke down, -1 = sgp_magic has not run. */
int sgp_last_tail_path(const sgp_ctx* ctx);
/* Which path the last sgp_bcm_nll took: 0 = on-chip Cholesky kernel, 1 = global-memory LU (reference arithmetic). */
int sgp_last_bcm_path(const sgp_ctx* ctx);
/* Which kernel the last sgp_laplace_nll* call ran: 0 = on chip (laplace_kernel), 1 = global memory (experts above the
 * on-chip limit, *_any_size entries only), -1 = none has run on this context. */
int sgp_last_laplace_path(const sgp_ctx* ctx);
/* Debug aid for SGP_PREC_I8: the first call arms a dump; later calls return, for the first 64-point unit of
 * the first CTA of the last launch, T = -q*log2(e) (128 active rows x 64 points, fp32) and the fixed-point words
 * (0x4B000000 | (u + 0x4040)), u = s2*2^15 + s1*2^7 + s0 in balanced digits. */
int sgp_debug_i8_tile(sgp_ctx* ctx, float* T_out /* 128*64 */, uint32_t* w_out /* 128*64 */);
/* GreedilyOptimizingActiveSetProvider (commons/ActiveSetProvider.scala:58-139) with rank-1 updates: selects m_target points
 * of the shard X (n x d fp64, host) by the reference's forward selection and returns their row indices.  The reference
 * recomputes the statistics, two m x m inverses and three quadratic forms per candidate in every round (ASP:83-137); here
 * the cross kernel stays on the device and grows by one row per round, the inverses and the per-point p_i, q_i, mu_i
 * (ASP:109-113) are updated through the bordered-matrix identities: O(n m) per round.  Selection semantics are the
 * reference's (point i belongs to expert i % n_experts, per-expert fold with later-wins ties and NaN poisoning, first
 * expert with the maximal score, sigma2 = the kernel's whiteNoiseVar, ASP:76, 108-135).  first_index replaces
 * takeSample(1, seed) (ASP:70).  Needs 8 n (m_target + d + 8) bytes of device memory: SGP_E_NOMEM otherwise.
 * Errors: SGP_E_NOT_PD as assertSymPositiveDefinite (PGPH:62-65), SGP_E_BADARG "empty.max" when every expert is poisoned. */
int sgp_greedy_active_set(sgp_ctx* ctx, const sgp_kernel_desc* kernel, const double* X, const double* y, int64_t n,
                          int32_t d, int64_t n_experts, int64_t first_index, int32_t m_target, int64_t* indices_out);
/* sgp_greedy_active_set on dX (n x d fp64) and dy (n fp64) in device memory, read in place instead of copied in: the same
 * selection, indices and errors; 8 n (d + 1) bytes less device memory.  indices_out stays host memory. dX and dy
 * must be device (or managed) memory on the
 * context's device: anything else is refused with SGP_E_BADARG (checked with cudaPointerGetAttributes) before any
 * allocation or launch. */
int sgp_greedy_active_set_device(sgp_ctx* ctx, const sgp_kernel_desc* kernel, const double* dX, const double* dy,
                                 int64_t n, int32_t d, int64_t n_experts, int64_t first_index, int32_t m_target,
                                 int64_t* indices_out);

/* KMeansActiveSetProvider (commons/ActiveSetProvider.scala:22-46): Spark 3.1 MLlib KMeans with the reference's settings
 * (k-means|| seeding with 2 steps, Euclidean distance, unit weights; DESIGN.md 4.7 restates the algorithm).  X: n x d
 * row-major in HOST memory, fp64 or fp32 (x_is_f32 != 0), uploaded once.  init_centers (k x d fp64) replaces the seeding
 * (mllib's setInitialModel); NULL: k-means|| from `seed` through the library's counter-based generator (Spark's
 * XORShift streams depend on the partitioning and are not reproduced).  Lloyd runs until max_iter iterations or until
 * every non-empty cluster moved by at most tol (squared distance <= tol^2); an empty cluster keeps its centre.
 * Outputs (host): centers_out (k_out x d; k_out < k when the data have fewer distinct points), labels_out (n, or NULL)
 * and cost_out (sum of squared distances) of the last assignment pass -- against the centres before the last update, as
 * Spark's trainingCost --, iterations_out.  Distances are fp32 direct form on points and centres shifted by a common
 * origin and scaled by a common power of two 2^s in fp64 (then returned times 2^-2s, in fp64); centre sums are fp64 in
 * point order: two calls return identical bits.  s = 0 while the largest column standard deviation sd is within
 * [2^-16, 2^16]; otherwise s brings it into [1, 2), so data whose largest sd lies in [2^-511, 2^512) (about 1.5e-154 to
 * 1.3e154) keep their spread in the fp32 distances at any scale.  Errors: SGP_E_BADARG for k < 2, max_iter < 0, tol < 0
 * or NaN, n < 1, d < 1, n > 2^31 - 1 and NaN / infinity in X; SGP_E_RANGE before any k-means step when the largest sd is
 * outside [2^-511, 2^512) or a column's sum of squares overflows fp64 (|x| above about 1e154), and at the end when a
 * point's squared distance to its nearest centre is beyond the fp32 range after the prescale (above about 3.4e38 4^-s:
 * initial centres far outside the data's spread).  Works outside any begin..finish window and leaves an open window's
 * statistics untouched; rank-local (no communicator). */
int sgp_kmeans(sgp_ctx* ctx, const void* X, int32_t x_is_f32, int64_t n, int32_t d, int32_t k, int32_t max_iter,
               double tol, int64_t seed, const double* init_centers /* k x d, or NULL: k-means|| */,
               double* centers_out /* k x d */, int32_t* k_out, int32_t* labels_out /* n, or NULL */,
               int32_t* iterations_out, double* cost_out);
/* sgp_kmeans on dX in device memory (fp64, or fp32 when x_is_f32 != 0), read in place instead of copied in: the same
 * algorithm and the same bits in every output; the few rows the host reads (the seeding's candidates) are gathered on
 * the device.  init_centers and every output stay host memory.  dX must be device (or managed) memory on the context's
 * device: SGP_E_BADARG otherwise, before any allocation or launch. */
int sgp_kmeans_device(sgp_ctx* ctx, const void* dX, int32_t x_is_f32, int64_t n, int32_t d, int32_t k, int32_t max_iter,
                      double tol, int64_t seed, const double* init_centers /* k x d, or NULL: k-means|| */,
                      double* centers_out /* k x d */, int32_t* k_out, int32_t* labels_out /* n, or NULL */,
                      int32_t* iterations_out, double* cost_out);

/* sgp_kmeans on the concatenation of the ranks' rows over the context's communicator (sgp_comm_init): this rank holds the
 * global rows [offset, offset + n) of n_total, the ranks' blocks following each other in rank order (n = 0 is allowed).
 * The algorithm is sgp_kmeans's on the n_total rows: draws at the global row index, the first centre from its owner, the
 * origin's column sums and the k-means|| cost sums as each rank's fixed-order sum summed over the ranks, the chosen
 * candidates gathered in global index order (their rows' bit patterns summed as integers, so exact), candidate weights as
 * int64 counts summed over the ranks, and each Lloyd step's per-cluster fp64 sums (point order on each rank) and counts
 * summed over the ranks before every rank moves the centres by sum * (1 / count).  Everything that follows from the
 * summed values (the distinct filter, the local k-means++ and its Lloyd iterations, convergence) runs identically on
 * every rank, so every rank returns the same centres, k_out, iterations and cost; labels_out gets this rank's n labels.
 * With one rank, or without a communicator, the outputs are sgp_kmeans's on X bit for bit; on data whose fp32 distances
 * and fp64 sums are exact (integer coordinates), they are sgp_kmeans's on the concatenation at any number of ranks.
 * Every rank must make the call with the same d, k, max_iter, tol, seed, n_total and initial centres.  Refusals: those of
 * sgp_kmeans on every rank alike (the arguments every rank shares are checked first; the layout -- n, offset, a null or
 * foreign X -- and NaN / infinity are summed over the ranks before any rank refuses, so every rank refuses together;
 * the prescale comes from the summed statistics, and SGP_E_RANGE from a flag summed over the ranks, so both agree).
 * SGP_E_NOMEM and CUDA errors stay rank-local. */
int sgp_kmeans_sharded(sgp_ctx* ctx, const void* X, int32_t x_is_f32, int64_t n, int64_t offset, int64_t n_total,
                       int32_t d, int32_t k, int32_t max_iter, double tol, int64_t seed,
                       const double* init_centers /* k x d, or NULL */, double* centers_out /* k x d */, int32_t* k_out,
                       int32_t* labels_out /* n, or NULL */, int32_t* iterations_out, double* cost_out);
/* sgp_kmeans_sharded on dX in device memory, read in place (as sgp_kmeans_device). */
int sgp_kmeans_sharded_device(sgp_ctx* ctx, const void* dX, int32_t x_is_f32, int64_t n, int64_t offset, int64_t n_total,
                              int32_t d, int32_t k, int32_t max_iter, double tol, int64_t seed,
                              const double* init_centers, double* centers_out, int32_t* k_out, int32_t* labels_out,
                              int32_t* iterations_out, double* cost_out);

/* Evaluate K(X_test, Z) (n x m row-major fp64 out) with the current kernel -- the `crossKernel`
 * contract of kernel/Kernel.scala:69-74 (used by the golden-vector tests). */
int sgp_cross_kernel(sgp_ctx* ctx, const double* X, int64_t n, double* K_out);

/* ---- K_nm sweep (BASELINE configs[4]: the HBM-bound member of the family) ---------------------------------------
 * Materialises crossKernel(X) against the active set of the last sgp_stats_begin: K[i][j] = k(x_i, z_j), n x m row-major,
 * in FP32; sgp_cross_kernel is the fp64 form.  The relative error of an element grows with the scaled squared norms
 * s = |x^|^2 + |z^|^2 of its pair (x^ = sqrt(log2 e) beta (x - active-set mean)): measured up to 5.2e-6 at s ~ 13 (H100),
 * bounded in the tests by 3e-7 + 24 ln2 2^-24 s.  What commons/ActiveSetProvider.scala:90-92
 * materialises and caches per expert (transposed) and commons/GaussianProcessCommons.scala:121-125 evaluates row by row.
 * Tensor-core distance contraction + exp + coalesced stores; kernels with one non-Eye term, d <= 32.
 * The host form returns SGP_E_RANGE if the active set or this call's points leave the operand range (scaled squared
 * norm above 4096).
 * _device: X (fp32 / fp64) and K_out are device pointers.  It is asynchronous on the context's stream (synchronise with
 * sgp_sync before reading K_out) and reports no range errors: out-of-range rows come back as garbage.
 * Neither form changes the statistics of an open begin..finish window. */
int sgp_kmn_sweep(sgp_ctx* ctx, const void* X, int32_t x_is_f32, int64_t n, float* K_out);
int sgp_kmn_sweep_device(sgp_ctx* ctx, const void* dX, int32_t x_is_f32, int64_t n, float* dK_out);

/* ---- Kernel evaluation: crossKernel, trainingKernel, trainingKernelAndDerivative (kernel/Kernel.scala:12-98) ---------
 * Evaluates `kernel` on the vectors passed in, in fp64; no context state is read or changed (an open begin..finish
 * window's statistics and status and an installed magic pair stay as they are).
 *   SGP_KEVAL_CROSS:    K[i][j] = k(A_i, B_j), n x m row-major.  Eye terms contribute nothing (Kernel.scala:157).  Equal,
 *                       bit for bit, to sgp_cross_kernel on the same kernel with B as its active set.
 *   SGP_KEVAL_TRAINING: B must be NULL and m == n: K = k(A, A) plus every Eye term's scale on the diagonal
 *                       (Kernel.scala:151), exactly symmetric.
 * dK_out (n_hypers x n x m, or NULL to skip): dK_out[h] = dK / d theta_h, h in the order of `hypers`, which must be the
 * kernel's descriptors as sgp_bcm_nll takes them: one ARD_BETA per feature of every ARD term and one RBF_SIGMA per RBF
 * term, each with the term's own value, and any SCALE descriptors.  ARD beta_k of term t: -2 beta_k (a_k - b_k)^2 C_t e_t
 * (ARDRBFKernel.scala:61-79); RBF sigma: |a - b|^2 / sigma^3 C_t e_t (RBFKernel.scala:56-64); SCALE: sum_t coef_t times
 * term t's element, Eye terms only on the TRAINING diagonal (ScalarTimesKernel.scala:93-97).  In TRAINING mode every dK
 * is exactly symmetric too.
 * A is fp64, or fp32 when a_is_f32 (converted to fp64 first: the same bits as its fp64 upcast).  An element's arithmetic
 * does not depend on how the rows are split over calls or windows.
 * SGP_E_BADARG, before any allocation or launch: n, m or d < 1; NULL A or K_out; a mode outside {CROSS, TRAINING}; B
 * missing in CROSS or given in TRAINING; descriptors that do not match the kernel; a kernel with no terms (or more than
 * 4 non-Eye terms); an output beyond 64-bit sizes.
 * Host entry: A, B and the outputs are host memory.  Rows of A go through the device in windows whose K and dK stay
 * within 256 MiB (at least one row); B (TRAINING: A) is copied to the device once.  SGP_E_NOMEM, before any
 * allocation, when the windows and that copy do not fit in free device memory.
 * _device: A, B (fp64) and both outputs are device (or managed) memory on the context's device, SGP_E_BADARG otherwise;
 * asynchronous on the context's stream (sgp_sync before reading the outputs). */
enum { SGP_KEVAL_CROSS = 0, SGP_KEVAL_TRAINING = 1 };
int sgp_kernel_eval(sgp_ctx* ctx, const sgp_kernel_desc* kernel, const sgp_hyper* hypers, int32_t n_hypers, const void* A,
                    int32_t a_is_f32, int64_t n, const double* B, int32_t m, int32_t d, int32_t mode,
                    double* K_out /* n x m */, double* dK_out /* n_hypers x n x m, or NULL */);
int sgp_kernel_eval_device(sgp_ctx* ctx, const sgp_kernel_desc* kernel, const sgp_hyper* hypers, int32_t n_hypers,
                           const void* dA, int32_t a_is_f32, int64_t n, const double* dB, int32_t m, int32_t d,
                           int32_t mode, double* dK_out /* n x m */, double* ddK_out /* n_hypers x n x m, or NULL */);

/* ---- Feature standardisation: commons/util/Scaling.scala:10-25 on device-resident rows -----------------------------
 * dX is n x d row-major in device memory on the context's device, fp64 (x_is_f32 = 0) or fp32 (x_is_f32 = 1), read in
 * place on the context's stream.  Refused with SGP_E_BADARG before any allocation or launch: x_is_f32 other than 0 or 1,
 * n < 0, d < 1, and where n > 0 a null dX or a dX that is not device (or managed) memory on the context's device.  n = 0
 * launches nothing.  Work outside any begin..finish window and leave its statistics untouched; rank-local.
 *
 * sgp_column_sums_device: out[k] (host, d values) = sum_i x_ik, or with center (host, d values, or NULL)
 * sum_i (x_ik - center_k)^2, every x converted exactly to fp64 and every subtraction and square rounded once.  The sum
 * order is fixed: rows go in blocks of 2048, each block gets one fp64 partial per column, and the partials are added in
 * block order, so the same inputs give the same bits on any H100 whatever the grid or the other work on the GPU.  n = 0
 * writes d zeros.  Returns when out is written (SGP_E_BADARG also for a null out). */
int sgp_column_sums_device(sgp_ctx* ctx, const void* dX, int32_t x_is_f32, int64_t n, int32_t d, const double* center,
                           double* out);
/* sgp_scale_apply_device: dY[i][k] = (x_ik - mean_k) / sd_k (n x d row-major fp64, device memory on the context's
 * device) with mean and sd host arrays of d values: a correctly rounded fp64 subtraction, then a correctly rounded
 * division (the reference's operation order; no reciprocal), so every element equals the host formula's on the same mean
 * and sd.  Refuses, besides the above, a null mean, sd or dY and a dY that is not device memory on the context's device,
 * where n > 0.  Asynchronous on the context's stream: synchronise with sgp_sync before reading dY. */
int sgp_scale_apply_device(sgp_ctx* ctx, const void* dX, int32_t x_is_f32, int64_t n, int32_t d, const double* mean,
                           const double* sd, double* dY);

#ifdef __cplusplus
}
#endif
#endif /* SGP_H_ */
