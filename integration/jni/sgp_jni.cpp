// JNI glue: org.apache.spark.ml.commons.NativeProjectedProcess  ->  the C-ABI of include/sgp.h.
// Not compiled in this repository's build (there is no JDK in the image): `__has_include(<jni.h>)` guards it so that
// `g++ -shared -fPIC -I$JAVA_HOME/include -I$JAVA_HOME/include/linux -Iinclude integration/jni/sgp_jni.cpp
//      -L spark_gp_b200 -lsgp -o libsgp_jni.so` builds it where a JDK exists.
// Arrays: Get<Primitive>ArrayElements copies/pins on the JVM side; the native context owns every device buffer.
#if __has_include(<jni.h>)
#include <jni.h>

#include <string>
#include <vector>

#include "../../include/sgp.h"

namespace {
// Every failure surfaces as ONE top-level exception class with a (String) constructor,
// org.apache.spark.ml.commons.SgpNativeException, whose message starts with "SGP<code>: ".  The Scala shim
// (NativeProjectedProcess.rethrow) turns the code back into the reference's exception types -- NotPositiveDefiniteException
// is an inner class of the trait ProjectedGaussianProcessHelper (PGPH:9-11) and cannot be constructed from JNI with
// ThrowNew (no (String) constructor, needs the outer instance).
void throw_for(JNIEnv* env, sgp_ctx* ctx, int rc) {
  std::string msg = "SGP" + std::to_string(rc) + ": " + sgp_last_error(ctx);
  jclass cls = env->FindClass("org/apache/spark/ml/commons/SgpNativeException");
  if (cls == nullptr) { env->ExceptionClear(); cls = env->FindClass("java/lang/RuntimeException"); }
  env->ThrowNew(cls, msg.c_str());
}
}  // namespace

extern "C" {

JNIEXPORT jlong JNICALL Java_org_apache_spark_ml_commons_NativeProjectedProcess_create(JNIEnv* env, jclass, jint device) {
  sgp_ctx* ctx = nullptr;
  const int rc = sgp_ctx_create(&ctx, device);
  if (rc != SGP_OK) { throw_for(env, nullptr, rc); return 0; }
  return reinterpret_cast<jlong>(ctx);
}

JNIEXPORT void JNICALL Java_org_apache_spark_ml_commons_NativeProjectedProcess_destroy(JNIEnv*, jclass, jlong h) {
  sgp_ctx_destroy(reinterpret_cast<sgp_ctx*>(h));
}

// terms: parallel arrays describing the flattened kernel (type, scale, sigma) + concatenated ARD betas (d each)
JNIEXPORT void JNICALL Java_org_apache_spark_ml_commons_NativeProjectedProcess_begin(
    JNIEnv* env, jclass, jlong h, jintArray types, jdoubleArray scales, jdoubleArray sigmas, jdoubleArray betas,
    jdoubleArray activeSet, jint m, jint d) {
  sgp_ctx* ctx = reinterpret_cast<sgp_ctx*>(h);
  const jsize nt = env->GetArrayLength(types);
  jint* ty = env->GetIntArrayElements(types, nullptr);
  jdouble* sc = env->GetDoubleArrayElements(scales, nullptr);
  jdouble* sg = env->GetDoubleArrayElements(sigmas, nullptr);
  jdouble* be = env->GetDoubleArrayElements(betas, nullptr);
  jdouble* z = env->GetDoubleArrayElements(activeSet, nullptr);
  std::vector<sgp_kernel_term> terms(nt);
  int ard = 0;
  for (jsize t = 0; t < nt; ++t) {
    terms[t].type = ty[t]; terms[t].reserved = 0; terms[t].scale = sc[t]; terms[t].sigma = sg[t];
    terms[t].beta = (ty[t] == SGP_TERM_ARD) ? be + (ard++) * d : nullptr;
  }
  sgp_kernel_desc desc{static_cast<int32_t>(nt), 0, terms.data()};
  const int rc = sgp_stats_begin(ctx, &desc, z, m, d);
  env->ReleaseIntArrayElements(types, ty, JNI_ABORT);
  env->ReleaseDoubleArrayElements(scales, sc, JNI_ABORT);
  env->ReleaseDoubleArrayElements(sigmas, sg, JNI_ABORT);
  env->ReleaseDoubleArrayElements(betas, be, JNI_ABORT);
  env->ReleaseDoubleArrayElements(activeSet, z, JNI_ABORT);
  if (rc != SGP_OK) throw_for(env, ctx, rc);
}

// one partition's points, packed row-major by the Scala side: X (n*d doubles), y (n doubles)
JNIEXPORT void JNICALL Java_org_apache_spark_ml_commons_NativeProjectedProcess_accumulate(
    JNIEnv* env, jclass, jlong h, jdoubleArray X, jdoubleArray y, jlong n) {
  sgp_ctx* ctx = reinterpret_cast<sgp_ctx*>(h);
  // NOT Get/ReleasePrimitiveArrayCritical: sgp_stats_accumulate allocates device memory, synchronises streams and does
  // blocking host->device copies -- none of which is allowed inside a JNI critical region (it can stall GC for the JVM)
  jdouble* x = env->GetDoubleArrayElements(X, nullptr);
  jdouble* yy = env->GetDoubleArrayElements(y, nullptr);
  const int rc = sgp_stats_accumulate(ctx, x, /*x_is_f32=*/0, yy, n);   // returns after the last H2D copy
  env->ReleaseDoubleArrayElements(y, yy, JNI_ABORT);
  env->ReleaseDoubleArrayElements(X, x, JNI_ABORT);
  if (rc != SGP_OK) throw_for(env, ctx, rc);
}

JNIEXPORT void JNICALL Java_org_apache_spark_ml_commons_NativeProjectedProcess_finish(
    JNIEnv* env, jclass, jlong h, jdoubleArray G, jdoubleArray b) {
  sgp_ctx* ctx = reinterpret_cast<sgp_ctx*>(h);
  jdouble* g = env->GetDoubleArrayElements(G, nullptr);
  jdouble* bb = env->GetDoubleArrayElements(b, nullptr);
  const int rc = sgp_stats_finish(ctx, g, bb);
  env->ReleaseDoubleArrayElements(G, g, 0);
  env->ReleaseDoubleArrayElements(b, bb, 0);
  if (rc != SGP_OK) throw_for(env, ctx, rc);
}

JNIEXPORT void JNICALL Java_org_apache_spark_ml_commons_NativeProjectedProcess_magic(
    JNIEnv* env, jclass, jlong h, jdoubleArray G, jdoubleArray b, jdoubleArray magicVector, jdoubleArray magicMatrix) {
  sgp_ctx* ctx = reinterpret_cast<sgp_ctx*>(h);
  jdouble* g = env->GetDoubleArrayElements(G, nullptr);
  jdouble* bb = env->GetDoubleArrayElements(b, nullptr);
  jdouble* mv = env->GetDoubleArrayElements(magicVector, nullptr);
  jdouble* mm = env->GetDoubleArrayElements(magicMatrix, nullptr);
  const int rc = sgp_magic(ctx, g, bb, mv, mm);
  env->ReleaseDoubleArrayElements(G, g, JNI_ABORT);
  env->ReleaseDoubleArrayElements(b, bb, JNI_ABORT);
  env->ReleaseDoubleArrayElements(magicVector, mv, 0);
  env->ReleaseDoubleArrayElements(magicMatrix, mm, 0);
  if (rc != SGP_OK) throw_for(env, ctx, rc);
}

// ---- prediction (GaussianProcessCommons.scala:121-125) ---------------------------------------------------------------
// M may come in Breeze's column-major order: k M k^T = k M^T k^T, and the library reads M through its symmetric part.
JNIEXPORT void JNICALL Java_org_apache_spark_ml_commons_NativeProjectedProcess_setMagic(
    JNIEnv* env, jclass, jlong h, jdoubleArray magicVector, jdoubleArray magicMatrix) {
  sgp_ctx* ctx = reinterpret_cast<sgp_ctx*>(h);
  jdouble* mv = env->GetDoubleArrayElements(magicVector, nullptr);
  jdouble* mm = env->GetDoubleArrayElements(magicMatrix, nullptr);
  const int rc = sgp_set_magic(ctx, mv, mm);          // copies both before returning
  env->ReleaseDoubleArrayElements(magicVector, mv, JNI_ABORT);
  env->ReleaseDoubleArrayElements(magicMatrix, mm, JNI_ABORT);
  if (rc != SGP_OK) throw_for(env, ctx, rc);
}

// a block of rows packed row-major by the Scala side: X (n*d doubles); var may be null (mean only)
JNIEXPORT void JNICALL Java_org_apache_spark_ml_commons_NativeProjectedProcess_predict(
    JNIEnv* env, jclass, jlong h, jdoubleArray X, jlong n, jdoubleArray mean, jdoubleArray var) {
  sgp_ctx* ctx = reinterpret_cast<sgp_ctx*>(h);
  jdouble* x = env->GetDoubleArrayElements(X, nullptr);   // not a critical region: sgp_predict copies and synchronises
  jdouble* mo = env->GetDoubleArrayElements(mean, nullptr);
  jdouble* vo = var ? env->GetDoubleArrayElements(var, nullptr) : nullptr;
  const int rc = sgp_predict(ctx, x, n, mo, vo);
  env->ReleaseDoubleArrayElements(X, x, JNI_ABORT);
  env->ReleaseDoubleArrayElements(mean, mo, 0);
  if (vo) env->ReleaseDoubleArrayElements(var, vo, 0);
  if (rc != SGP_OK) throw_for(env, ctx, rc);
}

// the probability of class 1 averaged over the latent posterior (Integrator.scala's Gauss-Hermite rule with `nodes`
// nodes) of a block of rows; mean and var may be null
JNIEXPORT void JNICALL Java_org_apache_spark_ml_commons_NativeProjectedProcess_predictProbability(
    JNIEnv* env, jclass, jlong h, jdoubleArray X, jlong n, jint nodes, jdoubleArray p, jdoubleArray mean,
    jdoubleArray var) {
  sgp_ctx* ctx = reinterpret_cast<sgp_ctx*>(h);
  jdouble* x = env->GetDoubleArrayElements(X, nullptr);
  jdouble* po = env->GetDoubleArrayElements(p, nullptr);
  jdouble* mo = mean ? env->GetDoubleArrayElements(mean, nullptr) : nullptr;
  jdouble* vo = var ? env->GetDoubleArrayElements(var, nullptr) : nullptr;
  const int rc = sgp_predict_probability(ctx, x, n, nodes, po, mo, vo);
  env->ReleaseDoubleArrayElements(X, x, JNI_ABORT);
  env->ReleaseDoubleArrayElements(p, po, 0);
  if (mo) env->ReleaseDoubleArrayElements(mean, mo, 0);
  if (vo) env->ReleaseDoubleArrayElements(var, vo, 0);
  if (rc != SGP_OK) throw_for(env, ctx, rc);
}

// ---- hyper-parameter objective (GaussianProcessCommons.scala:73-78 treeAggregate of likelihoodAndGradient) ----------
// experts of this executor, packed expert-major by the Scala side: X (n*d), y (n), offsets (E+1)
JNIEXPORT void JNICALL Java_org_apache_spark_ml_commons_NativeProjectedProcess_expertsUpload(
    JNIEnv* env, jclass, jlong h, jdoubleArray X, jdoubleArray y, jlongArray offsets, jint d) {
  sgp_ctx* ctx = reinterpret_cast<sgp_ctx*>(h);
  const jsize ne = env->GetArrayLength(offsets) - 1;
  jdouble* x = env->GetDoubleArrayElements(X, nullptr);
  jdouble* yy = env->GetDoubleArrayElements(y, nullptr);
  jlong* off = env->GetLongArrayElements(offsets, nullptr);
  static_assert(sizeof(jlong) == sizeof(int64_t), "jlong is 64 bit");
  const int rc = sgp_experts_upload(ctx, x, yy, reinterpret_cast<const int64_t*>(off), ne, d);
  env->ReleaseDoubleArrayElements(X, x, JNI_ABORT);
  env->ReleaseDoubleArrayElements(y, yy, JNI_ABORT);
  env->ReleaseLongArrayElements(offsets, off, JNI_ABORT);
  if (rc != SGP_OK) throw_for(env, ctx, rc);
}

namespace {
// Kernel terms + hyper-parameter descriptors from the parallel arrays NativeProjectedProcess.describe produces:
// hyper i = (kind, term, dim, value) and, for kind SCALE, a row of n_terms coefficients d(scale_t)/d(theta_i).
struct Objective {
  std::vector<sgp_kernel_term> terms;
  std::vector<sgp_hyper> hypers;
  sgp_kernel_desc desc;
};
void build_objective(Objective& o, jsize nt, const jint* ty, const jdouble* sc, const jdouble* sg, const jdouble* be, jint d,
                     jsize nh, const jint* hk, const jint* ht, const jint* hd, const jdouble* hv, const jdouble* hc) {
  o.terms.resize(nt);
  int ard = 0;
  for (jsize t = 0; t < nt; ++t) {
    o.terms[t].type = ty[t]; o.terms[t].reserved = 0; o.terms[t].scale = sc[t]; o.terms[t].sigma = sg[t];
    o.terms[t].beta = (ty[t] == SGP_TERM_ARD) ? be + (ard++) * d : nullptr;
  }
  o.desc = sgp_kernel_desc{static_cast<int32_t>(nt), 0, o.terms.data()};
  o.hypers.resize(nh);
  for (jsize i = 0; i < nh; ++i) {
    o.hypers[i].kind = hk[i]; o.hypers[i].term = ht[i]; o.hypers[i].dim = hd[i]; o.hypers[i].reserved = 0;
    o.hypers[i].value = hv[i];
    o.hypers[i].coef = (hk[i] == SGP_HYPER_SCALE) ? hc + static_cast<size_t>(i) * nt : nullptr;
  }
}
}  // namespace

// returns [value, grad_0 .. grad_{h-1}]: the BCM negative log marginal likelihood (GPR:55-68) when tol <= 0, the
// Laplace objective of the classifier (GPCls:74-129) when tol > 0 -- summed over this context's experts (and
// all-reduced over ranks if a communicator was attached)
JNIEXPORT jdoubleArray JNICALL Java_org_apache_spark_ml_commons_NativeProjectedProcess_objective(
    JNIEnv* env, jclass, jlong h, jintArray types, jdoubleArray scales, jdoubleArray sigmas, jdoubleArray betas, jint d,
    jintArray hKind, jintArray hTerm, jintArray hDim, jdoubleArray hValue, jdoubleArray hCoef, jdouble tol) {
  sgp_ctx* ctx = reinterpret_cast<sgp_ctx*>(h);
  const jsize nt = env->GetArrayLength(types), nh = env->GetArrayLength(hKind);
  jint* ty = env->GetIntArrayElements(types, nullptr);
  jdouble* sc = env->GetDoubleArrayElements(scales, nullptr);
  jdouble* sg = env->GetDoubleArrayElements(sigmas, nullptr);
  jdouble* be = env->GetDoubleArrayElements(betas, nullptr);
  jint* hk = env->GetIntArrayElements(hKind, nullptr);
  jint* ht = env->GetIntArrayElements(hTerm, nullptr);
  jint* hd = env->GetIntArrayElements(hDim, nullptr);
  jdouble* hv = env->GetDoubleArrayElements(hValue, nullptr);
  jdouble* hc = env->GetDoubleArrayElements(hCoef, nullptr);
  Objective o;
  build_objective(o, nt, ty, sc, sg, be, d, nh, hk, ht, hd, hv, hc);
  std::vector<double> out(1 + nh, 0.0);
  const int rc = (tol > 0.0) ? sgp_laplace_nll_any_size(ctx, &o.desc, o.hypers.data(), nh, tol, &out[0], out.data() + 1)
                             : sgp_bcm_nll(ctx, &o.desc, o.hypers.data(), nh, &out[0], out.data() + 1);
  env->ReleaseIntArrayElements(types, ty, JNI_ABORT);
  env->ReleaseDoubleArrayElements(scales, sc, JNI_ABORT);
  env->ReleaseDoubleArrayElements(sigmas, sg, JNI_ABORT);
  env->ReleaseDoubleArrayElements(betas, be, JNI_ABORT);
  env->ReleaseIntArrayElements(hKind, hk, JNI_ABORT);
  env->ReleaseIntArrayElements(hTerm, ht, JNI_ABORT);
  env->ReleaseIntArrayElements(hDim, hd, JNI_ABORT);
  env->ReleaseDoubleArrayElements(hValue, hv, JNI_ABORT);
  env->ReleaseDoubleArrayElements(hCoef, hc, JNI_ABORT);
  if (rc != SGP_OK) { throw_for(env, ctx, rc); return nullptr; }
  jdoubleArray res = env->NewDoubleArray(1 + nh);
  env->SetDoubleArrayRegion(res, 0, 1 + nh, out.data());
  return res;
}

// the classifier's latent modes f after optimisation (GPCls:61-66), in the packed expert-major order of expertsUpload
JNIEXPORT void JNICALL Java_org_apache_spark_ml_commons_NativeProjectedProcess_expertsGetF(JNIEnv* env, jclass, jlong h,
                                                                                          jdoubleArray f) {
  sgp_ctx* ctx = reinterpret_cast<sgp_ctx*>(h);
  jdouble* ff = env->GetDoubleArrayElements(f, nullptr);
  const int rc = sgp_experts_get_f(ctx, ff);
  env->ReleaseDoubleArrayElements(f, ff, 0);
  if (rc != SGP_OK) throw_for(env, ctx, rc);
}

// GreedilyOptimizingActiveSetProvider (ActiveSetProvider.scala:58-139) on one executor's points: row indices of the selected
// points (rank-1 updates on the device, sgp_greedy_active_set); firstIndex replaces takeSample(1, seed), ASP:70
JNIEXPORT jlongArray JNICALL Java_org_apache_spark_ml_commons_NativeProjectedProcess_greedyActiveSet(
    JNIEnv* env, jclass, jlong h, jintArray types, jdoubleArray scales, jdoubleArray sigmas, jdoubleArray betas,
    jdoubleArray X, jdoubleArray y, jlong n, jint d, jlong nExperts, jlong firstIndex, jint activeSetSize) {
  sgp_ctx* ctx = reinterpret_cast<sgp_ctx*>(h);
  const jsize nt = env->GetArrayLength(types);
  jint* ty = env->GetIntArrayElements(types, nullptr);
  jdouble* sc = env->GetDoubleArrayElements(scales, nullptr);
  jdouble* sg = env->GetDoubleArrayElements(sigmas, nullptr);
  jdouble* be = env->GetDoubleArrayElements(betas, nullptr);
  jdouble* xx = env->GetDoubleArrayElements(X, nullptr);
  jdouble* yy = env->GetDoubleArrayElements(y, nullptr);
  std::vector<sgp_kernel_term> terms(nt);
  int ard = 0;
  for (jsize t = 0; t < nt; ++t) {
    terms[t].type = ty[t]; terms[t].reserved = 0; terms[t].scale = sc[t]; terms[t].sigma = sg[t];
    terms[t].beta = (ty[t] == SGP_TERM_ARD) ? be + (ard++) * d : nullptr;
  }
  sgp_kernel_desc desc{static_cast<int32_t>(nt), 0, terms.data()};
  std::vector<int64_t> idx(activeSetSize);
  const int rc = sgp_greedy_active_set(ctx, &desc, xx, yy, n, d, nExperts, firstIndex, activeSetSize, idx.data());
  env->ReleaseIntArrayElements(types, ty, JNI_ABORT);
  env->ReleaseDoubleArrayElements(scales, sc, JNI_ABORT);
  env->ReleaseDoubleArrayElements(sigmas, sg, JNI_ABORT);
  env->ReleaseDoubleArrayElements(betas, be, JNI_ABORT);
  env->ReleaseDoubleArrayElements(X, xx, JNI_ABORT);
  env->ReleaseDoubleArrayElements(y, yy, JNI_ABORT);
  if (rc != SGP_OK) { throw_for(env, ctx, rc); return nullptr; }
  jlongArray res = env->NewLongArray(activeSetSize);
  static_assert(sizeof(jlong) == sizeof(int64_t), "jlong is 64 bits");
  env->SetLongArrayRegion(res, 0, activeSetSize, reinterpret_cast<const jlong*>(idx.data()));
  return res;
}

// KMeansActiveSetProvider (ActiveSetProvider.scala:22-46) on the collected points x (n x d row-major): Spark 3.1 MLlib KMeans
// (k-means|| + Lloyd, tol 1e-4) on the device, sgp_kmeans.  Returns k_out x d centres row-major (k_out < k when the data
// have fewer distinct points).
JNIEXPORT jdoubleArray JNICALL Java_org_apache_spark_ml_commons_NativeProjectedProcess_kmeansActiveSet(
    JNIEnv* env, jclass, jlong h, jdoubleArray X, jlong n, jint d, jint k, jint maxIter, jlong seed) {
  sgp_ctx* ctx = reinterpret_cast<sgp_ctx*>(h);
  jdouble* xx = env->GetDoubleArrayElements(X, nullptr);
  std::vector<double> centres(static_cast<size_t>(k > 0 ? k : 0) * (d > 0 ? d : 0));
  int32_t k_out = 0, iterations = 0;
  double cost = 0.0;
  const int rc = sgp_kmeans(ctx, xx, /*x_is_f32=*/0, n, d, k, maxIter, 1e-4, seed, nullptr, centres.data(), &k_out, nullptr,
                            &iterations, &cost);
  env->ReleaseDoubleArrayElements(X, xx, JNI_ABORT);
  if (rc != SGP_OK) { throw_for(env, ctx, rc); return nullptr; }
  const jsize len = static_cast<jsize>(k_out) * d;
  jdoubleArray res = env->NewDoubleArray(len);
  env->SetDoubleArrayRegion(res, 0, len, centres.data());
  return res;
}

}  // extern "C"
#endif  // __has_include(<jni.h>)
