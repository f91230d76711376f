/*
 * pio_als_jni.c -- JNI shim of the `native-als` module: binds org.apache.predictionio.nativeals.NativeALS$ (the Scala
 * object in ../scala/.../NativeALS.scala) to the C ABI of include/pio_als.h.  Nothing is computed here: primitive arrays
 * are pinned (GetPrimitiveArrayCritical) for the duration of one library call -- the library copies them to the device
 * itself -- and a status < 0 becomes a java.lang.RuntimeException carrying pio_als_last_error().
 *
 * Replaces the MLlib calls the reference templates make:
 *   new ALS()...run(mllibRatings)     examples/scala-parallel-recommendation/blacklist-items/src/main/scala/ALSAlgorithm.scala:76-86
 *   ALS.train / ALS.trainImplicit     examples/scala-parallel-ecommercerecommendation/train-with-rate-event/src/main/scala/ECommAlgorithm.scala:116-122,
 *                                     examples/scala-parallel-similarproduct/multi-events-multi-algos/src/main/scala/ALSAlgorithm.scala:121-128
 *   recommendProductsWithFilter       examples/scala-parallel-recommendation/blacklist-items/src/main/scala/ALSModel.scala:44-60
 *   cosine scan + getTopN             examples/scala-parallel-similarproduct/multi-events-multi-algos/src/main/scala/ALSAlgorithm.scala:138-234
 *   ALSModel.save / ALSModel.apply    examples/scala-parallel-recommendation/blacklist-items/src/main/scala/ALSModel.scala:63-100
 *
 * Build (needs a JDK for jni.h; see ../../../Makefile):
 *   cc -O2 -fPIC -shared -I$JAVA_HOME/include -I$JAVA_HOME/include/linux -I../../../../include \
 *      pio_als_jni.c -L<dir of libpio_als.so> -lpio_als -o libpio_als_jni.so
 * The build container of this repository has no JDK; tests/test_native_als_sources.py type-checks this file against
 * include/pio_als.h with a minimal stand-in for jni.h (tests/jni_mock/jni.h).
 */
#include <jni.h>
#include <stdint.h>
#include <string.h>

#include "pio_als.h"

#define JNAME(fn) Java_org_apache_predictionio_nativeals_NativeALS_00024_##fn
#define H(x) ((pio_als_handle*)(intptr_t)(x))

static void throw_rt(JNIEnv* env, const char* msg) {
  jclass c = (*env)->FindClass(env, "java/lang/RuntimeException");
  if (c) (*env)->ThrowNew(env, c, msg ? msg : "pio_als: unknown error");
}
static int check(JNIEnv* env, pio_als_handle* h, int rc) {
  if (rc != PIO_ALS_OK) throw_rt(env, pio_als_last_error(h));
  return rc;
}
static void* pin(JNIEnv* env, jarray a) { return a ? (*env)->GetPrimitiveArrayCritical(env, a, 0) : NULL; }
static void unpin(JNIEnv* env, jarray a, void* p, jint mode) {
  if (a && p) (*env)->ReleasePrimitiveArrayCritical(env, a, p, mode);
}

/* long create(int rank, boolean implicitPrefs, int nUsers, int nItems, double lambda, double alpha, long seed,
 *             int device, int worldSize, int worldRank, byte[] ncclId) */
JNIEXPORT jlong JNICALL JNAME(create)(JNIEnv* env, jobject self, jint rank, jboolean implicitPrefs, jint nUsers,
                                      jint nItems, jdouble lambda, jdouble alpha, jlong seed, jint device,
                                      jint worldSize, jint worldRank, jbyteArray ncclId) {
  pio_als_config cfg;
  pio_als_handle* h = NULL;
  (void)self;
  memset(&cfg, 0, sizeof cfg);
  cfg.abi_version = PIO_ALS_ABI_VERSION;
  cfg.rank = rank;
  cfg.implicit_prefs = implicitPrefs ? 1 : 0;
  cfg.n_users = nUsers;
  cfg.n_items = nItems;
  cfg.device = device;
  cfg.world_size = worldSize;
  cfg.world_rank = worldRank;
  cfg.init_mode = PIO_ALS_INIT_HASH;
  cfg.lambda = lambda;
  cfg.alpha = alpha;
  cfg.seed = seed;
  if (ncclId) (*env)->GetByteArrayRegion(env, ncclId, 0, 128, (jbyte*)cfg.nccl_id);
  if (pio_als_create(&cfg, &h) != PIO_ALS_OK) {
    throw_rt(env, pio_als_last_error(NULL));
    return 0;
  }
  return (jlong)(intptr_t)h;
}

/* void destroy(long h) */
JNIEXPORT void JNICALL JNAME(destroy)(JNIEnv* env, jobject self, jlong h) {
  (void)env; (void)self;
  pio_als_destroy(H(h));
}

/* byte[] ncclUniqueId(): created on the driver, shipped to the executors by a Spark broadcast */
JNIEXPORT jbyteArray JNICALL JNAME(ncclUniqueId)(JNIEnv* env, jobject self) {
  uint8_t id[128];
  jbyteArray out;
  (void)self;
  if (pio_als_nccl_unique_id(id) != PIO_ALS_OK) {
    throw_rt(env, pio_als_last_error(NULL));
    return NULL;
  }
  out = (*env)->NewByteArray(env, 128);
  if (out) (*env)->SetByteArrayRegion(env, out, 0, 128, (const jbyte*)id);
  return out;
}

/* void setRatings(long h, int[] user, int[] item, float[] rating, int dedup, long[] ts) */
JNIEXPORT void JNICALL JNAME(setRatings)(JNIEnv* env, jobject self, jlong h, jintArray user, jintArray item,
                                         jfloatArray rating, jint dedup, jlongArray ts) {
  jsize nnz = (*env)->GetArrayLength(env, user);
  jint* u = pin(env, user);
  jint* i = pin(env, item);
  jfloat* r = pin(env, rating);
  jlong* t = pin(env, ts);
  int rc = pio_als_set_ratings_coo(H(h), (const int32_t*)u, (const int32_t*)i, r, (int64_t)nnz, dedup, (const int64_t*)t);
  (void)self;
  unpin(env, ts, t, JNI_ABORT);
  unpin(env, rating, r, JNI_ABORT);
  unpin(env, item, i, JNI_ABORT);
  unpin(env, user, u, JNI_ABORT);
  check(env, H(h), rc);
}

/* void setInit(long h, float[] userFactors, float[] itemFactors)   (itemFactors may be null) */
JNIEXPORT void JNICALL JNAME(setInit)(JNIEnv* env, jobject self, jlong h, jfloatArray userFactors, jfloatArray itemFactors) {
  jfloat* uf = pin(env, userFactors);
  jfloat* itf = pin(env, itemFactors);
  int rc = pio_als_set_init(H(h), uf, itf);
  (void)self;
  unpin(env, itemFactors, itf, JNI_ABORT);
  unpin(env, userFactors, uf, JNI_ABORT);
  check(env, H(h), rc);
}

/* void run(long h, int iterations) */
JNIEXPORT void JNICALL JNAME(run)(JNIEnv* env, jobject self, jlong h, jint iterations) {
  (void)self;
  check(env, H(h), pio_als_run(H(h), iterations));
}

/* void getFactors(long h, float[] userOut, float[] itemOut, byte[] userHas, byte[] itemHas)   (any may be null) */
JNIEXPORT void JNICALL JNAME(getFactors)(JNIEnv* env, jobject self, jlong h, jfloatArray userOut, jfloatArray itemOut,
                                         jbyteArray userHas, jbyteArray itemHas) {
  jfloat* uo = pin(env, userOut);
  jfloat* io = pin(env, itemOut);
  jbyte* uh = pin(env, userHas);
  jbyte* ih = pin(env, itemHas);
  int rc = pio_als_get_factors(H(h), uo, io, (uint8_t*)uh, (uint8_t*)ih);
  (void)self;
  unpin(env, itemHas, ih, 0);
  unpin(env, userHas, uh, 0);
  unpin(env, itemOut, io, 0);
  unpin(env, userOut, uo, 0);
  check(env, H(h), rc);
}

/* void train(long h, int[] user, int[] item, float[] rating, int dedup, long[] ts, float[] userInit, float[] itemInit,
 *            int iterations, float[] userOut, float[] itemOut, byte[] userHas, byte[] itemHas)
 * One-shot ALS.train / ALS.trainImplicit: ratings in, factors out. */
JNIEXPORT void JNICALL JNAME(train)(JNIEnv* env, jobject self, jlong h, jintArray user, jintArray item, jfloatArray rating,
                                    jint dedup, jlongArray ts, jfloatArray userInit, jfloatArray itemInit, jint iterations,
                                    jfloatArray userOut, jfloatArray itemOut, jbyteArray userHas, jbyteArray itemHas) {
  JNAME(setRatings)(env, self, h, user, item, rating, dedup, ts);
  if ((*env)->ExceptionCheck(env)) return;
  if (userInit) {
    JNAME(setInit)(env, self, h, userInit, itemInit);
    if ((*env)->ExceptionCheck(env)) return;
  }
  JNAME(run)(env, self, h, iterations);
  if ((*env)->ExceptionCheck(env)) return;
  JNAME(getFactors)(env, self, h, userOut, itemOut, userHas, itemHas);
}

/* void recommend(long h, int[] users, int topk, byte[] itemMask, double[] itemWeight,
 *                int[] outItems, float[] outScores, int[] outCount)      outItems/outScores: users.length x topk */
JNIEXPORT void JNICALL JNAME(recommend)(JNIEnv* env, jobject self, jlong h, jintArray users, jint topk, jbyteArray itemMask,
                                        jdoubleArray itemWeight, jintArray outItems, jfloatArray outScores,
                                        jintArray outCount) {
  jsize n = (*env)->GetArrayLength(env, users);
  jint* us = pin(env, users);
  jbyte* mk = pin(env, itemMask);
  jdouble* wt = pin(env, itemWeight);
  jint* oi = pin(env, outItems);
  jfloat* os = pin(env, outScores);
  jint* oc = pin(env, outCount);
  int rc = pio_als_recommend(H(h), (const int32_t*)us, (int)n, topk, (const uint8_t*)mk, wt, (int32_t*)oi, os, (int32_t*)oc);
  (void)self;
  unpin(env, outCount, oc, 0);
  unpin(env, outScores, os, 0);
  unpin(env, outItems, oi, 0);
  unpin(env, itemWeight, wt, JNI_ABORT);
  unpin(env, itemMask, mk, JNI_ABORT);
  unpin(env, users, us, JNI_ABORT);
  check(env, H(h), rc);
}

/* int similar(long h, int[] queryItems, int topk, byte[] itemMask, double[] itemWeight, int flags,
 *             int[] outItems, float[] outScores)    returns the number of valid entries */
JNIEXPORT jint JNICALL JNAME(similar)(JNIEnv* env, jobject self, jlong h, jintArray queryItems, jint topk,
                                      jbyteArray itemMask, jdoubleArray itemWeight, jint flags, jintArray outItems,
                                      jfloatArray outScores) {
  jsize nq = (*env)->GetArrayLength(env, queryItems);
  int32_t cnt = 0;
  jint* q = pin(env, queryItems);
  jbyte* mk = pin(env, itemMask);
  jdouble* wt = pin(env, itemWeight);
  jint* oi = pin(env, outItems);
  jfloat* os = pin(env, outScores);
  int rc = pio_als_similar(H(h), (const int32_t*)q, (int)nq, topk, (const uint8_t*)mk, wt, flags, (int32_t*)oi, os, &cnt);
  (void)self;
  unpin(env, outScores, os, 0);
  unpin(env, outItems, oi, 0);
  unpin(env, itemWeight, wt, JNI_ABORT);
  unpin(env, itemMask, mk, JNI_ABORT);
  unpin(env, queryItems, q, JNI_ABORT);
  check(env, H(h), rc);
  return (jint)cnt;
}

/* void similarBatch(long h, long[] queryPtr, int[] queryItems, int topk, byte[] itemMask, double[] itemWeight, int flags,
 *                   int[] outItems, float[] outScores, int[] outCount)     queryPtr: nQueries + 1 offsets into queryItems */
JNIEXPORT void JNICALL JNAME(similarBatch)(JNIEnv* env, jobject self, jlong h, jlongArray queryPtr, jintArray queryItems,
                                           jint topk, jbyteArray itemMask, jdoubleArray itemWeight, jint flags,
                                           jintArray outItems, jfloatArray outScores, jintArray outCount) {
  jsize nqr = (*env)->GetArrayLength(env, queryPtr) - 1;
  jlong* qp = pin(env, queryPtr);
  jint* q = pin(env, queryItems);
  jbyte* mk = pin(env, itemMask);
  jdouble* wt = pin(env, itemWeight);
  jint* oi = pin(env, outItems);
  jfloat* os = pin(env, outScores);
  jint* oc = pin(env, outCount);
  int rc = pio_als_similar_batch(H(h), (const int64_t*)qp, (const int32_t*)q, (int)nqr, topk, (const uint8_t*)mk, wt, flags,
                                 (int32_t*)oi, os, (int32_t*)oc);
  (void)self;
  unpin(env, outCount, oc, 0);
  unpin(env, outScores, os, 0);
  unpin(env, outItems, oi, 0);
  unpin(env, itemWeight, wt, JNI_ABORT);
  unpin(env, itemMask, mk, JNI_ABORT);
  unpin(env, queryItems, q, JNI_ABORT);
  unpin(env, queryPtr, qp, JNI_ABORT);
  check(env, H(h), rc);
}

/* the filter arrays of the two filtered calls, pinned for one call (any of them may be null) */
typedef struct filter_pins {
  jlong *ex_ptr, *wl_ptr;
  jint *ex_items, *wl_items, *set_ix;
  jbyte *has_wl, *item_sets;
} filter_pins;
static pio_als_query_filter pin_filter(JNIEnv* env, filter_pins* p, jlongArray exPtr, jintArray exItems, jbyteArray hasWl,
                                       jlongArray wlPtr, jintArray wlItems, jintArray setIx, jbyteArray itemSets, jint nSets) {
  pio_als_query_filter f;
  p->ex_ptr = pin(env, exPtr);
  p->ex_items = pin(env, exItems);
  p->has_wl = pin(env, hasWl);
  p->wl_ptr = pin(env, wlPtr);
  p->wl_items = pin(env, wlItems);
  p->set_ix = pin(env, setIx);
  p->item_sets = pin(env, itemSets);
  f.ex_ptr = (const int64_t*)p->ex_ptr;
  f.ex_items = (const int32_t*)p->ex_items;
  f.has_wl = (const uint8_t*)p->has_wl;
  f.wl_ptr = (const int64_t*)p->wl_ptr;
  f.wl_items = (const int32_t*)p->wl_items;
  f.set_ix = (const int32_t*)p->set_ix;
  f.item_sets = (const uint8_t*)p->item_sets;
  f.n_sets = nSets;
  return f;
}
static void unpin_filter(JNIEnv* env, filter_pins* p, jlongArray exPtr, jintArray exItems, jbyteArray hasWl, jlongArray wlPtr,
                         jintArray wlItems, jintArray setIx, jbyteArray itemSets) {
  unpin(env, itemSets, p->item_sets, JNI_ABORT);
  unpin(env, setIx, p->set_ix, JNI_ABORT);
  unpin(env, wlItems, p->wl_items, JNI_ABORT);
  unpin(env, wlPtr, p->wl_ptr, JNI_ABORT);
  unpin(env, hasWl, p->has_wl, JNI_ABORT);
  unpin(env, exItems, p->ex_items, JNI_ABORT);
  unpin(env, exPtr, p->ex_ptr, JNI_ABORT);
}

/* void recommendFiltered(long h, int[] users, int topk, byte[] itemMask, double[] itemWeight, long[] exPtr, int[] exItems,
 *                        byte[] hasWl, long[] wlPtr, int[] wlItems, int[] setIx, byte[] itemSets, int nSets,
 *                        int[] outItems, float[] outScores, int[] outCount)       pio_als_query_filter as arrays */
JNIEXPORT void JNICALL JNAME(recommendFiltered)(JNIEnv* env, jobject self, jlong h, jintArray users, jint topk,
                                                jbyteArray itemMask, jdoubleArray itemWeight, jlongArray exPtr,
                                                jintArray exItems, jbyteArray hasWl, jlongArray wlPtr, jintArray wlItems,
                                                jintArray setIx, jbyteArray itemSets, jint nSets, jintArray outItems,
                                                jfloatArray outScores, jintArray outCount) {
  jsize n = (*env)->GetArrayLength(env, users);
  jint* us = pin(env, users);
  jbyte* mk = pin(env, itemMask);
  jdouble* wt = pin(env, itemWeight);
  jint* oi = pin(env, outItems);
  jfloat* os = pin(env, outScores);
  jint* oc = pin(env, outCount);
  filter_pins fp;
  pio_als_query_filter f = pin_filter(env, &fp, exPtr, exItems, hasWl, wlPtr, wlItems, setIx, itemSets, nSets);
  int rc = pio_als_recommend_filtered(H(h), (const int32_t*)us, (int)n, topk, (const uint8_t*)mk, wt, &f, (int32_t*)oi, os,
                                      (int32_t*)oc);
  (void)self;
  unpin_filter(env, &fp, exPtr, exItems, hasWl, wlPtr, wlItems, setIx, itemSets);
  unpin(env, outCount, oc, 0);
  unpin(env, outScores, os, 0);
  unpin(env, outItems, oi, 0);
  unpin(env, itemWeight, wt, JNI_ABORT);
  unpin(env, itemMask, mk, JNI_ABORT);
  unpin(env, users, us, JNI_ABORT);
  check(env, H(h), rc);
}

/* void similarBatchFiltered(long h, long[] queryPtr, int[] queryItems, int topk, byte[] itemMask, double[] itemWeight,
 *                           int flags, <the filter arrays as above>, int[] outItems, float[] outScores, int[] outCount) */
JNIEXPORT void JNICALL JNAME(similarBatchFiltered)(JNIEnv* env, jobject self, jlong h, jlongArray queryPtr,
                                                   jintArray queryItems, jint topk, jbyteArray itemMask,
                                                   jdoubleArray itemWeight, jint flags, jlongArray exPtr, jintArray exItems,
                                                   jbyteArray hasWl, jlongArray wlPtr, jintArray wlItems, jintArray setIx,
                                                   jbyteArray itemSets, jint nSets, jintArray outItems,
                                                   jfloatArray outScores, jintArray outCount) {
  jsize nqr = (*env)->GetArrayLength(env, queryPtr) - 1;
  jlong* qp = pin(env, queryPtr);
  jint* q = pin(env, queryItems);
  jbyte* mk = pin(env, itemMask);
  jdouble* wt = pin(env, itemWeight);
  jint* oi = pin(env, outItems);
  jfloat* os = pin(env, outScores);
  jint* oc = pin(env, outCount);
  filter_pins fp;
  pio_als_query_filter f = pin_filter(env, &fp, exPtr, exItems, hasWl, wlPtr, wlItems, setIx, itemSets, nSets);
  int rc = pio_als_similar_batch_filtered(H(h), (const int64_t*)qp, (const int32_t*)q, (int)nqr, topk, (const uint8_t*)mk, wt,
                                          flags, &f, (int32_t*)oi, os, (int32_t*)oc);
  (void)self;
  unpin_filter(env, &fp, exPtr, exItems, hasWl, wlPtr, wlItems, setIx, itemSets);
  unpin(env, outCount, oc, 0);
  unpin(env, outScores, os, 0);
  unpin(env, outItems, oi, 0);
  unpin(env, itemWeight, wt, JNI_ABORT);
  unpin(env, itemMask, mk, JNI_ABORT);
  unpin(env, queryItems, q, JNI_ABORT);
  unpin(env, queryPtr, qp, JNI_ABORT);
  check(env, H(h), rc);
}

/* void save(long h, String path) */
JNIEXPORT void JNICALL JNAME(save)(JNIEnv* env, jobject self, jlong h, jstring path) {
  const char* p = (*env)->GetStringUTFChars(env, path, NULL);
  int rc;
  (void)self;
  if (!p) return;
  rc = pio_als_save(H(h), p);
  (*env)->ReleaseStringUTFChars(env, path, p);
  check(env, H(h), rc);
}

/* long load(String path, int device) */
JNIEXPORT jlong JNICALL JNAME(load)(JNIEnv* env, jobject self, jstring path, jint device) {
  const char* p = (*env)->GetStringUTFChars(env, path, NULL);
  pio_als_handle* h = NULL;
  int rc;
  (void)self;
  if (!p) return 0;
  rc = pio_als_load(p, device, &h);
  (*env)->ReleaseStringUTFChars(env, path, p);
  if (rc != PIO_ALS_OK) {
    throw_rt(env, pio_als_last_error(NULL));
    return 0;
  }
  return (jlong)(intptr_t)h;
}

/* long importModel(int rank, int nUsers, int nItems, int device, float[] userFactors, float[] itemFactors,
 *                  byte[] userHas, byte[] itemHas): a scoring handle from factors held by the JVM
 *                  (the P2LAlgorithm templates keep Map[Int, Array[Double]] models) */
JNIEXPORT jlong JNICALL JNAME(importModel)(JNIEnv* env, jobject self, jint rank, jint nUsers, jint nItems, jint device,
                                           jfloatArray userFactors, jfloatArray itemFactors, jbyteArray userHas,
                                           jbyteArray itemHas) {
  pio_als_config cfg;
  pio_als_handle* h = NULL;
  jfloat *uf, *itf;
  jbyte *uh, *ih;
  int rc;
  (void)self;
  memset(&cfg, 0, sizeof cfg);
  cfg.abi_version = PIO_ALS_ABI_VERSION;
  cfg.rank = rank;
  cfg.n_users = nUsers;
  cfg.n_items = nItems;
  cfg.device = device;
  cfg.world_size = 1;
  uf = pin(env, userFactors);
  itf = pin(env, itemFactors);
  uh = pin(env, userHas);
  ih = pin(env, itemHas);
  rc = pio_als_model_import(&cfg, uf, itf, (const uint8_t*)uh, (const uint8_t*)ih, &h);
  unpin(env, itemHas, ih, JNI_ABORT);
  unpin(env, userHas, uh, JNI_ABORT);
  unpin(env, itemFactors, itf, JNI_ABORT);
  unpin(env, userFactors, uf, JNI_ABORT);
  if (rc != PIO_ALS_OK) {
    throw_rt(env, pio_als_last_error(NULL));
    return 0;
  }
  return (jlong)(intptr_t)h;
}

/* long[] stats(long h): {nnz after dedup, kernel launches, last run us, last ingest us} */
JNIEXPORT jlongArray JNICALL JNAME(stats)(JNIEnv* env, jobject self, jlong h) {
  pio_als_stats st;
  jlong v[4];
  jlongArray out;
  (void)self;
  if (check(env, H(h), pio_als_get_stats(H(h), &st)) != PIO_ALS_OK) return NULL;
  v[0] = (jlong)st.nnz;
  v[1] = (jlong)st.kernel_launches;
  v[2] = (jlong)(st.last_run_ms * 1000.0);
  v[3] = (jlong)(st.last_ingest_ms * 1000.0);
  out = (*env)->NewLongArray(env, 4);
  if (out) (*env)->SetLongArrayRegion(env, out, 0, 4, v);
  return out;
}

/* NaiveBayes (classification template): double[] nbTrain(int device, int[] label, float[] x, int nFeat, int nClass, double lambda)
 * returns pi (nClass) followed by theta (nClass x nFeat) */
JNIEXPORT jdoubleArray JNICALL JNAME(nbTrain)(JNIEnv* env, jobject self, jint device, jintArray label, jfloatArray x,
                                              jint nFeat, jint nClass, jdouble lambda) {
  jsize n = (*env)->GetArrayLength(env, label);
  jdoubleArray out = (*env)->NewDoubleArray(env, nClass * (nFeat + 1));
  jint* lb;
  jfloat* xs;
  jdouble* o;
  int rc;
  (void)self;
  if (!out) return NULL;
  lb = pin(env, label);
  xs = pin(env, x);
  o = pin(env, out);
  rc = pio_nb_train(device, (const int32_t*)lb, xs, (int64_t)n, nFeat, nClass, lambda, o, o + nClass);
  unpin(env, out, o, 0);
  unpin(env, x, xs, JNI_ABORT);
  unpin(env, label, lb, JNI_ABORT);
  if (rc != PIO_ALS_OK) {
    throw_rt(env, pio_als_last_error(NULL));
    return NULL;
  }
  return out;
}

/* int[] encodeIds(int device, byte[] bytes, long[] offsets, long[] outFirst):  (outFirst: capacity n, nullable)
 * BiMap.stringInt on the device -- returns the dense index of every string; outFirst[id] = position of the first
 * occurrence of the string with that index (the inverse map); the number of distinct ids is max(index) + 1. */
JNIEXPORT jintArray JNICALL JNAME(encodeIds)(JNIEnv* env, jobject self, jint device, jbyteArray bytes, jlongArray offsets,
                                             jlongArray outFirst) {
  jsize n = (*env)->GetArrayLength(env, offsets) - 1;
  jintArray out = (*env)->NewIntArray(env, n > 0 ? n : 0);
  int32_t nuniq = 0;
  jbyte* b;
  jlong *off, *first;
  jint* o;
  int rc;
  (void)self;
  if (!out) return NULL;
  b = pin(env, bytes);
  off = pin(env, offsets);
  first = pin(env, outFirst);
  o = pin(env, out);
  rc = pio_ids_encode(device, (const uint8_t*)b, (const int64_t*)off, (int64_t)n, (int32_t*)o, (int64_t*)first, &nuniq);
  unpin(env, out, o, 0);
  unpin(env, outFirst, first, 0);
  unpin(env, offsets, off, JNI_ABORT);
  unpin(env, bytes, b, JNI_ABORT);
  if (rc != PIO_ALS_OK) {
    throw_rt(env, pio_als_last_error(NULL));
    return NULL;
  }
  return out;
}

/* void coocTrain(int device, int[] user, int[] item, int nUsers, int nItems, int topn, int[] outItem, int[] outCount, int[] outN):
 * CooccurrenceAlgorithm.trainCooccurrence (outItem / outCount: nItems x topn, outN: nItems) */
JNIEXPORT void JNICALL JNAME(coocTrain)(JNIEnv* env, jobject self, jint device, jintArray user, jintArray item, jint nUsers,
                                        jint nItems, jint topn, jintArray outItem, jintArray outCount, jintArray outN) {
  jsize n = (*env)->GetArrayLength(env, user);
  jint* u = pin(env, user);
  jint* i = pin(env, item);
  jint* oi = pin(env, outItem);
  jint* oc = pin(env, outCount);
  jint* on = pin(env, outN);
  int rc = pio_cooc_train(device, (const int32_t*)u, (const int32_t*)i, (int64_t)n, nUsers, nItems, topn, (int32_t*)oi,
                          (int32_t*)oc, (int32_t*)on);
  (void)self;
  unpin(env, outN, on, 0);
  unpin(env, outCount, oc, 0);
  unpin(env, outItem, oi, 0);
  unpin(env, item, i, JNI_ABORT);
  unpin(env, user, u, JNI_ABORT);
  if (rc != PIO_ALS_OK) throw_rt(env, pio_als_last_error(NULL));
}
