/*
 * pio_als.h -- C ABI of the H100-native ALS hot path for PredictionIO engine templates.
 *
 * This is the drop-in boundary: exactly what a JNI shim in a `native-als` Scala module
 * binds in place of the Spark-MLlib calls the templates make today (INTEGRATION.md shows
 * the binding).  Plain C: opaque handle, plain pointers and sizes, int status returns
 * (0 = OK, <0 = error; text via pio_als_last_error).  The caller owns every host buffer;
 * the library owns all device memory behind the handle.  One handle = one training job /
 * one trained model; a handle is not thread-safe for mutation, but pio_als_recommend /
 * pio_als_similar on a trained handle serialise internally and may be called from
 * several threads (the reference calls predict from concurrent HTTP threads,
 * core/src/main/scala/org/apache/predictionio/workflow/CreateServer.scala:508-510).
 *
 * There is NO CPU fallback: every entry point that computes fails with
 * PIO_ALS_ERR_CUDA when no sm_90 device / CUDA runtime is usable.
 *
 * Reference interfaces replaced (paths relative to the reference repository root):
 *   pio_als_create + pio_als_set_ratings_coo + pio_als_run + pio_als_get_factors  (or the
 *   one-shot pio_als_train) replace
 *     new ALS().setRank(..)...run(mllibRatings)
 *       examples/scala-parallel-recommendation/blacklist-items/src/main/scala/ALSAlgorithm.scala:76-86
 *     ALS.train(ratings, rank, iterations, lambda, -1, seed)
 *       examples/scala-parallel-ecommercerecommendation/train-with-rate-event/src/main/scala/ECommAlgorithm.scala:116-122
 *     ALS.trainImplicit(ratings, rank, iterations, lambda, -1, 1.0, seed)
 *       examples/scala-parallel-similarproduct/multi-events-multi-algos/src/main/scala/ALSAlgorithm.scala:121-128
 *   pio_als_recommend replaces recommendProductsWithFilter / recommend
 *       examples/scala-parallel-recommendation/blacklist-items/src/main/scala/ALSModel.scala:44-60
 *     and the cartesian batchPredict
 *       examples/scala-parallel-recommendation/blacklist-items/src/main/scala/ALSAlgorithm.scala:117-158
 *   pio_als_similar replaces the cosine scan + getTopN
 *       examples/scala-parallel-similarproduct/multi-events-multi-algos/src/main/scala/ALSAlgorithm.scala:138-234
 *   pio_als_save / pio_als_load / pio_als_model_import replace ALSModel.save / ALSModel.apply
 *       examples/scala-parallel-recommendation/blacklist-items/src/main/scala/ALSModel.scala:63-100
 *   pio_nb_train / pio_nb_predict replace NaiveBayes.train / model.predict
 *       examples/scala-parallel-classification/add-algorithm/src/main/scala/NaiveBayesAlgorithm.scala:41-57
 *   pio_rf_train / pio_rf_predict replace RandomForest.trainClassifier / model.predict
 *       examples/scala-parallel-classification/add-algorithm/src/main/scala/RandomForestAlgorithm.scala:46-70
 *   pio_eval_folds_* run the recommendation template's k-fold evaluation
 *       examples/scala-parallel-recommendation/blacklist-items/src/main/scala/{DataSource.scala readEval, Evaluation.scala}
 *   pio_cls_folds_* run the classification template's k-fold evaluation
 *       examples/scala-parallel-classification/add-algorithm/src/main/scala/{DataSource.scala readEval, Evaluation.scala}
 *   pio_assoc_train / pio_assoc_model_* replace the complementary purchase template's Algorithm.train
 *       docs/manual/source/templates/complementarypurchase/dase.html.md.erb:293-314
 */
#ifndef PIO_ALS_H_
#define PIO_ALS_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#if defined(__GNUC__)
#define PIO_API __attribute__((visibility("default")))
#else
#define PIO_API
#endif

#define PIO_ALS_ABI_VERSION 2

/* status codes */
#define PIO_ALS_OK 0
#define PIO_ALS_ERR_ARG (-1)      /* bad argument (the templates' require(...) failures) */
#define PIO_ALS_ERR_CUDA (-2)     /* CUDA runtime / no usable device */
#define PIO_ALS_ERR_STATE (-3)    /* call order (e.g. run before set_ratings) */
#define PIO_ALS_ERR_NUMERIC (-4)  /* a normal equation was not positive definite (MLlib: dppsv info != 0) */
#define PIO_ALS_ERR_IO (-5)
#define PIO_ALS_ERR_COMM (-6)     /* NCCL */
#define PIO_ALS_ERR_NOMEM (-7)    /* host memory exhausted (pio_cooc_model_*, pio_popular_model_*) */

/* how repeated (user,item) pairs are treated by pio_als_set_ratings_coo */
#define PIO_ALS_DEDUP_NONE 0      /* recommendation template: every event is its own rating (ALSAlgorithm.scala:62-65) */
#define PIO_ALS_DEDUP_SUM 1       /* similarproduct: reduceByKey(_ + _) (multi-events ALSAlgorithm.scala:106) */
#define PIO_ALS_DEDUP_KEEP_LAST 2 /* ecommerce: latest timestamp wins (ECommAlgorithm.scala:189-197) */

#define PIO_ALS_INIT_CALLER 0     /* pio_als_set_init supplies initial factors */
#define PIO_ALS_INIT_HASH 1       /* unit-norm Gaussian rows from the counter hash (synth.py synth_init_factors) */

typedef struct pio_als_handle pio_als_handle;

typedef struct pio_als_config {
  int32_t abi_version;    /* PIO_ALS_ABI_VERSION */
  int32_t rank;           /* ALSAlgorithmParams.rank, 1..128 */
  int32_t implicit_prefs; /* setImplicitPrefs */
  int32_t n_users;        /* size of userStringIntMap */
  int32_t n_items;        /* size of itemStringIntMap */
  int32_t device;         /* CUDA device ordinal for this process */
  int32_t world_size;     /* number of cooperating processes (1 GPU each); 1 = single GPU */
  int32_t world_rank;
  int32_t init_mode;      /* PIO_ALS_INIT_* */
  int32_t reserved0;
  double lambda;          /* setLambda */
  double alpha;           /* setAlpha (implicit only) */
  int64_t seed;           /* setSeed; used by PIO_ALS_INIT_HASH */
  uint8_t nccl_id[128];   /* world_size > 1: the same ncclUniqueId on every rank (pio_als_nccl_unique_id on rank 0) */
} pio_als_config;

typedef struct pio_als_stats {
  int64_t nnz;              /* ratings after dedup (global) */
  int64_t kernel_launches;  /* kernels of this library launched on behalf of this handle */
  int64_t solve_launches;   /* of which half-step solve kernels */
  double last_run_ms;       /* device time of the last pio_als_run (CUDA events) */
  double last_solve_ms;     /* device time inside solve kernels during the last pio_als_run */
  double last_gram_ms;      /* ... inside YtY kernels */
  double last_comm_ms;      /* ... inside all-gathers */
  double last_ingest_ms;    /* device time of the last set_ratings (H2D + CSR build) */
  int32_t n_users_active;   /* users owning a factor */
  int32_t n_items_active;
  int32_t sm_count;
  int32_t last_score_path;  /* PIO_ALS_PATH_* bits: the scoring kernels the last recommend / similar call launched */
} pio_als_stats;

/* pio_als_stats.last_score_path: which scoring kernels ran (DESIGN.md 4.6); reset when each scoring call
 * starts, before its arguments are checked, so a rejected call or one with nothing to score leaves 0 */
#define PIO_ALS_PATH_SCORE_ONE 0x01    /* fused single-query kernel (one launch, result in mapped host memory) */
#define PIO_ALS_PATH_DOT_BLOCKED 0x02  /* blocked batch recommend kernel (rank <= 64, topk <= 32) */
#define PIO_ALS_PATH_COS_BLOCKED 0x04  /* blocked batch similar kernel (rank <= 64, topk <= 32) */
#define PIO_ALS_PATH_DOT_BATCHED 0x08  /* general recommend kernel (one item per thread, groups of 16 users) */
#define PIO_ALS_PATH_COS_MULTI 0x10    /* similar kernel for groups of 8 queries with <= 40 query vectors */
#define PIO_ALS_PATH_COS_BATCHED 0x20  /* long single similar query, query vectors in shared memory */
#define PIO_ALS_PATH_COS_FALLBACK 0x40 /* long single similar query too large for shared memory */
#define PIO_ALS_PATH_MULTI_PASS 0x80   /* more than one pass of <= 128 results (topk > 128) */
/* further bits of last_score_path that only the filtered calls set (pio_als_recommend_filtered /
 * pio_als_similar_batch_filtered); the PIO_ALS_PATH_* kernels above are the same for filtered and plain calls */
#define PIO_ALS_FPATH_FILTERED 0x100   /* a batch kernel ran with the per-query filter test at its pool insertion */
#define PIO_ALS_FPATH_LISTED 0x200     /* white-listed queries were scored over their lists (score_listed_kernel) */

PIO_API int pio_als_abi_version(void);
/* number of visible sm_90 devices, or PIO_ALS_ERR_CUDA */
PIO_API int pio_als_device_count(void);
PIO_API int pio_als_nccl_unique_id(uint8_t out_id[128]);

PIO_API int pio_als_create(const pio_als_config* cfg, pio_als_handle** out);
PIO_API void pio_als_destroy(pio_als_handle* h);
/* h may be NULL: returns the last error of a failed pio_als_create / pio_als_load on this thread */
PIO_API const char* pio_als_last_error(const pio_als_handle* h);

/* Ratings as COO triplets in HOST memory (indices from BiMap.stringInt, data/.../storage/BiMap.scala:116-128).
 * ts (int64, nullable) is only read for PIO_ALS_DEDUP_KEEP_LAST (NULL = input order is time order).
 * world_size > 1: every rank passes the same full COO; each keeps the rows it owns. nnz == 0 is
 * PIO_ALS_ERR_ARG (the templates' require(!ratings.isEmpty)). */
PIO_API int pio_als_set_ratings_coo(pio_als_handle* h, const int32_t* user, const int32_t* item,
                                    const float* rating, int64_t nnz, int dedup_mode,
                                    const int64_t* ts);
/* Same, the three arrays already resident in device memory of cfg.device. */
PIO_API int pio_als_set_ratings_coo_device(pio_als_handle* h, const int32_t* d_user,
                                           const int32_t* d_item, const float* d_rating,
                                           int64_t nnz, int dedup_mode, const int64_t* d_ts);
/* world_size > 1, sharded input: every rank passes ITS OWN slice of the events (HOST / DEVICE variants), the slices are
 * disjoint and rank r's slice precedes rank r + 1's in event order (what matters for PIO_ALS_DEDUP_SUM's fold order
 * and PIO_ALS_DEDUP_KEEP_LAST's ties).  The library routes every rating to the rank that owns its user row and to the
 * rank that owns its item row (NCCL send/recv) and sums the degrees over the ranks: no rank holds the full COO -- the
 * way an RDD[Rating] partition per executor reaches the GPUs (the reference shuffles the ratings into ALS's in/out
 * blocks, SURVEY.md 8(c)-2).  A rank's slice may be empty; the union may not.  Collective: all ranks must call it.
 * With world_size == 1 it is pio_als_set_ratings_coo[_device]. */
PIO_API int pio_als_set_ratings_coo_sharded(pio_als_handle* h, const int32_t* user, const int32_t* item,
                                            const float* rating, int64_t nnz_local, int dedup_mode,
                                            const int64_t* ts);
PIO_API int pio_als_set_ratings_coo_sharded_device(pio_als_handle* h, const int32_t* d_user, const int32_t* d_item,
                                                   const float* d_rating, int64_t nnz_local, int dedup_mode,
                                                   const int64_t* d_ts);
/* Initial factors, HOST, row-major n_users x rank / n_items x rank (item_factors may be NULL:
 * MLlib overwrites item factors in the first half-step). Rows that own no rating are zeroed. */
PIO_API int pio_als_set_init(pio_als_handle* h, const float* user_factors, const float* item_factors);
/* n_iters ALS iterations: each = item half-step (from user factors) then user half-step. May be
 * called repeatedly. */
PIO_API int pio_als_run(pio_als_handle* h, int n_iters);
/* Device-time breakdown of the last pio_als_run (CUDA events on the handle's stream), for bench.py's roofline:
 * out[0] item half-step solve kernels (ms, summed over the run), out[1] user half-step solve kernels, out[2] YtY
 * kernels, out[3] all-gathers, out[4]/out[5] = solve kernel of the item / user side (0 FP32 CUDA-core kernel, 1 wgmma
 * kernel, 2 warp-level mma.sync kernel, 3 pair kernel), out[6] iterations of that run, out[7] reserved.  No reference counterpart (Spark's stage timings,
 * core/.../workflow/CoreWorkflow.scala:74-81, are the nearest thing). */
PIO_API int pio_als_get_phase_ms(pio_als_handle* h, double out[8]);

/* Factors back to HOST. user_has/item_has (nullable): 1 if the row owns a factor (occurs in the
 * ratings), else 0 and the row is all zeros (MLlib emits no factor for it). */
PIO_API int pio_als_get_factors(pio_als_handle* h, float* user_out, float* item_out,
                                uint8_t* user_has, uint8_t* item_has);
/* One-shot: create-less convenience used by the JNI shim for ALS.train / ALS.trainImplicit:
 * set_ratings + (init) + run(iters) + get_factors on an existing handle. */
PIO_API int pio_als_train(pio_als_handle* h, const int32_t* user, const int32_t* item,
                          const float* rating, int64_t nnz, int dedup_mode, const int64_t* ts,
                          const float* user_init, const float* item_init, int n_iters,
                          float* user_out, float* item_out, uint8_t* user_has, uint8_t* item_has);

/* Top-k scoring on a trained (or loaded / imported) handle; HOST buffers.  topk >= 1, any size (more than 128 results
 * per query are produced in several passes over the item matrix).  All paths return identical results; which kernels
 * run is a matter of shape: ONE query (n == 1, or one similar query of <= 8 items; topk <= 128, rank <= 64) is a single
 * fused launch whose result the call polls from mapped host memory (tens of microseconds: the Serving.serve path of a
 * deployed engine, core/src/main/scala/org/apache/predictionio/workflow/CreateServer.scala:508-510); batches (rank <= 64,
 * topk <= 32) run the blocked kernels; everything else the general ones (DESIGN.md 4.6).
 * recommend: for each users[q]: score_i = <x_u, y_i> (fp64, index order) over items that own a factor and have
 *   item_mask[i] == 0 (nullable = no filter), times item_weight[i] if item_weight != NULL (fp64; the ecommerce
 *   template's weightedItems, examples/scala-parallel-ecommercerecommendation/adjust-score/src/main/scala/
 *   ECommAlgorithm.scala:258-266,490-497); out_items/out_scores are n x topk, best first, padded with -1 / 0;
 *   out_count[q] (nullable) = number of valid entries (0 for an unknown user).  Ties: smaller item index first. */
PIO_API int pio_als_recommend(pio_als_handle* h, const int32_t* users, int n, int topk,
                              const uint8_t* item_mask, const double* item_weight, int32_t* out_items,
                              float* out_scores, int32_t* out_count);
/* similar: score_i = (sum_q cosine(y_q, y_i)) * item_weight[i] over query items that own a factor; candidates are
 *   items owning a factor, item_mask[i] == 0, score > 0, and -- unless PIO_ALS_SIM_KEEP_QUERY_ITEMS is set -- not in
 *   the query (similarproduct: `!queryList.contains(i)`, multi-events ALSAlgorithm.scala:243-245; the ecommerce
 *   template's predictSimilar has no such rule, train-with-rate-event ECommAlgorithm.scala:492-525 -> pass the flag). */
#define PIO_ALS_SIM_KEEP_QUERY_ITEMS 1
PIO_API int pio_als_similar(pio_als_handle* h, const int32_t* query_items, int nq, int topk,
                            const uint8_t* item_mask, const double* item_weight, int flags, int32_t* out_items,
                            float* out_scores, int32_t* out_count);
/* n_queries similar() queries in one call (batchPredict / offline evaluation): query j = q_items[q_ptr[j] .. q_ptr[j+1]);
 * out_items/out_scores are n_queries x topk, out_count n_queries.  Same arithmetic as pio_als_similar. */
PIO_API int pio_als_similar_batch(pio_als_handle* h, const int64_t* q_ptr, const int32_t* q_items, int n_queries,
                                  int topk, const uint8_t* item_mask, const double* item_weight, int flags,
                                  int32_t* out_items, float* out_scores, int32_t* out_count);

/* Per-query filters of a batch scoring call: what every template query carries (blackList, whiteList, categories, the
 * user's seen items; examples/scala-parallel-similarproduct/multi-events-multi-algos/src/main/scala/ALSAlgorithm.scala:
 * 236-262, examples/scala-parallel-ecommercerecommendation/train-with-rate-event/src/main/scala/ECommAlgorithm.scala:
 * 527-575).  Every pointer is HOST memory and nullable. */
typedef struct pio_als_query_filter {
  const int64_t* ex_ptr;    /* n_queries + 1: query j excludes ex_items[ex_ptr[j] .. ex_ptr[j+1]) */
  const int32_t* ex_items;  /* item ids in any order; duplicates, ids < 0 or >= n_items are ignored */
  const uint8_t* has_wl;    /* n_queries: 1 = query j has a white list (an empty one means no candidate) */
  const int64_t* wl_ptr;    /* n_queries + 1 */
  const int32_t* wl_items;  /* same id rules as ex_items */
  const int32_t* set_ix;    /* n_queries: row of item_sets that applies to query j, or -1 */
  const uint8_t* item_sets; /* n_sets x n_items bytes, 1 = not a candidate (category filters; queries share rows) */
  int32_t n_sets;
} pio_als_query_filter;

/* pio_als_recommend / pio_als_similar_batch with a filter per query.  Row j of the result is, bit for bit, what the
 * unfiltered call returns for query j alone with the dense mask
 *   item_mask | item_sets[set_ix[j]] | (ex list of j) | (complement of the wl list of j, if has_wl[j])
 * and the same item_weight / flags.  f == NULL or a filter of null pointers is the unfiltered call.  Queries without a
 * white list scan the item matrix in the batch kernels, which test a candidate against its query's set row and sorted
 * exclusion list only when it is about to enter a top-k pool; white-listed queries are scored over their lists, at a
 * cost that follows the list length (DESIGN.md 4.6).  ex_ptr / wl_ptr not non-decreasing, a missing list where its
 * ptr array says one is read, set_ix outside [-1, n_sets), n_sets < 0 or rows without item_sets: PIO_ALS_ERR_ARG
 * before any device work. */
PIO_API int pio_als_recommend_filtered(pio_als_handle* h, const int32_t* users, int n, int topk,
                                       const uint8_t* item_mask, const double* item_weight,
                                       const pio_als_query_filter* f, int32_t* out_items, float* out_scores,
                                       int32_t* out_count);
PIO_API int pio_als_similar_batch_filtered(pio_als_handle* h, const int64_t* q_ptr, const int32_t* q_items,
                                           int n_queries, int topk, const uint8_t* item_mask,
                                           const double* item_weight, int flags, const pio_als_query_filter* f,
                                           int32_t* out_items, float* out_scores, int32_t* out_count);

/* A scoring handle from factors held by the caller (HOST, row-major n x rank; has flags nullable = every row owns a
 * factor): what ALSModel.apply / a P2LAlgorithm's driver-local Map[Int, Array[Double]] model becomes on the device
 * (examples/scala-parallel-similarproduct/multi-events-multi-algos/src/main/scala/ALSAlgorithm.scala:39-55,131).
 * cfg: rank, n_users, n_items, device (+ lambda / alpha / implicit_prefs kept as metadata); n_users may be 0 with
 * user_factors == NULL for an item-only model (similarproduct). */
PIO_API int pio_als_model_import(const pio_als_config* cfg, const float* user_factors, const float* item_factors,
                                 const uint8_t* user_has, const uint8_t* item_has, pio_als_handle** out);

/* Model persistence (one little-endian file: header, has flags, fp32 factors). */
PIO_API int pio_als_save(pio_als_handle* h, const char* path);
PIO_API int pio_als_load(const char* path, int device, pio_als_handle** out);

PIO_API int pio_als_get_stats(const pio_als_handle* h, pio_als_stats* out);

/* Device pointers to the library-owned rating generator output, for benchmarks that must start
 * with inputs resident in HBM: fills d_user/d_item/d_rating (device, nnz each) with the
 * synthetic events of SURVEY 8(d) (bit-identical to synth.py). */
PIO_API int pio_als_synth_ratings_device(int device, int32_t n_users, int32_t n_items, int64_t nnz,
                                         int64_t seed, int implicit, int64_t start,
                                         int32_t* d_user, int32_t* d_item, float* d_rating);

/* String ids -> dense indices on the GPU: BiMap.stringInt(keys) (data/src/main/scala/org/apache/predictionio/data/storage/
 * BiMap.scala:116-128: keys.distinct.collect -> index) as the templates apply it to the user and item id columns before
 * building MLlibRating (examples/scala-parallel-recommendation/blacklist-items/src/main/scala/ALSAlgorithm.scala:59-65).
 * The n strings are passed as one byte buffer plus n + 1 offsets (offsets[0] == 0); HOST buffers.
 *   out_index[e]   : dense index of string e; indices are handed out in order of first occurrence (the reference's
 *                    collect order is unspecified: compare by string id)
 *   out_first[id]  : nullable, capacity n: position of the first occurrence of the string with index id (the inverse map)
 *   out_n_unique   : number of distinct strings
 * Hash + radix sort + byte-wise verification: two different strings never share an index. */
PIO_API int pio_ids_encode(int device, const uint8_t* bytes, const int64_t* offsets, int64_t n, int32_t* out_index,
                           int64_t* out_first, int32_t* out_n_unique);

/* k-fold evaluation on the device: the recommendation template's `pio eval` (examples/scala-parallel-recommendation/
 * blacklist-items/src/main/scala/{DataSource.scala readEval, Evaluation.scala}) without per-rating host objects
 * (DESIGN.md 4.11).  An opaque object owns device copies of n ratings given by GLOBAL user / item indices (pio_ids_encode
 * of the whole columns) and their fp64 values; rating e is in the test set of fold e % k_fold and in the training set of
 * every other fold.  Per fold f, as the template computes them from that fold's strings:
 *   users / items  BiMap.stringInt of the training ratings: fold-local indices in order of first training occurrence
 *   training COO   the training ratings in rating order (fold-local indices, float32 ratings)
 *   queries        the distinct users of the test ratings in order of first occurrence among them (the template's
 *                  by_user order); each with its fold-local training index, or -1 when it has no training rating
 * Errors: status codes as above, text via pio_als_last_error(NULL); arguments are checked before any device work. */
typedef struct pio_eval_folds pio_eval_folds;

/* user, item: n global indices >= 0 each (HOST); rating: n fp64 (HOST); 1 <= n < 2^31, k_fold >= 1. */
PIO_API int pio_eval_folds_create(int device, const int32_t* user, const int32_t* item, const double* rating, int64_t n,
                                  int32_t k_fold, pio_eval_folds** out);
/* out[0] users, out[1] items, out[2] training ratings, out[3] queries of fold `fold`. */
PIO_API int pio_eval_folds_sizes(const pio_eval_folds* ef, int32_t fold, int64_t out[4]);
/* HOST, each nullable: user (out[0] entries) / item (out[1]) = global index of each fold-local index; query_user
 * (out[3]) = global user of each query; query_train_user (out[3]) = its fold-local training index or -1. */
PIO_API int pio_eval_folds_maps(const pio_eval_folds* ef, int32_t fold, int32_t* user, int32_t* item,
                                int32_t* query_user, int32_t* query_train_user);
/* pio_als_set_ratings_coo_device(h, fold's training COO, PIO_ALS_DEDUP_NONE) on a handle created with the fold's
 * user and item counts on the same device (world_size 1). */
PIO_API int pio_eval_folds_set_ratings(pio_eval_folds* ef, int32_t fold, pio_als_handle* h);
/* Keeps a top-N result of fold `fold` on the object: items (n_queries x num, fold-local item indices, as
 * pio_als_recommend returns them for the fold's query_train_user) and count (valid entries per query, 0..num);
 * n_queries must be the fold's.  *out_result names it until pio_eval_folds_result_free; results of any folds may be
 * kept at once. */
PIO_API int pio_eval_folds_result_add(pio_eval_folds* ef, int32_t fold, const int32_t* items, const int32_t* count,
                                      int32_t n_queries, int32_t num, int32_t* out_result);
PIO_API int pio_eval_folds_result_free(pio_eval_folds* ef, int32_t result);
/* Per query q of the result's fold (HOST, n_queries each), ratings compared in fp64 with rating >= threshold:
 *   hits[q]  of the first min(k, count[q]) predicted items, those whose largest test rating of q passes
 *   npos[q]  distinct test items of q whose largest rating passes (items unknown to the fold's training count too)
 *   nraw[q]  test ratings of q that pass
 * PrecisionAtK = hits / min(k, npos) where npos > 0; PositiveCount = nraw (Evaluation.scala:32-62).  k >= 1. */
PIO_API int pio_eval_folds_rank_counts(pio_eval_folds* ef, int32_t result, int32_t k, double threshold, int32_t* hits,
                                       int32_t* npos, int32_t* nraw);
PIO_API int pio_eval_folds_destroy(pio_eval_folds* ef);

/* Event file scan: PEventStore.find (data/src/main/scala/org/apache/predictionio/data/store/PEventStore.scala:59-119)
 * over text in the `pio import` / `pio export` JSON-lines format (tools/src/main/scala/org/apache/predictionio/tools/
 * imprt/FileToEvents.scala:93-103), producing event columns instead of Event objects (DESIGN.md 3.1).
 * Strings are NUL-terminated UTF-8. */
#define PIO_EVENTS_TARGET_ANY 0      /* targetEntityType not restricted */
#define PIO_EVENTS_TARGET_ABSENT 1   /* targetEntityType must be absent (Some(None)) */
#define PIO_EVENTS_TARGET_EQUALS 2   /* targetEntityType must equal target_entity_type (Some(Some(x))) */
#define PIO_EVENTS_MIN_EVENT_BYTES 64 /* no matched line is shorter: n_bytes / 64 + 1 events always fit */
#define PIO_EVENTS_HAS_VALUE 1       /* out_flags bits */
#define PIO_EVENTS_HAS_TARGET 2

typedef struct pio_events_filter {
  const char* entity_type;             /* NULL = any entity type */
  const char* const* event_names;      /* an event's output code is the index of its name here; NULL = any event
                                          name (code -1), as eventNames = None in find */
  int32_t n_event_names;               /* with event_names != NULL, 0 = an empty list: no event matches */
  int32_t target_entity_type_mode;     /* PIO_EVENTS_TARGET_* */
  const char* target_entity_type;      /* for PIO_EVENTS_TARGET_EQUALS */
  const char* property;                /* numeric property to extract (DataMap.get(name, Double)); NULL = none */
  int32_t has_start, has_until;        /* eventTime >= start_us, eventTime < until_us (half-open, as in find) */
  int64_t start_us, until_us;          /* microseconds since 1970-01-01T00:00:00Z */
} pio_events_filter;

/* text[0 .. n_bytes): complete lines, ended by "\n", "\r\n" or a lone "\r" (the last one may lack its terminator); HOST
 * buffers.  Lines are numbered from 0, blank ones included; a line that is empty after stripping spaces and tabs is
 * no event.  Every line is either parsed on the device -- exactly as Event.from_json(json.loads(line)) and find's
 * filter would take it -- or listed as a fallback line for the caller to parse (anything outside the accepted grammar,
 * DESIGN.md 3.1; falling back is always correct).
 * Per matched event, in line order (capacity entries, capacity >= n_bytes / PIO_EVENTS_MIN_EVENT_BYTES + 1):
 *   out_line (line index), out_code (event-name index), out_value + out_flags & PIO_EVENTS_HAS_VALUE (the property as
 *   a double; a property value that is not a number exact in double makes the line a fallback line), out_time_us,
 *   out_flags & PIO_EVENTS_HAS_TARGET (targetEntityId present), and the decoded entityId / targetEntityId bytes:
 *   event e's id is out_eid_bytes[out_eid_off[e] .. out_eid_off[e + 1]) (offsets: capacity + 1 entries; bytes: n_bytes
 *   suffice, decoded ids are never longer than their JSON text).
 * Fallback lines, in line order: out_fb_line, and the line's bytes text[out_fb_begin .. out_fb_end) without the
 *   terminator.  *out_n_fallback is the number of fallback lines; when it exceeds fb_capacity only the first
 *   fb_capacity were written: call again with room for all of them.
 * *out_n_lines = number of lines.  PIO_ALS_ERR_ARG for a bad filter or sizes; PIO_ALS_ERR_CUDA without a device.
 * Device memory is bounded by the device chunk (64 MB), not by n_bytes; the copy of one chunk overlaps the scan of the
 * one before. */
PIO_API int pio_events_scan(int device, const uint8_t* text, int64_t n_bytes, const pio_events_filter* filter,
                            int64_t capacity, int64_t* out_line, int32_t* out_code, double* out_value,
                            uint8_t* out_flags, int64_t* out_time_us, uint8_t* out_eid_bytes, int64_t* out_eid_off,
                            uint8_t* out_tid_bytes, int64_t* out_tid_off, int64_t* out_n_events, int64_t fb_capacity,
                            int64_t* out_fb_line, int64_t* out_fb_begin, int64_t* out_fb_end, int64_t* out_n_fallback,
                            int64_t* out_n_lines);

/* Keyed event scan: pio_events_scan (same filter, chunking, pinned staging, fallback protocol and capacity bound) that
 * also reads the top-level keys keys[0 .. n_keys) of each matched event's `properties` (DESIGN.md 3.2); what
 * PEventStore.aggregatePropertyColumns folds.  Keys are compared with the JSON keys after unescaping.
 * Per matched event e, next to everything pio_events_scan writes:
 *   out_present[e] bit q : key q is in `properties` (a null value counts; absent or null `properties` has no keys)
 *   out_number[e] bit q  : its value is a JSON number exact in double (integer <= 2^53 in magnitude, or Clinger's fast
 *                          path), in out_num[e * n_keys + q] (0 otherwise)
 *   token slot e * n_keys + q: the value's raw JSON token, out_tok_bytes[out_tok_off[slot] .. out_tok_off[slot + 1]):
 *                          a string with its quotes, an array, an object, true / false / null, an integer, or a number
 *                          off the fast path; empty for an absent key and for a fraction / exponent number on the fast
 *                          path (out_num holds it).  out_tok_off: capacity * n_keys + 1 entries; out_tok_bytes: n_bytes.
 * A tracked key twice in one `properties` object makes the line a fallback line; a number off the fast path does not.
 * PIO_ALS_ERR_ARG for n_keys outside 1..8, a NULL, empty or repeated key, or filter->property != NULL. */
PIO_API int pio_events_scan_keys(int device, const uint8_t* text, int64_t n_bytes, const pio_events_filter* filter,
                                 const char* const* keys, int n_keys, int64_t capacity, int64_t* out_line,
                                 int32_t* out_code, double* out_value, uint8_t* out_flags, int64_t* out_time_us,
                                 uint8_t* out_eid_bytes, int64_t* out_eid_off, uint8_t* out_tid_bytes,
                                 int64_t* out_tid_off, uint8_t* out_present, uint8_t* out_number, double* out_num,
                                 uint8_t* out_tok_bytes, int64_t* out_tok_off, int64_t* out_n_events,
                                 int64_t fb_capacity, int64_t* out_fb_line, int64_t* out_fb_begin, int64_t* out_fb_end,
                                 int64_t* out_n_fallback, int64_t* out_n_lines);

/* LEventAggregator's $set / $unset / $delete fold (data/src/main/scala/org/apache/predictionio/data/storage/
 * LEventAggregator.scala) restricted to tracked keys, over n events in file order (HOST buffers): entity ids as bytes +
 * n + 1 offsets (eid_off[0] == 0), code[e] 0 = $set / 1 = $unset / 2 = $delete, time_us[e], and present[e] (bit q: key
 * q is in the event's properties; unused when n_keys == 0).  Events of one entity are taken in (time, file order).
 * Per distinct entity, in order of first occurrence among the events (capacity n):
 *   out_first_event   index of its first event (its id)
 *   out_exists        1 when its last $set comes after its last $delete (the aggregate exists)
 *   out_first_us / out_last_us   min / max time over all its events, also those before a $delete
 *   out_winner[g * n_keys + q]   the $set whose value key q holds, or -1 when the key is absent: the last event among
 *                                {$delete, $set with q present, $unset with q present} when that is a $set
 * *out_n_entities = number of entities.  Deterministic.  PIO_ALS_ERR_ARG for n_keys outside 0..8, a code outside
 * 0..2, n >= 2^31 or missing buffers. */
PIO_API int pio_events_fold(int device, const uint8_t* eid_bytes, const int64_t* eid_off, const int32_t* code,
                            const int64_t* time_us, const uint8_t* present, int64_t n, int n_keys,
                            int64_t* out_first_event, uint8_t* out_exists, int64_t* out_first_us, int64_t* out_last_us,
                            int64_t* out_winner, int64_t* out_n_entities);

/* Whole-map event scan: pio_events_scan (same filter, chunking, pinned staging, fallback protocol and capacity bound)
 * that also reads every top-level key of each matched event's `properties`, in object order (DESIGN.md 3.4); what
 * PEventStore.aggregatePropertyMaps folds.  Per matched event e, next to everything pio_events_scan writes:
 *   out_utc_offset[e]   eventTime's UTC offset in minutes (0 for "Z" or no offset)
 *   out_prop_off[e]     its records are out_prop_off[e] .. out_prop_off[e + 1) (capacity + 1 entries); none for absent,
 *                       null or {} properties
 * Per record r, one per key in object order (a key twice in one object gives two records):
 *   the key, unescaped to UTF-8: out_key_bytes[out_key_off[r] .. out_key_off[r + 1])
 *   the value's raw JSON token: out_tok_bytes[out_tok_off[r] .. out_tok_off[r + 1]) (numbers too: the caller decodes)
 * rec_capacity >= n_bytes / PIO_EVENTS_MIN_RECORD_BYTES + 1 (a record takes at least `"":0` of line text);
 * out_key_off / out_tok_off: rec_capacity + 1 entries; out_key_bytes / out_tok_bytes: n_bytes each.
 * *out_n_records = number of records.  PIO_ALS_ERR_ARG for a bad filter or sizes, or filter->property != NULL. */
#define PIO_EVENTS_MIN_RECORD_BYTES 4
PIO_API int pio_events_scan_props(int device, const uint8_t* text, int64_t n_bytes, const pio_events_filter* filter,
                                  int64_t capacity, int64_t* out_line, int32_t* out_code, double* out_value,
                                  uint8_t* out_flags, int64_t* out_time_us, uint8_t* out_eid_bytes, int64_t* out_eid_off,
                                  uint8_t* out_tid_bytes, int64_t* out_tid_off, int16_t* out_utc_offset,
                                  int64_t* out_prop_off, int64_t rec_capacity, uint8_t* out_key_bytes,
                                  int64_t* out_key_off, uint8_t* out_tok_bytes, int64_t* out_tok_off,
                                  int64_t* out_n_events, int64_t* out_n_records, int64_t fb_capacity,
                                  int64_t* out_fb_line, int64_t* out_fb_begin, int64_t* out_fb_end,
                                  int64_t* out_n_fallback, int64_t* out_n_lines);

/* LEventAggregator's $set / $unset / $delete fold of every key (DESIGN.md 3.4), over n events in file order (HOST
 * buffers): entity ids as bytes + n + 1 offsets (eid_off[0] == 0), code[e] 0 = $set / 1 = $unset / 2 = $delete,
 * time_us[e], and the records of event e, prop_off[e] .. prop_off[e + 1) (prop_off[0] == 0), one per key of its
 * properties in object order, whose keys are key_bytes[key_off[r] .. key_off[r + 1]).  Events of one entity are taken in
 * (time, file order); records of a $delete are ignored.
 * Per distinct entity g, in order of first occurrence among the events (capacity n, out_win_off n + 1):
 *   out_first_event        index of its first event (its id)
 *   out_exists             1 when its last $set comes after its last $delete (the PropertyMap exists)
 *   out_first_time_event   the event that gives firstUpdated: the first in (time, file order)
 *   out_last_time_event    the event that gives lastUpdated: the first in file order among those at the latest time
 *   out_win_rec[out_win_off[g] .. out_win_off[g + 1])   the record holding the value of each key of the PropertyMap, in
 *                          the map's order; out_win_key[w] its key code (capacity prop_off[n] each)
 * A key k is present when the last $set record with k comes after remover(k) = max(the last $delete, the last $unset
 * with k); that record holds its value, and its place in the map is that of the first $set record with k after
 * remover(k): (event, index in the object).  Key codes number distinct keys in order of first occurrence among the
 * records; out_key_first[c] is the first record of code c (capacity prop_off[n]).  *out_n_entities, *out_n_keys: the
 * numbers of entities and key codes.  Deterministic.  PIO_ALS_ERR_ARG for a code outside 0..2, decreasing prop_off,
 * n or prop_off[n] >= 2^31, or missing buffers. */
PIO_API int pio_events_fold_props(int device, const uint8_t* eid_bytes, const int64_t* eid_off, const int32_t* code,
                                  const int64_t* time_us, const int64_t* prop_off, int64_t n, const uint8_t* key_bytes,
                                  const int64_t* key_off, int64_t* out_first_event, uint8_t* out_exists,
                                  int64_t* out_first_time_event, int64_t* out_last_time_event, int64_t* out_win_off,
                                  int64_t* out_win_rec, int32_t* out_win_key, int64_t* out_key_first,
                                  int64_t* out_n_entities, int64_t* out_n_keys);

/* Event index: LEventStore.findByEntity (data/src/main/scala/org/apache/predictionio/data/store/LEventStore.scala:76)
 * for one view -- a `find` filter (entity type, event names, target entity type) -- of an append-only event file, kept
 * on the device (DESIGN.md 3.3).  Per matched event it holds the hash of the decoded entityId, eventTime, the byte
 * offset and length of the event's line in the file, and the id bytes, in two runs (main, delta) ordered by
 * (hash, eventTime descending, offset ascending).  An append is sorted and merged into delta; delta is merged into main
 * once it holds more than 1 / PIO_EVENTS_INDEX_MERGE_DIVISOR of main's entries.  HOST buffers throughout. */
#define PIO_EVENTS_INDEX_MERGE_DIVISOR 16

typedef struct pio_events_index pio_events_index;

typedef struct pio_events_index_stats {
  int64_t n_main, n_delta;   /* entries in each run */
  int64_t n_merges;          /* delta -> main merges so far */
  double scan_ms, sort_ms, merge_ms;   /* the last append / add_host: chunk loop, sort + merge into delta, delta -> main
                                          merge (0 when none); wall milliseconds, device work included */
} pio_events_index_stats;

/* An empty index of `view` on `device` (the filter's strings are copied).  PIO_ALS_ERR_ARG for a view with `property`
 * set or with time bounds. */
PIO_API int pio_events_index_create(int device, const pio_events_filter* view, pio_events_index** out);

/* Adds the events of text[0 .. n_bytes): complete lines as pio_events_scan takes them, whose first byte is at
 * `base_offset` in the file; every offset must be larger than those already indexed.  The matched events stay on the
 * device.  Fallback lines are reported as pio_events_scan reports them (byte ranges relative to text, line order);
 * when *out_n_fallback exceeds fb_capacity nothing was added: call again with room for all of them.  The caller parses
 * the fallback lines and adds the matching ones with pio_events_index_add_host. */
PIO_API int pio_events_index_append(pio_events_index* ix, const uint8_t* text, int64_t n_bytes, int64_t base_offset,
                                    int64_t fb_capacity, int64_t* out_fb_begin, int64_t* out_fb_end,
                                    int64_t* out_n_fallback);

/* Adds n events parsed by the caller: entityId k = id_bytes[id_off[k] .. id_off[k + 1]) (id_off[0] == 0), its
 * eventTime, and its line's byte offset and length in the file. */
PIO_API int pio_events_index_add_host(pio_events_index* ix, const uint8_t* id_bytes, const int64_t* id_off,
                                      const int64_t* time_us, const int64_t* offset, const int32_t* length, int64_t n);

/* For each of n ids (id k = id_bytes[id_off[k] .. id_off[k + 1])): out_count[k] = its events, at most `limit` (limit < 0:
 * all).  *out_total = the sum.  When *out_total <= capacity, id k's events are at out_offset / out_len
 * [sum(out_count[0 .. k)) ..), as (line offset, line length), latest eventTime first and in file order among equal
 * times; otherwise nothing is written there: call again with capacity >= *out_total. */
PIO_API int pio_events_index_lookup(pio_events_index* ix, const uint8_t* id_bytes, const int64_t* id_off, int32_t n,
                                    int64_t limit, int64_t capacity, int64_t* out_count, int64_t* out_total,
                                    int64_t* out_offset, int32_t* out_len);

PIO_API int pio_events_index_get_stats(const pio_events_index* ix, pio_events_index_stats* out);
PIO_API int pio_events_index_destroy(pio_events_index* ix);

/* Item co-occurrence of the similarproduct template's CooccurrenceAlgorithm.trainCooccurrence
 * (examples/scala-parallel-similarproduct/multi-events-multi-algos/src/main/scala/CooccurrenceAlgorithm.scala:72-105):
 * (user, item) view events (indices, HOST) -> distinct -> for every user all item pairs -> count per pair -> for every item the
 * topn co-occurring items with the largest counts.  out_item / out_count are n_items x topn (padded with -1 / 0),
 * out_n[i] = number of valid entries of item i.  Ties (unspecified in the reference): larger count first, then the smaller
 * item index.  Limits: n_items <= 2^20, fewer than 2^31 (user, item1, item2) triples. */
PIO_API int pio_cooc_train(int device, const int32_t* user, const int32_t* item, int64_t n, int32_t n_users,
                           int32_t n_items, int topn, int32_t* out_item, int32_t* out_count, int32_t* out_n);

/* Batch scoring of CooccurrenceAlgorithm.predict (CooccurrenceAlgorithm.scala:107-175) over a trained co-occurrence model
 * (DESIGN.md 4.9).  An opaque object holds the model: top_items / top_counts n_items x topn and top_n n_items, HOST
 * arrays in the layout pio_cooc_train returns.  Errors: status codes as above, text via pio_als_last_error(NULL). */
typedef struct pio_cooc_model pio_cooc_model;

typedef struct pio_cooc_stats {
  int64_t kernel_launches;        /* kernels launched on behalf of this model, over all calls */
  int64_t last_expanded;          /* (query, candidate) entries the last pio_cooc_predict_filtered expanded, all parts */
  int64_t last_rows;              /* distinct (query, item) rows of the last call that passed the filters */
  int64_t last_budget;            /* expanded entries per part the last call was split by */
  int32_t last_parts;             /* parts of the last call (0: no query, or rejected) */
  int32_t last_max_part_queries;  /* most queries in one part of the last call */
} pio_cooc_stats;

/* Default number of expanded entries per part of a pio_cooc_predict_filtered call (about 48 bytes of device memory
 * each); the environment variable PIO_COOC_PREDICT_BUDGET (a positive integer) overrides it.  Results do not depend
 * on it. */
#define PIO_COOC_PREDICT_BUDGET (1ll << 24)

/* Checks the arrays on the host -- 0 <= top_n[i] <= topn, top_items[i][t] in [0, n_items) and top_counts[i][t] >= 0 for
 * t < top_n[i] -- and copies them: PIO_ALS_ERR_ARG naming the item and slot of the first violation.  n_items >= 1, topn
 * >= 1.  The device copy is made on `device` by the first pio_cooc_predict_filtered, so that a model
 * holds no device memory until it scores. */
PIO_API int pio_cooc_model_create(int device, int32_t n_items, int32_t topn, const int32_t* top_items,
                                  const int32_t* top_counts, const int32_t* top_n, pio_cooc_model** out);
PIO_API int pio_cooc_model_destroy(pio_cooc_model* m);
/* n_queries queries: query j = q_items[q_ptr[j] .. q_ptr[j+1]) (HOST); ids outside [0, n_items) and repeats are ignored.
 * Row j of out_items (int32) / out_scores (int64), n_queries x topk, best first, padded with -1 / 0, and out_count[j]
 * (nullable): for the set Q of query j's known items, the candidates are the items of the first top_n[q] entries of each
 * q in Q, scored by the sum of their counts over Q (exact, int64); a candidate is dropped when query j has a white list
 * (f->has_wl[j]) that does not hold it, when its exclusion list or set row (f: pio_als_query_filter, nullable, with the
 * argument rules of pio_als_similar_batch_filtered) holds it, or when it is in Q; the rest are ordered by score
 * descending, then item index ascending, and cut at topk >= 1.
 * The batch runs in parts of consecutive queries whose expansions -- the sum of top_n over each query's listed known
 * ids, a repeated id counted each time -- stay within PIO_COOC_PREDICT_BUDGET entries, at least one query per part.
 * Rejected with PIO_ALS_ERR_ARG before any device work: bad arguments, q_ptr not non-decreasing from 0 or naming
 * entries of a NULL q_items, a bad filter, and a query whose expansion is 2^32 entries or more. */
PIO_API int pio_cooc_predict_filtered(pio_cooc_model* m, const int64_t* q_ptr, const int32_t* q_items,
                                      int32_t n_queries, int32_t topk, const pio_als_query_filter* f,
                                      int32_t* out_items, int64_t* out_scores, int32_t* out_count);
PIO_API int pio_cooc_model_get_stats(const pio_cooc_model* m, pio_cooc_stats* out);

/* Batch top-N of one fixed per-item score under per-query filters: the ecommerce template's predictDefault
 * (adjust-score ECommAlgorithm.scala:508-538), the popularity rule of users with no factor and no recent items
 * (DESIGN.md 4.14).  An opaque object holds the scores; the caller folds any weights into them.  Errors: status codes as
 * above, text via pio_als_last_error(NULL). */
typedef struct pio_popular_model pio_popular_model;

typedef struct pio_popular_stats {
  int64_t kernel_launches;        /* over all calls on this model */
  int64_t last_walked;            /* ranked entries the last call's walk examined, all queries */
  int64_t last_listed;            /* white-list entries the last call sorted */
  int32_t last_parts, last_max_part_queries;
} pio_popular_stats;

/* Default number of entries per part of a pio_popular_predict_filtered call (about 28 bytes of device memory each); the
 * environment variable PIO_POPULAR_PREDICT_BUDGET (a positive integer) overrides it.  Results do not depend on it. */
#define PIO_POPULAR_PREDICT_BUDGET (1ll << 24)   /* env PIO_POPULAR_PREDICT_BUDGET overrides */

/* Checks scores[0 .. n_items) on the host -- PIO_ALS_ERR_ARG naming the first NaN; infinities are allowed -- and
 * copies them.  n_items >= 1.  The device copy and the ranked order are made on `device` by the first
 * pio_popular_predict_filtered, so that a model holds no device memory until it scores. */
PIO_API int pio_popular_model_create(int device, int32_t n_items, const double* scores, pio_popular_model** out);
/* n_queries queries, each with the filter of f (pio_als_query_filter, nullable, with the argument rules of
 * pio_als_similar_batch_filtered; ids out of range and duplicates are ignored).  The candidates of query j are the
 * items i in [0, n_items) that are not in j's exclusion list, not set in j's item_sets row, and in j's white list if
 * has_wl[j].  They are ordered by scores[i] descending, with -0.0 == +0.0; equal scores go by item index ascending; the
 * list is cut at topk >= 1.  Row j of out_items (int32) / out_scores (fp64), n_queries x topk, padded with -1 / 0;
 * out_scores holds scores[i] exactly (a -0.0 stays -0.0), and out_count[j] is the number of results.
 * The batch runs in parts of consecutive queries whose entries -- the entries ex_ptr and wl_ptr name for each query plus
 * its topk output slots -- stay within PIO_POPULAR_PREDICT_BUDGET, at least one query per part.  Rejected with
 * PIO_ALS_ERR_ARG before any device work: topk < 1, n_queries < 0, a NULL output, a bad filter, and a query whose
 * entries are 2^32 or more (a part's entries are numbered in 32 bits). */
PIO_API int pio_popular_predict_filtered(pio_popular_model* m, int32_t n_queries, int32_t topk,
                                         const pio_als_query_filter* f, int32_t* out_items, double* out_scores,
                                         int32_t* out_count);
PIO_API int pio_popular_model_get_stats(const pio_popular_model* m, pio_popular_stats* out);
PIO_API int pio_popular_model_destroy(pio_popular_model* m);

/* Default number of entries per part of a pio_serve_zscore_merge call (about 90 bytes of device memory each); the
 * environment variable PIO_SERVE_MERGE_BUDGET (a positive integer) overrides it.  Results do not depend on it. */
#define PIO_SERVE_MERGE_BUDGET (1ll << 24)

/* The similarproduct template's Serving.serve (Serving.scala:29-69) over a batch of n_queries queries, on `device`
 * (DESIGN.md 4.13).  For each of n_algos algorithms a, HOST arrays: items[a] (int32) and scores[a] (fp64), both
 * n_queries x widths[a], and counts[a] (int32, n_queries): the first counts[a][j] entries of row j are query j's list,
 * with item ids in one numbering [0, n_items).  num[j] is query j's num.  Per query j:
 *   - unless num[j] == 1, each list of n entries is standardised: mean = sum / n (0 for n = 0), sd = sqrt(sum((s -
 *     mean)^2) / (n - 1)) for n > 1 else 0, z = 0 where sd == 0 else (s - mean) / sd, with numpy's pairwise summation
 *     started from 0.0 (np.add.reduce); with num[j] == 1 the scores are used as they are;
 *   - the values are summed per item as 0.0 + z0 + z1 + ..., in algorithm order, then list order;
 *   - the items are ordered by sum descending, equal sums in order of the item's first (algorithm, position), and cut
 *     at min(num[j], topk).
 * Row j of out_items (int32) / out_scores (fp64), n_queries x topk, best first, padded with -1 / 0; out_count[j] is the
 * number of results.  Every operation is rounded as numpy and Python round it, so the results equal Serving.serve's bit
 * for bit.  The batch runs in parts of consecutive queries whose entries (sums of counts) stay within
 * PIO_SERVE_MERGE_BUDGET, at least one query per part.  Rejected with PIO_ALS_ERR_ARG before any device work: n_algos,
 * n_items or topk below 1, a NULL array, a negative width, a count outside [0, widths[a]], an id outside [0, n_items), a
 * score that is not finite, num[j] < 1, and a query with 2^32 entries or more.  Errors: pio_als_last_error(NULL). */
PIO_API int pio_serve_zscore_merge(int device, int32_t n_queries, int32_t n_algos, int32_t n_items,
                                   const int32_t* const* items, const double* const* scores,
                                   const int32_t* const* counts, const int32_t* widths, const int32_t* num,
                                   int32_t topk, int32_t* out_items, double* out_scores, int32_t* out_count);

/* MLlib multinomial NaiveBayes (classification template). HOST buffers.
 * label: class index 0..n_class-1; x: n x n_feat, non-negative. pi: n_class, theta: n_class x n_feat
 * (fp64 log-probabilities, as MLlib's NaiveBayesModel.pi/theta). */
PIO_API int pio_nb_train(int device, const int32_t* label, const float* x, int64_t n, int n_feat,
                         int n_class, double lambda, double* pi, double* theta);
PIO_API int pio_nb_predict(int device, const float* x, int64_t n, int n_feat, int n_class,
                           const double* pi, const double* theta, int32_t* out_label);

/* MLlib 2.4 RandomForest.trainClassifier with continuous features (classification template, RandomForestAlgorithm
 *   examples/scala-parallel-classification/add-algorithm/src/main/scala/RandomForestAlgorithm.scala:46-70).
 * The rules, and which of them are this project's choices, are stated in tests/forest_ref.py and DESIGN.md 4.10: every
 * random draw (split sample, bootstrap, feature subsets) is a pure function of (seed, stream, tree, index), counts are
 * integers, and the forest does not depend on the device, launch order or how trees are grouped.
 * Limits of this implementation (PIO_ALS_ERR_ARG): num_classes <= 64, max_bins <= 65536, n < 2^31.  Arguments, labels
 * and features are checked on the host before any device work; a label < 0 or >= num_classes fails with the message
 * of MLlib's GiniAggregator / EntropyAggregator, a non-finite label or feature is rejected. */
#define PIO_RF_GINI 0
#define PIO_RF_ENTROPY 1

typedef struct pio_rf_params {
  int32_t num_classes;                  /* >= 2 */
  int32_t num_trees;                    /* >= 1 */
  int32_t max_depth;                    /* 0 .. 30 */
  int32_t max_bins;                     /* >= 2 */
  int32_t impurity;                     /* PIO_RF_GINI / PIO_RF_ENTROPY */
  int32_t reserved0;
  const char* feature_subset_strategy;  /* auto | all | sqrt | log2 | onethird | integer k > 0 | fraction in (0, 1] */
  int64_t seed;
} pio_rf_params;

typedef struct pio_rf_forest pio_rf_forest;   /* a trained forest, host memory only */

/* label: n class labels (class = trunc(label)); x: n x n_feat row-major fp64 (HOST buffers). */
PIO_API int pio_rf_train(int device, const pio_rf_params* params, const double* label, const double* x, int64_t n,
                         int32_t n_feat, pio_rf_forest** out);
/* The forest's size: trees and nodes over all trees (after MLlib's pruning of equal leaf pairs). */
PIO_API int pio_rf_forest_size(const pio_rf_forest* f, int32_t* n_trees, int64_t* n_nodes);
/* Flat per-node arrays, trees one after the other, each in preorder: tree_off [n_trees + 1] (first node of each tree),
 * and per node: feature (-1 at a leaf), threshold (x[feature] <= threshold goes left; 0 at a leaf), left / right
 * (indices into these arrays, -1 at a leaf), prediction (class), impurity, gain (0 at a leaf) and count (the node's
 * bootstrap-weighted row count).  Any output pointer may be null. */
PIO_API int pio_rf_forest_get(const pio_rf_forest* f, int32_t* tree_off, int32_t* feature, double* threshold,
                              int32_t* left, int32_t* right, int32_t* prediction, double* impurity, double* gain,
                              int64_t* count);
PIO_API int pio_rf_forest_destroy(pio_rf_forest* f);
/* The forest's majority vote (ties to the smaller class) for n rows x (n x n_feat fp64, HOST) into out (class index),
 * from the flat arrays of pio_rf_forest_get. */
PIO_API int pio_rf_predict(int device, int32_t n_trees, const int32_t* tree_off, int64_t n_nodes, const int32_t* feature,
                           const double* threshold, const int32_t* left, const int32_t* right, const int32_t* prediction,
                           int32_t num_classes, const double* x, int64_t n, int32_t n_feat, int32_t* out);

/* k-fold evaluation of the classification template on the device: its `pio eval` (examples/scala-parallel-classification/
 * add-algorithm/src/main/scala/{DataSource.scala readEval, Evaluation.scala, PrecisionEvaluation.scala}) without a host
 * copy of a fold's rows per training (DESIGN.md 4.12).  An opaque object owns device copies of n labeled points (fp64
 * labels, n x n_feat fp64 features, row-major) and each row's index among the distinct labels; row i is in the test set
 * of fold i % k_fold and in the training set of every other fold, in row order.  Labels must be finite; -0.0 and 0.0 are
 * one label.  Errors: status codes as above, text via pio_als_last_error(NULL); arguments are checked before any device
 * work. */
typedef struct pio_cls_folds pio_cls_folds;

/* label: n (HOST), x: n x n_feat (HOST); 1 <= n < 2^31, n_feat >= 1, k_fold >= 1. */
PIO_API int pio_cls_folds_create(int device, const double* label, const double* x, int64_t n, int32_t n_feat,
                                 int32_t k_fold, pio_cls_folds** out);
/* out[0] training rows, out[1] test rows of fold `fold`. */
PIO_API int pio_cls_folds_sizes(const pio_cls_folds* f, int32_t fold, int64_t out[2]);
/* The distinct labels of the fold's training rows, ascending (np.unique of them): *n_class their number, labels
 * (nullable) receives them. */
PIO_API int pio_cls_folds_classes(const pio_cls_folds* f, int32_t fold, int32_t* n_class, double* labels);
/* pio_nb_train on the fold's training rows: features rounded to float32, class = index among the fold's training
 * labels.  n_class must be the fold's (pio_cls_folds_classes); pi: n_class, theta: n_class x n_feat (HOST).  A negative
 * float32 feature in a training row fails with PIO_ALS_ERR_NUMERIC and MLlib's message. */
PIO_API int pio_cls_folds_nb_train(pio_cls_folds* f, int32_t fold, double lambda, int32_t n_class, double* pi,
                                   double* theta);
/* pio_rf_train on the fold's training rows, with its checks and messages (a row number is the row's position in the
 * fold's training set); the forest is identical to pio_rf_train's on those rows copied to the host. */
PIO_API int pio_cls_folds_rf_train(pio_cls_folds* f, int32_t fold, const pio_rf_params* params, pio_rf_forest** out);
/* Predicts every test row of the fold and keeps the predicted labels on the object (8 bytes per row) until
 * pio_cls_folds_result_free: nb_predict with a NaiveBayes model (pio_nb_predict's class index -> class_label[index],
 * class_label: n_class entries), rf_predict with a forest given as pio_rf_predict takes it (label = class index). */
PIO_API int pio_cls_folds_nb_predict(pio_cls_folds* f, int32_t fold, int32_t n_class, const double* pi,
                                     const double* theta, const double* class_label, int32_t* out_result);
PIO_API int pio_cls_folds_rf_predict(pio_cls_folds* f, int32_t fold, int32_t n_trees, const int32_t* tree_off,
                                     int64_t n_nodes, const int32_t* feature, const double* threshold,
                                     const int32_t* left, const int32_t* right, const int32_t* prediction,
                                     int32_t num_classes, int32_t* out_result);
/* The predicted label of every test row of the result's fold, in row order (HOST, out[1] of pio_cls_folds_sizes). */
PIO_API int pio_cls_folds_result_labels(const pio_cls_folds* f, int32_t result, double* out);
/* out[0] test rows, out[1] rows with predicted == actual label, out[2] rows with predicted == label, out[3] those of
 * out[2] that are correct (fp64 ==).  Accuracy = out[1] / out[0], Precision(label) = out[3] / out[2]. */
PIO_API int pio_cls_folds_result_counts(const pio_cls_folds* f, int32_t result, double label, int64_t out[4]);
PIO_API int pio_cls_folds_result_free(pio_cls_folds* f, int32_t result);
PIO_API int pio_cls_folds_destroy(pio_cls_folds* f);

/* Association rules of the complementary purchase template: its Algorithm.train, which the reference elides
 *   (docs/manual/source/templates/complementarypurchase/dase.html.md.erb:293-314; parameters :241-262).
 * The rules are stated in tests/assoc_ref.py and DESIGN.md 4.15: the buys of each user, in time order, are cut into
 * baskets wherever a gap exceeds basket_window * 1000 ms; a basket is the set of its items; baskets of fewer than
 * min_basket_size items are dropped, T baskets are kept.  Every item set of size 1 .. max_rule_length of a kept basket
 * is counted and is frequent when count >= min_support * T (fp64).  Every frequent S with |S| >= 2 and c in S gives
 * the rule cond = S \ {c} -> c with support = count(S) / T, confidence = count(S) / count(cond), lift = confidence /
 * (count({c}) / T) in fp64, kept when confidence >= min_confidence and lift >= min_lift; per cond the rules are ranked
 * by lift descending, then by c ascending (this project's tie rule), and cut at max_num_rules_per_cond.
 * Errors: status codes as above, text via pio_als_last_error(NULL).  Parameters and indices are checked on the host
 * before any device work. */
typedef struct pio_assoc_params {
  int32_t basket_window;            /* seconds */
  int32_t max_rule_length;          /* >= 2 */
  double min_support;               /* [0, 1] */
  double min_confidence;            /* [0, 1] */
  double min_lift;
  int32_t min_basket_size;          /* >= 2 */
  int32_t max_num_rules_per_cond;   /* >= 1 */
} pio_assoc_params;

typedef struct pio_assoc_model pio_assoc_model;   /* a trained model, host memory only */

/* Most candidate item sets one level may count (about 40 bytes of device memory each).  Before a level is enumerated
 * its candidates -- the extensions of every occurrence of a frequent set one item shorter by the later frequent items
 * of its basket -- are counted exactly; above this limit pio_assoc_train fails with PIO_ALS_ERR_ARG naming minSupport,
 * maxRuleLength and basketWindow, and nothing is allocated or launched for that level. */
#define PIO_ASSOC_MAX_CANDIDATES (1ll << 29)

/* n buy events (HOST): user in [0, n_users), item in [0, n_items) (the item index orders ties), t_ms milliseconds
 * since the epoch; 0 <= n < 2^32.  No basket surviving min_basket_size gives an empty model, not an error. */
PIO_API int pio_assoc_train(int device, const int32_t* user, const int32_t* item, const int64_t* t_ms, int64_t n,
                            int32_t n_users, int32_t n_items, const pio_assoc_params* params, pio_assoc_model** out);
/* The model's size: levels (the longest frequent set), frequent sets over all levels, rules, and T. */
PIO_API int pio_assoc_model_size(const pio_assoc_model* m, int32_t* n_levels, int64_t* n_sets, int64_t* n_rules,
                                 int64_t* n_transactions);
/* Flat arrays.  Sets, by length, then in lexicographic order of their items (ascending in each set): level_off
 * [n_levels + 1] (the sets of length l are [level_off[l - 1], level_off[l])), and per set: set_prefix (the set without
 * its largest item, as an index into these arrays; -1 for a single item), set_item (its largest item) and set_count.
 * Rules, grouped by cond in set order and ranked within each cond: rule_cond (set index), rule_conseq (item), support,
 * confidence, lift.  Any output pointer may be null. */
PIO_API int pio_assoc_model_get(const pio_assoc_model* m, int64_t* level_off, int64_t* set_prefix, int32_t* set_item,
                                int64_t* set_count, int64_t* rule_cond, int32_t* rule_conseq, double* support,
                                double* confidence, double* lift);
PIO_API int pio_assoc_model_destroy(pio_assoc_model* m);

#ifdef __cplusplus
}
#endif
#endif /* PIO_ALS_H_ */
