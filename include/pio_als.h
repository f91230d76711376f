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

/* Item co-occurrence of the similarproduct template's CooccurrenceAlgorithm.trainCooccurrence
 * (examples/scala-parallel-similarproduct/multi-events-multi-algos/src/main/scala/CooccurrenceAlgorithm.scala:72-105):
 * (user, item) view events (indices, HOST) -> distinct -> for every user all item pairs -> count per pair -> for every item the
 * topn co-occurring items with the largest counts.  out_item / out_count are n_items x topn (padded with -1 / 0),
 * out_n[i] = number of valid entries of item i.  Ties (unspecified in the reference): larger count first, then the smaller
 * item index.  Limits: n_items <= 2^20, fewer than 2^31 (user, item1, item2) triples. */
PIO_API int pio_cooc_train(int device, const int32_t* user, const int32_t* item, int64_t n, int32_t n_users,
                           int32_t n_items, int topn, int32_t* out_item, int32_t* out_count, int32_t* out_n);

/* MLlib multinomial NaiveBayes (classification template). HOST buffers.
 * label: class index 0..n_class-1; x: n x n_feat, non-negative. pi: n_class, theta: n_class x n_feat
 * (fp64 log-probabilities, as MLlib's NaiveBayesModel.pi/theta). */
PIO_API int pio_nb_train(int device, const int32_t* label, const float* x, int64_t n, int n_feat,
                         int n_class, double lambda, double* pi, double* theta);
PIO_API int pio_nb_predict(int device, const float* x, int64_t n, int n_feat, int n_class,
                           const double* pi, const double* theta, int32_t* out_label);

#ifdef __cplusplus
}
#endif
#endif /* PIO_ALS_H_ */
