/*
 * als_oracle.c -- CPU ORACLE (TEST INFRASTRUCTURE, NOT PRODUCT CODE).
 *
 * A plain-C/OpenMP restatement of the arithmetic that PredictionIO's engine
 * templates delegate to Spark MLlib:
 *
 *   - `als.run(mllibRatings)`                       (reference call site:
 *     examples/scala-parallel-recommendation/blacklist-items/src/main/scala/ALSAlgorithm.scala:76-86)
 *   - `ALS.trainImplicit(ratings, rank, iterations, lambda, blocks=-1, alpha=1.0, seed)`
 *     (examples/scala-parallel-similarproduct/multi-events-multi-algos/src/main/scala/ALSAlgorithm.scala:121-128)
 *   - `ALS.train(ratings, rank, iterations, lambda, -1, seed)`
 *     (examples/scala-parallel-ecommercerecommendation/train-with-rate-event/src/main/scala/ECommAlgorithm.scala:116-122)
 *   - `recommendProductsWithFilter` / `recommend`   (.../blacklist-items/src/main/scala/ALSModel.scala:44-60)
 *   - similarproduct `predict` / `cosine` / `getTopN`
 *     (.../multi-events-multi-algos/src/main/scala/ALSAlgorithm.scala:138-234)
 *   - `NaiveBayes.train(labeledPoints, lambda)`
 *     (examples/scala-parallel-classification/add-algorithm/src/main/scala/NaiveBayesAlgorithm.scala:41-57)
 *
 * The arithmetic itself lives in the third-party, un-vendored dependency
 * org.apache.spark:spark-mllib_2.11:2.4.0 (`provided`, e.g.
 * examples/scala-parallel-recommendation/blacklist-items/build.sbt:24), which is
 * absent from /root/reference and cannot run in this environment (no JVM).
 * This file restates Spark 2.4 `ml.recommendation.ALS.train` semantics as laid
 * out in SURVEY.md section 8(c) items 1-8:
 *   fp32 ratings and factors; per destination row a packed-upper fp64 normal
 *   equation (dspr rank-1 updates + daxpy), ridge lambda*n added to the
 *   diagonal, packed Cholesky solve (dppsv), result narrowed to fp32;
 *   every iteration = item half-step (from user factors) then user half-step
 *   (from item factors); implicit mode adds YtY over all source rows and uses
 *   confidence c1 = alpha*|r|, b += (1+c1)*y only for r > 0, n = #(r > 0).
 *
 * PARITY UNPINNED: the reference's own tests hold no golden vector for ALS
 * (tests/pio_tests/scenarios/quickstart_test.py:163-167 only checks
 * len(itemScores)==4), and MLlib cannot be executed here, so this oracle is
 * validated by mathematical invariants (tests/test_oracle.py) and not against
 * reference outputs.
 *
 * Only tests/, __graft_entry__.smoke() and bench.py's cpu_baseline /
 * --impl reference leg may load this library.
 */
#include <math.h>
#include <stdint.h>
#include <stdlib.h>
#include <string.h>
#ifdef _OPENMP
#include <omp.h>
#endif

#define ORACLE_API __attribute__((visibility("default")))

/* ------------------------------------------------------------------ */
/* CSR build: stable counting sort of COO by row (rows with no entry   */
/* get an empty range). Order inside a row = input order, mirroring    */
/* MLlib's in-block arrays where duplicate (row,col) stay separate     */
/* (SURVEY 8(c) 5b).                                                   */
/* ------------------------------------------------------------------ */
ORACLE_API int oracle_csr_build(int32_t n_rows, int64_t nnz, const int32_t *row,
                                const int32_t *col, const float *val,
                                int64_t *ptr /* n_rows+1 */, int32_t *out_col,
                                float *out_val) {
  memset(ptr, 0, sizeof(int64_t) * ((size_t)n_rows + 1));
  for (int64_t e = 0; e < nnz; ++e) {
    if (row[e] < 0 || row[e] >= n_rows) return -1;
    ptr[row[e] + 1]++;
  }
  for (int32_t r = 0; r < n_rows; ++r) ptr[r + 1] += ptr[r];
  int64_t *cur = (int64_t *)malloc(sizeof(int64_t) * (size_t)(n_rows > 0 ? n_rows : 1));
  if (!cur) return -2;
  memcpy(cur, ptr, sizeof(int64_t) * (size_t)n_rows);
  for (int64_t e = 0; e < nnz; ++e) {
    int64_t p = cur[row[e]]++;
    out_col[p] = col[e];
    out_val[p] = val[e];
  }
  free(cur);
  return 0;
}

/* ------------------------------------------------------------------ */
/* Packed-upper helpers. Layout = LAPACK 'U' packed, column-major:     */
/* element (i,j), i<=j, at ata[j*(j+1)/2 + i]  (diagonal at 0,2,5,9..) */
/* ------------------------------------------------------------------ */

/* dspr('U', k, alpha, x, ata): ata += alpha * x x^T (upper part) */
static inline void dspr_upper(int k, double alpha, const double *x, double *ata) {
  for (int j = 0; j < k; ++j) {
    const double t = alpha * x[j];
    double *colp = ata + (size_t)j * (j + 1) / 2;
    for (int i = 0; i <= j; ++i) colp[i] += x[i] * t;
  }
}

/* dppsv('U', k, 1, ata, b): Cholesky A = U^T U on the packed upper triangle,
 * then solve U^T y = b, U x = y in place. Returns 0, or j+1 if the leading
 * minor of order j+1 is not positive definite (LAPACK info convention). */
static int dppsv_upper(int k, double *ap, double *b) {
  for (int j = 0; j < k; ++j) {
    double *cj = ap + (size_t)j * (j + 1) / 2;
    /* solve U(0:j,0:j)^T * u = a(0:j, j) */
    for (int i = 0; i < j; ++i) {
      const double *ci = ap + (size_t)i * (i + 1) / 2;
      double s = cj[i];
      for (int t = 0; t < i; ++t) s -= ci[t] * cj[t];
      cj[i] = s / ci[i];
    }
    double d = cj[j];
    for (int t = 0; t < j; ++t) d -= cj[t] * cj[t];
    if (!(d > 0.0)) return j + 1;
    cj[j] = sqrt(d);
  }
  /* forward: U^T y = b */
  for (int j = 0; j < k; ++j) {
    const double *cj = ap + (size_t)j * (j + 1) / 2;
    double s = b[j];
    for (int t = 0; t < j; ++t) s -= cj[t] * b[t];
    b[j] = s / cj[j];
  }
  /* backward: U x = y */
  for (int j = k - 1; j >= 0; --j) {
    const double *cj = ap + (size_t)j * (j + 1) / 2;
    b[j] /= cj[j];
    const double xj = b[j];
    for (int t = 0; t < j; ++t) b[t] -= cj[t] * xj;
  }
  return 0;
}

/* YtY over all source rows that own a factor (fp64), SURVEY 8(c)-5. */
ORACLE_API void oracle_gram(int32_t n_rows, int k, const float *f, const uint8_t *has,
                            double *ata /* k(k+1)/2 packed upper */) {
  const int tri = k * (k + 1) / 2;
  memset(ata, 0, sizeof(double) * (size_t)tri);
#pragma omp parallel
  {
    double *loc = (double *)calloc((size_t)tri, sizeof(double));
    double *x = (double *)malloc(sizeof(double) * (size_t)k);
#pragma omp for schedule(static)
    for (int32_t r = 0; r < n_rows; ++r) {
      if (has && !has[r]) continue;
      for (int i = 0; i < k; ++i) x[i] = (double)f[(size_t)r * k + i];
      dspr_upper(k, 1.0, x, loc);
    }
#pragma omp critical
    for (int i = 0; i < tri; ++i) ata[i] += loc[i];
    free(loc);
    free(x);
  }
}

/* ------------------------------------------------------------------ */
/* One half-step over destination rows [row_begin,row_end) with stride */
/* row_stride (stride>1 is used only by bench.py's bounded cpu sample).*/
/* dst rows with an empty rating range are left untouched (MLlib emits */
/* no factor for them).  Returns the number of rows whose Cholesky     */
/* failed (0 on success).                                              */
/* ------------------------------------------------------------------ */
/* normal equation + Cholesky solve of ONE destination row (SURVEY 8(c) items 5-6); scratch ata/atb/da are
 * caller-provided.  Returns 1 if the row was solved into x, 0 if it has no ratings, -1 if dppsv failed. */
static int solve_row(int k, int64_t b, int64_t e, const int32_t *idx, const float *val, const float *src,
                     double lambda, int implicit, double alpha, const double *yty, double *ata, double *atb,
                     double *da, float *x) {
  const int tri = k * (k + 1) / 2;
  if (e == b) return 0;
  if (implicit && yty) memcpy(ata, yty, sizeof(double) * (size_t)tri);
  else memset(ata, 0, sizeof(double) * (size_t)tri);
  memset(atb, 0, sizeof(double) * (size_t)k);
  int64_t n = 0;
  for (int64_t p = b; p < e; ++p) {
    const float *y = src + (size_t)idx[p] * k;
    for (int i = 0; i < k; ++i) da[i] = (double)y[i];
    const double rating = (double)val[p];
    if (implicit) {
      const double c1 = alpha * fabs(rating);
      dspr_upper(k, c1, da, ata);
      if (rating > 0.0) {
        const double w = 1.0 + c1;
        for (int i = 0; i < k; ++i) atb[i] += w * da[i];
        n += 1;
      }
    } else {
      dspr_upper(k, 1.0, da, ata);
      for (int i = 0; i < k; ++i) atb[i] += rating * da[i];
      n += 1;
    }
  }
  const double ridge = lambda * (double)n;
  for (int j = 0; j < k; ++j) ata[(size_t)j * (j + 1) / 2 + j] += ridge;
  if (dppsv_upper(k, ata, atb) != 0) return -1;
  for (int i = 0; i < k; ++i) x[i] = (float)atb[i];
  return 1;
}

ORACLE_API int oracle_als_half_step(int32_t n_dst, int k, const int64_t *ptr,
                                    const int32_t *idx, const float *val,
                                    const float *src, float *dst, double lambda,
                                    int implicit, double alpha,
                                    const double *yty /* packed upper or NULL */,
                                    int32_t row_begin, int32_t row_end,
                                    int32_t row_stride) {
  const int tri = k * (k + 1) / 2;
  int fails = 0;
  if (row_end > n_dst) row_end = n_dst;
  if (row_stride < 1) row_stride = 1;
#pragma omp parallel reduction(+ : fails)
  {
    double *ata = (double *)malloc(sizeof(double) * (size_t)tri);
    double *atb = (double *)malloc(sizeof(double) * (size_t)k);
    double *da = (double *)malloc(sizeof(double) * (size_t)k);
#pragma omp for schedule(dynamic, 16)
    for (int32_t r = row_begin; r < row_end; r += row_stride) {
      if (solve_row(k, ptr[r], ptr[r + 1], idx, val, src, lambda, implicit, alpha, yty, ata, atb, da,
                    dst + (size_t)r * k) < 0)
        fails += 1;
    }
    free(ata);
    free(atb);
    free(da);
  }
  return fails;
}

/* Same arithmetic for an explicit LIST of destination rows (bench.py's parity sample of the benchmarked workload):
 * out is n_list x k, row j = the solution of destination row rows[j] (left untouched if that row has no ratings). */
ORACLE_API int oracle_als_half_step_rows(int k, const int64_t *ptr, const int32_t *idx, const float *val,
                                         const float *src, double lambda, int implicit, double alpha,
                                         const double *yty, const int32_t *rows, int32_t n_list, float *out) {
  const int tri = k * (k + 1) / 2;
  int fails = 0;
#pragma omp parallel reduction(+ : fails)
  {
    double *ata = (double *)malloc(sizeof(double) * (size_t)tri);
    double *atb = (double *)malloc(sizeof(double) * (size_t)k);
    double *da = (double *)malloc(sizeof(double) * (size_t)k);
#pragma omp for schedule(dynamic, 1)
    for (int32_t j = 0; j < n_list; ++j) {
      const int32_t r = rows[j];
      if (solve_row(k, ptr[r], ptr[r + 1], idx, val, src, lambda, implicit, alpha, yty, ata, atb, da,
                    out + (size_t)j * k) < 0)
        fails += 1;
    }
    free(ata);
    free(atb);
    free(da);
  }
  return fails;
}

/* reduceByKey(_ + _) on a CSR (rows in input order, oracle_csr_build): inside every row the entries are ordered by
 * column, ties in input order, and repeated columns are folded left to right in fp32 -- the same result as
 * als_oracle.py dedup_coo(mode="sum") (examples/scala-parallel-similarproduct/multi-events-multi-algos/src/main/
 * scala/ALSAlgorithm.scala:106), fast enough for the 100 M-rating bench workload.  Compacts col/val in place,
 * rewrites ptr, returns the new nnz. */
typedef struct { int32_t c; int32_t pos; float v; } dd_ent;
static int dd_cmp(const void *a, const void *b) {
  const dd_ent *x = (const dd_ent *)a, *y = (const dd_ent *)b;
  if (x->c != y->c) return x->c < y->c ? -1 : 1;
  return x->pos < y->pos ? -1 : (x->pos > y->pos);
}
ORACLE_API int64_t oracle_csr_dedup_sum(int32_t n_rows, int64_t *ptr, int32_t *col, float *val) {
  int64_t *newlen = (int64_t *)calloc((size_t)n_rows + 1, sizeof(int64_t));
  if (!newlen) return -2;
#pragma omp parallel
  {
    dd_ent *buf = NULL;
    int64_t cap = 0;
#pragma omp for schedule(dynamic, 64)
    for (int32_t r = 0; r < n_rows; ++r) {
      const int64_t b = ptr[r], n = ptr[r + 1] - b;
      if (n > cap) {
        free(buf);
        cap = n * 2;
        buf = (dd_ent *)malloc(sizeof(dd_ent) * (size_t)cap);
      }
      for (int64_t t = 0; t < n; ++t) { buf[t].c = col[b + t]; buf[t].pos = (int32_t)t; buf[t].v = val[b + t]; }
      qsort(buf, (size_t)n, sizeof(dd_ent), dd_cmp);
      int64_t o = 0;
      for (int64_t t = 0; t < n;) {
        float acc = buf[t].v;   /* reduceByKey(_ + _): a run of one keeps its value, -0.0 included */
        int64_t u = t + 1;
        while (u < n && buf[u].c == buf[t].c) { acc = acc + buf[u].v; ++u; }
        col[b + o] = buf[t].c;
        val[b + o] = acc;
        ++o;
        t = u;
      }
      newlen[r] = o;
    }
    free(buf);
  }
  int64_t w = 0;
  for (int32_t r = 0; r < n_rows; ++r) {
    const int64_t b = ptr[r], n = newlen[r];
    if (w != b) { memmove(col + w, col + b, sizeof(int32_t) * (size_t)n); memmove(val + w, val + b, sizeof(float) * (size_t)n); }
    ptr[r] = w;
    w += n;
  }
  ptr[n_rows] = w;
  free(newlen);
  return w;
}

/* ------------------------------------------------------------------ */
/* Full training run. user_f / item_f: in = initial factors, out =     */
/* trained factors (row-major, n x k, fp32). user_has/item_has (out):  */
/* 1 if the row occurs in the ratings (owns a factor), else the row is */
/* zeroed (MLlib emits nothing for it).                                */
/* ------------------------------------------------------------------ */
ORACLE_API int oracle_als_train(int32_t n_users, int32_t n_items, int64_t nnz,
                                const int32_t *user, const int32_t *item,
                                const float *rating, int k, int iters, double lambda,
                                int implicit, double alpha, float *user_f,
                                float *item_f, uint8_t *user_has, uint8_t *item_has) {
  int rc = 0;
  int64_t *uptr = (int64_t *)malloc(sizeof(int64_t) * ((size_t)n_users + 1));
  int64_t *iptr = (int64_t *)malloc(sizeof(int64_t) * ((size_t)n_items + 1));
  int32_t *ucol = (int32_t *)malloc(sizeof(int32_t) * (size_t)(nnz > 0 ? nnz : 1));
  int32_t *icol = (int32_t *)malloc(sizeof(int32_t) * (size_t)(nnz > 0 ? nnz : 1));
  float *uval = (float *)malloc(sizeof(float) * (size_t)(nnz > 0 ? nnz : 1));
  float *ival = (float *)malloc(sizeof(float) * (size_t)(nnz > 0 ? nnz : 1));
  uint8_t *uh = (uint8_t *)malloc((size_t)(n_users > 0 ? n_users : 1));
  uint8_t *ih = (uint8_t *)malloc((size_t)(n_items > 0 ? n_items : 1));
  const int tri = k * (k + 1) / 2;
  double *yty = (double *)malloc(sizeof(double) * (size_t)tri);
  if (!uptr || !iptr || !ucol || !icol || !uval || !ival || !uh || !ih || !yty) {
    rc = -2;
    goto done;
  }
  if (oracle_csr_build(n_users, nnz, user, item, rating, uptr, ucol, uval) != 0 ||
      oracle_csr_build(n_items, nnz, item, user, rating, iptr, icol, ival) != 0) {
    rc = -1;
    goto done;
  }
  for (int32_t u = 0; u < n_users; ++u) {
    uh[u] = (uint8_t)(uptr[u + 1] > uptr[u]);
    if (!uh[u]) memset(user_f + (size_t)u * k, 0, sizeof(float) * (size_t)k);
  }
  for (int32_t i = 0; i < n_items; ++i) {
    ih[i] = (uint8_t)(iptr[i + 1] > iptr[i]);
    if (!ih[i]) memset(item_f + (size_t)i * k, 0, sizeof(float) * (size_t)k);
  }
  for (int it = 0; it < iters; ++it) {
    /* item half-step from user factors, then user half-step (SURVEY 8(c)-4) */
    if (implicit) oracle_gram(n_users, k, user_f, uh, yty);
    rc += oracle_als_half_step(n_items, k, iptr, icol, ival, user_f, item_f, lambda,
                               implicit, alpha, implicit ? yty : NULL, 0, n_items, 1);
    if (implicit) oracle_gram(n_items, k, item_f, ih, yty);
    rc += oracle_als_half_step(n_users, k, uptr, ucol, uval, item_f, user_f, lambda,
                               implicit, alpha, implicit ? yty : NULL, 0, n_users, 1);
  }
  if (user_has) memcpy(user_has, uh, (size_t)n_users);
  if (item_has) memcpy(item_has, ih, (size_t)n_items);
done:
  free(uptr); free(iptr); free(ucol); free(icol); free(uval); free(ival);
  free(uh); free(ih); free(yty);
  return rc;
}

/* ------------------------------------------------------------------ */
/* Top-k scoring.                                                      */
/* ------------------------------------------------------------------ */
typedef struct { double s; int32_t i; } scored_t;

/* "better" = larger score; ties broken by smaller index (the reference
 * leaves ties unspecified: RDD.top / PriorityQueue order). */
static inline int better(double s1, int32_t i1, double s2, int32_t i2) {
  return (s1 > s2) || (s1 == s2 && i1 < i2);
}

static void topk_insert(scored_t *heap, int *n, int k, double s, int32_t i) {
  /* small k: keep a sorted array, best first */
  if (*n == k && !better(s, i, heap[k - 1].s, heap[k - 1].i)) return;
  int pos = (*n < k) ? (*n)++ : k - 1;
  while (pos > 0 && better(s, i, heap[pos - 1].s, heap[pos - 1].i)) {
    heap[pos] = heap[pos - 1];
    --pos;
  }
  heap[pos].s = s;
  heap[pos].i = i;
}

/* recommendProducts(WithFilter): score_i = ddot(x_u, y_i) in fp64 over the
 * fp32->fp64 widened factors (ALSModel.scala:52-58); items with has==0 own no
 * factor and are not candidates; mask[i]!=0 excludes item i (blackList,
 * ALSAlgorithm.scala:104-106). Unknown user (has==0) -> count 0
 * (ALSAlgorithm.scala:109-112). out_* are n_q x topk, padded with -1 / 0. */
ORACLE_API void oracle_recommend(int32_t n_items, int k, const float *user_f,
                                 const uint8_t *user_has, const float *item_f,
                                 const uint8_t *item_has, const int32_t *users, int n_q,
                                 int topk, const uint8_t *mask, const double *weight,
                                 int32_t *out_items, float *out_scores, int32_t *out_count) {
  /* weight (nullable): adjustedScore = s * weights(i), the ecommerce template's weightedItems
   * (examples/scala-parallel-ecommercerecommendation/adjust-score/src/main/scala/ECommAlgorithm.scala:490-497) */
#pragma omp parallel for schedule(dynamic, 1)
  for (int q = 0; q < n_q; ++q) {
    scored_t *best = (scored_t *)malloc(sizeof(scored_t) * (size_t)(topk > 0 ? topk : 1));
    int n = 0;
    const int32_t u = users[q];
    if (u >= 0 && (!user_has || user_has[u])) {
      const float *x = user_f + (size_t)u * k;
      for (int32_t i = 0; i < n_items; ++i) {
        if (item_has && !item_has[i]) continue;
        if (mask && mask[i]) continue;
        const float *y = item_f + (size_t)i * k;
        double s = 0.0;
        for (int t = 0; t < k; ++t) s += (double)x[t] * (double)y[t];
        if (weight) s = s * weight[i];
        topk_insert(best, &n, topk, s, i);
      }
    }
    for (int t = 0; t < topk; ++t) {
      out_items[(size_t)q * topk + t] = t < n ? best[t].i : -1;
      out_scores[(size_t)q * topk + t] = t < n ? (float)best[t].s : 0.0f;
    }
    if (out_count) out_count[q] = n;
    free(best);
  }
}

/* similarproduct predict: score_i = sum_q cosine(y_q, y_i) (fp64), keep
 * score > 0, drop the query items themselves and masked items, top-N
 * (ALSAlgorithm.scala:138-197, cosine :220-234). Query items without a
 * factor are skipped (:146-149). */
ORACLE_API void oracle_similar(int32_t n_items, int k, const float *item_f,
                               const uint8_t *item_has, const int32_t *query, int nq,
                               int topk, const uint8_t *mask, const double *weight,
                               int keep_query /* ecommerce predictSimilar: query items stay candidates */,
                               int32_t *out_items, float *out_scores, int32_t *out_count) {
  scored_t *best = (scored_t *)malloc(sizeof(scored_t) * (size_t)(topk > 0 ? topk : 1));
  int n = 0;
  int nvalid = 0;
  for (int q = 0; q < nq; ++q)
    if (query[q] >= 0 && query[q] < n_items && (!item_has || item_has[query[q]])) nvalid++;
  if (nvalid > 0) {
    for (int32_t i = 0; i < n_items; ++i) {
      if (item_has && !item_has[i]) continue;
      if (mask && mask[i]) continue;
      int is_query = 0;
      for (int q = 0; q < nq; ++q) if (query[q] == i) is_query = 1;
      if (is_query && !keep_query) continue;
      const float *f = item_f + (size_t)i * k;
      double score = 0.0;
      for (int q = 0; q < nq; ++q) {
        const int32_t qi = query[q];
        if (qi < 0 || qi >= n_items || (item_has && !item_has[qi])) continue;
        const float *qf = item_f + (size_t)qi * k;
        double n1 = 0, n2 = 0, d = 0;
        for (int t = 0; t < k; ++t) {
          n1 += (double)qf[t] * (double)qf[t];
          n2 += (double)f[t] * (double)f[t];
          d += (double)qf[t] * (double)f[t];
        }
        const double n1n2 = sqrt(n1) * sqrt(n2);
        score += (n1n2 == 0.0) ? 0.0 : d / n1n2;
      }
      if (weight) score = score * weight[i];
      if (score > 0.0) topk_insert(best, &n, topk, score, i);
    }
  }
  for (int t = 0; t < topk; ++t) {
    out_items[t] = t < n ? best[t].i : -1;
    out_scores[t] = t < n ? (float)best[t].s : 0.0f;
  }
  if (out_count) *out_count = n;
  free(best);
}

/* ------------------------------------------------------------------ */
/* MLlib multinomial NaiveBayes (SURVEY 8(a) A11, 8(c)-8):             */
/*   pi_c = log(n_c + lambda) - log(N + C*lambda)                      */
/*   theta_cj = log(s_cj + lambda) - log(sum_j s_cj + F*lambda)        */
/* labels are class indices 0..C-1 (already sorted ascending).         */
/* ------------------------------------------------------------------ */
ORACLE_API void oracle_nb_train(int64_t n, int n_feat, int n_class, const int32_t *label,
                                const float *x /* n x n_feat */, double lambda,
                                double *pi /* C */, double *theta /* C x F */) {
  double *cnt = (double *)calloc((size_t)n_class, sizeof(double));
  double *sum = (double *)calloc((size_t)n_class * n_feat, sizeof(double));
  for (int64_t r = 0; r < n; ++r) {
    const int c = label[r];
    cnt[c] += 1.0;
    for (int j = 0; j < n_feat; ++j) sum[(size_t)c * n_feat + j] += (double)x[(size_t)r * n_feat + j];
  }
  const double logden = log((double)n + n_class * lambda);
  for (int c = 0; c < n_class; ++c) {
    pi[c] = log(cnt[c] + lambda) - logden;
    double tot = 0;
    for (int j = 0; j < n_feat; ++j) tot += sum[(size_t)c * n_feat + j];
    const double lt = log(tot + n_feat * lambda);
    for (int j = 0; j < n_feat; ++j)
      theta[(size_t)c * n_feat + j] = log(sum[(size_t)c * n_feat + j] + lambda) - lt;
  }
  free(cnt);
  free(sum);
}

ORACLE_API void oracle_nb_predict(int64_t n, int n_feat, int n_class, const float *x,
                                  const double *pi, const double *theta, int32_t *out) {
#pragma omp parallel for schedule(static)
  for (int64_t r = 0; r < n; ++r) {
    int bestc = 0;
    double bests = -INFINITY;
    for (int c = 0; c < n_class; ++c) {
      double s = pi[c];
      for (int j = 0; j < n_feat; ++j)
        s += theta[(size_t)c * n_feat + j] * (double)x[(size_t)r * n_feat + j];
      if (s > bests) { bests = s; bestc = c; }
    }
    out[r] = bestc;
  }
}

ORACLE_API int oracle_num_threads(void) {
#ifdef _OPENMP
  return omp_get_max_threads();
#else
  return 1;
#endif
}

ORACLE_API void oracle_set_num_threads(int n) {
#ifdef _OPENMP
  if (n > 0) omp_set_num_threads(n);
#else
  (void)n;
#endif
}
