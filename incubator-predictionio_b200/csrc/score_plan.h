// score_plan.h -- which kernels a top-k scoring call runs, and with what geometry.  Pure host C++17: no CUDA header and
// no handle, so the rules can be checked without a GPU (tests/test_scoring_plan.py compiles this header alone).
// pio_als.cu asks for a plan and executes it.  Paths (the names of tests/test_gpu_scoring.py and DESIGN.md 4.6):
//
//   R1 recommend, n == 1, KP <= 64, topk <= 128       score_one      S1 one query of 1..8 ids, KP <= 64, topk <= 128
//   R2 n <= 16, topk <= 128 (serving arenas)         dot_batched    S2 one query of 1..40 ids, topk <= 128 (arenas)
//   R3 n > 16, KP <= 64, topk <= 32                  dot_blocked    S3 batch, KP <= 64, topk <= 32, <= 8 valid / query
//   R4 otherwise, several passes above topk 128      dot_batched    S4 batch, <= 40 valid vectors per 8-query group
//                                                                   S5 the rest, one query at a time: cos_batched if
//                                                                      its shared memory fits 100 KB, else cos_fallback
//
// Filtered calls (pio_als_recommend_filtered / pio_als_similar_batch_filtered): the queries with a white list take the
// listed route (L: score_listed, one CTA per query, any rank and topk); the others are scanned by the batch kernels in
// their filtered instantiation -- R3 / R4 whatever the number of users (plan_recommend_filtered), S3 / S4 as
// plan_similar_batch decides; S5 queries of a filtered call get their dense mask from the host.  The single-query
// paths never run for a filtered call.
//
// The similar paths are decided in three steps, as the information arrives: plan_similar before any launch (S1, S2, the
// batch gather, or per query); plan_similar_batch once the gather says which query items own a factor (S3, S4, or S5);
// plan_similar_query for every S5 query after its own gather.
#pragma once
#include <stddef.h>

#include <vector>

#include "../../include/pio_als.h"
#include "topk_geometry.h"

namespace pio {

constexpr int GROUP_CHUNK = 32768;              // query groups per launch (grid.y is limited to 65535)
constexpr size_t S5_SMEM_LIMIT = 100 * 1024;    // S5: cos_batched up to this much shared memory, cos_fallback above

struct ScoreEnv {
  int kp;              // padded rank: 16, 32, 64 or 128
  int sm_count;
  int n_internal;      // item rows the kernels scan
  bool serve_fused;    // PIO_ALS_SERVE_FUSED: single queries may take score_one
  bool score_blocked;  // PIO_ALS_SCORE_BLOCKED: batches may take the blocked kernels
};

enum ScoreRoute {
  ROUTE_NONE,       // nothing to launch
  ROUTE_ONE,        // R1 / S1: score_one_kernel; the host polls a flag in the mapped arena
  ROUTE_ARENA,      // R2 / S2: serving arenas, results merged into mapped host memory, one synchronisation
  ROUTE_BATCH,      // R3 / R4; similar: gather every query vector, then plan_similar_batch
  ROUTE_PER_QUERY,  // S5 for every query of the call (plan_similar_query)
};

struct ScorePlan {
  ScoreRoute route = ROUTE_NONE;
  unsigned kernel = 0;      // PIO_ALS_PATH_* bit of the scoring kernel (0: none, or not decided yet)
  int threads = 0;          // block of the scoring kernel
  int gx = 0;               // grid.x: persistent CTAs per query group
  int ngroups = 0;          // query groups of the call
  int qpg = 0;              // queries per group (0: bins of varying size, cos_blocked)
  int chunk = GROUP_CHUNK;  // query groups per launch
  int lists = 0;            // candidate lists per query, pass_k entries each
  int pass_k = 0;           // results per pass: min(topk, TK_MAXK)
  int passes = 0;           // passes of pass_k results (bounded by the last result of the one before)
  size_t smem = 0;          // dynamic shared memory of the scoring kernel
  int nvp = 0;              // score_one: query vectors per pass (1, 2, 4, 8)
  bool filtered = false;    // the scan kernel runs in its filtered instantiation (per-query test at the pool insertion)
  // the bits a launch of the scoring kernel records
  unsigned launch_bits() const { return kernel | (filtered ? (unsigned)PIO_ALS_FPATH_FILTERED : 0u); }
  // every bit the call leaves in pio_als_stats.last_score_path
  unsigned path() const { return launch_bits() | (passes > 1 ? (unsigned)PIO_ALS_PATH_MULTI_PASS : 0u); }
};

// persistent CTAs: `want`, but at least eight tiles / steps of `steps` each (the pools must warm up), and at least one
inline int persistent_gx(int want, int steps) {
  const int most = (steps + 7) / 8;
  const int gx = want < most ? want : most;
  return gx < 1 ? 1 : gx;
}
inline int sb_tiles(const ScoreEnv& e) { return (e.n_internal + SB_THREADS - 1) / SB_THREADS; }
inline int db_steps(const ScoreEnv& e) { return (e.n_internal + DB_RINGS * DB_ROWS - 1) / (DB_RINGS * DB_ROWS); }

inline void set_passes(ScorePlan& p, int topk) {
  p.pass_k = topk < TK_MAXK ? topk : TK_MAXK;
  p.passes = (topk + TK_MAXK - 1) / TK_MAXK;
}
// score_dot_topk_batched_kernel / score_cos_topk_multi_kernel: ngroups groups of qpg queries
inline void set_batched(ScorePlan& p, const ScoreEnv& e, unsigned kernel, int n_queries, int qpg, int topk) {
  set_passes(p, topk);
  p.kernel = kernel;
  p.threads = SB_THREADS;
  p.qpg = qpg;
  p.ngroups = (n_queries + qpg - 1) / qpg;
  p.gx = persistent_gx((2 * e.sm_count + p.ngroups - 1) / p.ngroups, sb_tiles(e));
  p.lists = p.gx;
  p.smem = kernel == PIO_ALS_PATH_DOT_BATCHED ? dot_batched_smem_bytes(e.kp, p.pass_k) : cos_multi_smem_bytes(e.kp, p.pass_k);
}
// score_dot_blocked_kernel / score_cos_blocked_kernel: ngroups groups of SB_QB queries or DB_WPR bins; topk <= DB_MAXK
inline void set_blocked(ScorePlan& p, const ScoreEnv& e, unsigned kernel, int ngroups, int qpg, int topk) {
  set_passes(p, topk);
  p.kernel = kernel;
  p.threads = 32 * DB_WARPS;
  p.qpg = qpg;
  p.ngroups = ngroups;
  p.gx = persistent_gx((e.sm_count + ngroups - 1) / ngroups, db_steps(e));
  p.lists = p.gx * DB_RINGS;
  p.smem = db_smem_bytes(e.kp, p.pass_k);
}

inline bool one_ok(const ScoreEnv& e, int nq, int topk) {
  return e.serve_fused && e.kp <= 64 && topk <= TK_MAXK && nq >= 1 && nq <= S1_MAXNV;
}
// R1 / S1: one CTA per SM, at most one per S1_THREADS items; the list merge reads one list head per thread
inline ScorePlan plan_one(const ScoreEnv& e, bool cos, int nq, int topk) {
  ScorePlan p;
  p.route = ROUTE_ONE;
  p.kernel = PIO_ALS_PATH_SCORE_ONE;
  set_passes(p, topk);
  p.threads = S1_THREADS;
  const int ntiles = (e.n_internal + S1_THREADS - 1) / S1_THREADS;
  int gx = e.sm_count < ntiles ? e.sm_count : ntiles;
  if (gx > S1_THREADS) gx = S1_THREADS;
  p.gx = gx < 1 ? 1 : gx;
  p.ngroups = 1;
  p.qpg = 1;
  p.lists = p.gx;
  p.nvp = !cos ? 1 : nq <= 1 ? 1 : nq <= 2 ? 2 : nq <= 4 ? 4 : 8;
  p.smem = s1_smem_bytes(e.kp, p.nvp, topk);
  return p;
}

// pio_als_recommend for n users
inline ScorePlan plan_recommend(const ScoreEnv& e, int n, int topk) {
  ScorePlan p;
  if (n < 1 || topk < 1) return p;
  if (n == 1 && one_ok(e, 1, topk)) return plan_one(e, false, 1, topk);
  if (n <= SB_QB && topk <= TK_MAXK) {
    set_batched(p, e, PIO_ALS_PATH_DOT_BATCHED, n, SB_QB, topk);
    p.route = ROUTE_ARENA;
  } else if (e.score_blocked && e.kp <= 64 && topk <= DB_MAXK) {
    set_blocked(p, e, PIO_ALS_PATH_DOT_BLOCKED, (n + SB_QB - 1) / SB_QB, SB_QB, topk);
    p.route = ROUTE_BATCH;
  } else {
    set_batched(p, e, PIO_ALS_PATH_DOT_BATCHED, n, SB_QB, topk);
    p.route = ROUTE_BATCH;
  }
  return p;
}

// the scanned users of a filtered recommend call: never the single-query or arena routes
inline ScorePlan plan_recommend_filtered(const ScoreEnv& e, int n, int topk) {
  ScorePlan p;
  if (n < 1 || topk < 1) return p;
  if (e.score_blocked && e.kp <= 64 && topk <= DB_MAXK)
    set_blocked(p, e, PIO_ALS_PATH_DOT_BLOCKED, (n + SB_QB - 1) / SB_QB, SB_QB, topk);
  else
    set_batched(p, e, PIO_ALS_PATH_DOT_BATCHED, n, SB_QB, topk);
  p.route = ROUTE_BATCH;
  p.filtered = true;
  return p;
}

// L: the n white-listed queries of a filtered call, one CTA each, one candidate list per warp
inline ScorePlan plan_listed(int n, int topk) {
  ScorePlan p;
  if (n < 1 || topk < 1) return p;
  set_passes(p, topk);
  p.route = ROUTE_BATCH;
  p.kernel = PIO_ALS_FPATH_LISTED;
  p.threads = LS_THREADS;
  p.gx = 1;
  p.ngroups = n;
  p.qpg = 1;
  p.lists = LS_WARPS;
  p.smem = listed_smem_bytes(p.pass_k);
  return p;
}

// Which queries of a filtered call are listed and which are scanned: has_wl[j] != 0 sends query j to the listed route
// (has_wl == nullptr: none).  Both lists keep the call's order; results go back to row listed[i] / scanned[i].
inline void split_listed(const unsigned char* has_wl, int n, std::vector<int>* listed, std::vector<int>* scanned) {
  listed->clear();
  scanned->clear();
  for (int j = 0; j < n; ++j) (has_wl && has_wl[j] ? listed : scanned)->push_back(j);
}

// the scanned queries of a filtered similar call before any launch: the batch gather, or per query (S5)
inline ScorePlan plan_similar_filtered(int n_queries, long long total, int topk) {
  ScorePlan p;
  if (n_queries < 1 || topk < 1) return p;
  p.route = total > 0 && total < (1ll << 31) ? ROUTE_BATCH : ROUTE_PER_QUERY;
  return p;
}

// pio_als_similar_batch before any launch: len0 = ids of the first query, total = ids of all queries
inline ScorePlan plan_similar(const ScoreEnv& e, int n_queries, long long len0, long long total, int topk) {
  ScorePlan p;
  if (n_queries < 1 || topk < 1) return p;
  if (n_queries == 1 && one_ok(e, (int)(len0 < (1 << 20) ? len0 : (1 << 20)), topk)) return plan_one(e, true, (int)len0, topk);
  if (n_queries == 1 && len0 >= 1 && len0 <= SM_NV && topk <= TK_MAXK) {   // ids, valid or not: no host round trip
    set_batched(p, e, PIO_ALS_PATH_COS_MULTI, 1, SM_QG, topk);
    p.route = ROUTE_ARENA;
    return p;
  }
  p.route = n_queries > 1 && total > 0 && total < (1ll << 31) ? ROUTE_BATCH : ROUTE_PER_QUERY;
  return p;
}

// A gathered batch: nvalid[j] = query vectors (ids with a factor) of query j.  S3 packs consecutive queries into bins of
// <= CB_QPW queries and <= DB_QW vectors; S4 takes groups of SM_QG queries with <= SM_NV vectors each.  q0 receives the
// first query of every bin / group and the end (n_queries); a query with too many vectors for either sends the whole
// batch to S5 (route ROUTE_PER_QUERY).
inline ScorePlan plan_similar_batch(const ScoreEnv& e, const std::vector<int>& nvalid, int topk, std::vector<int>* q0) {
  const int n = (int)nvalid.size();
  ScorePlan p;
  q0->clear();
  bool fits = e.score_blocked && e.kp <= 64 && topk <= DB_MAXK;
  for (int j = 0, bq = 0, bv = 0; j < n && fits; ++j) {   // bq / bv: queries / vectors in the open bin
    if (nvalid[j] > DB_QW) fits = false;
    else if (j == 0 || bq == CB_QPW || bv + nvalid[j] > DB_QW) {
      q0->push_back(j);
      bq = bv = 0;
    }
    ++bq;
    bv += nvalid[j];
  }
  if (fits) {
    q0->push_back(n);
    set_blocked(p, e, PIO_ALS_PATH_COS_BLOCKED, ((int)q0->size() - 1 + DB_WPR - 1) / DB_WPR, 0, topk);
    p.route = ROUTE_BATCH;
    return p;
  }
  q0->clear();
  for (int g = 0; g * SM_QG < n; ++g) {
    int nv = 0;
    for (int j = g * SM_QG; j < (g + 1) * SM_QG && j < n; ++j) nv += nvalid[j];
    if (nv > SM_NV) {
      q0->clear();
      p.route = ROUTE_PER_QUERY;
      return p;
    }
    q0->push_back(g * SM_QG);
  }
  q0->push_back(n);
  set_batched(p, e, PIO_ALS_PATH_COS_MULTI, n, SM_QG, topk);
  p.route = ROUTE_BATCH;
  return p;
}

// S5, one query after its gather: nqv of its nq ids own a factor.  No valid vector: nothing to score.
inline ScorePlan plan_similar_query(const ScoreEnv& e, int nqv, int nq, int topk) {
  ScorePlan p;
  if (nqv < 1) return p;
  p.route = ROUTE_PER_QUERY;
  set_passes(p, topk);
  p.ngroups = 1;
  p.qpg = 1;
  const size_t smem = cos_batched_smem_bytes(e.kp, nqv, nq, p.pass_k);
  if (smem <= S5_SMEM_LIMIT) {
    p.kernel = PIO_ALS_PATH_COS_BATCHED;
    p.threads = SB_THREADS;
    p.gx = persistent_gx(2 * e.sm_count, sb_tiles(e));
    p.lists = p.gx * (SB_THREADS / 32);   // one pool per warp
    p.smem = smem;
  } else {
    p.kernel = PIO_ALS_PATH_COS_FALLBACK;
    p.threads = TK_THREADS;
    p.gx = (e.n_internal + TK_TILE - 1) / TK_TILE;
    p.lists = p.gx;
  }
  return p;
}

}  // namespace pio
