// topk_geometry.h -- launch geometry of the top-k scoring kernels (topk.cuh): block sizes, pool shapes, and the dynamic
// shared memory of every kernel that takes any.  The kernels and the host-side planner (score_plan.h) read these
// definitions and nothing else, so a size can only change in one place.  Plain C++17: compiles under nvcc and g++.
#pragma once
#include <stddef.h>

#if defined(__CUDACC__)
#define PIO_HD __host__ __device__
#else
#define PIO_HD
#endif

namespace pio {

constexpr int TK_THREADS = 256;
constexpr int TK_ITEMS = 4;                       // items per thread
constexpr int TK_TILE = TK_THREADS * TK_ITEMS;    // items per CTA
constexpr int TK_MAXK = 128;                      // max supported topk

struct ScoreIdx {
  double s;
  int i;
};

// ---- score_dot_topk_batched_kernel: one item per thread, SB_QB queries per CTA ----
constexpr int SB_THREADS = 256;
constexpr int SB_QB = 16;
// staged tile [SB_THREADS][kp + 4] floats, large enough to be reused for the [SB_QB][SB_THREADS] fp64 score exchange + ids
PIO_HD inline size_t sb_tile_bytes(int kp) {
  const size_t a = sizeof(float) * (size_t)SB_THREADS * (kp + 4);
  const size_t b = sizeof(double) * (size_t)SB_QB * SB_THREADS + sizeof(int) * SB_THREADS;
  return a > b ? a : b;
}
// query values [kp][SB_QB] fp64, the staged tile, the pools [SB_QB][topk]
PIO_HD inline size_t dot_batched_smem_bytes(int kp, int topk) {
  return sizeof(double) * (size_t)kp * SB_QB + sb_tile_bytes(kp) + (sizeof(double) + sizeof(int)) * (size_t)SB_QB * topk;
}

// ---- score_dot_blocked_kernel / score_cos_blocked_kernel: rings of two warps, eight queries (vectors) per warp ----
constexpr int DB_QW = 8;                     // queries per warp
constexpr int DB_WPR = SB_QB / DB_QW;        // warps per ring
constexpr int DB_RINGS = 8;
constexpr int DB_WARPS = DB_RINGS * DB_WPR;  // 16
constexpr int DB_ROWS = 64;                  // rows per ring step (two per lane)
constexpr int DB_STAGES = 1;                 // a ring waits for its own rows while the other seven compute
constexpr int DB_MAXK = 32;
constexpr int CB_QPW = 4;                    // cosine: queries per warp (a bin)
struct alignas(16) DbPoolHdr {   // 32 bytes; the first 16 are read with one LDS.128 for the threshold test
  double thr;
  int cnt, wid, worst, pad[3];
};
PIO_HD inline size_t db_smem_bytes(int kp, int topk) {
  return sizeof(double) * (size_t)kp * SB_QB + sizeof(float) * (size_t)DB_RINGS * DB_STAGES * DB_ROWS * (kp + 4) +
         (size_t)DB_RINGS * SB_QB * (sizeof(DbPoolHdr) + (sizeof(double) + sizeof(int)) * (size_t)topk);
}

// ---- score_cos_topk_batched_kernel: one long similar query, its vectors in shared memory ----
constexpr int SC_G = 8;   // query vectors scored per pass over a staged row
// query vectors [kp][nqp] + their norms (nqp = nqv rounded up to SC_G), the staged tile, one pool per warp, the nq query
// ids (all of them, valid or not)
PIO_HD inline size_t cos_batched_smem_bytes(int kp, int nqv, int nq, int topk) {
  const size_t nqp = (size_t)(nqv + SC_G - 1) / SC_G * SC_G;
  return sizeof(double) * ((size_t)kp * nqp + nqp) + sizeof(float) * (size_t)SB_THREADS * (kp + 4) +
         (sizeof(double) + sizeof(int)) * (size_t)(SB_THREADS / 32) * topk + sizeof(int) * (size_t)nq + 16;
}

// ---- score_cos_topk_multi_kernel: groups of SM_QG similar queries ----
constexpr int SM_QG = 8;    // queries per group = warps per CTA
constexpr int SM_NV = 40;   // query vectors per group held in shared memory
constexpr int SM_QIDS = 64; // query item ids per query held in shared memory (longer lists are read from global memory)
// query vectors [kp][SM_NV] + norms, the staged tile, the pools [SM_QG][topk], vector -> query, the query ids
PIO_HD inline size_t cos_multi_smem_bytes(int kp, int topk) {
  return sizeof(double) * ((size_t)kp * SM_NV + SM_NV) + sb_tile_bytes(kp) + (sizeof(double) + sizeof(int)) * (size_t)SM_QG * topk +
         sizeof(int) * (SM_NV + SM_QG * SM_QIDS) + 16;
}

// ---- score_listed_kernel: one white-listed query per CTA, scored over its list ----
constexpr int LS_THREADS = 256;
constexpr int LS_WARPS = LS_THREADS / 32;   // one pool, and one candidate list, per warp
PIO_HD inline size_t listed_smem_bytes(int topk) { return (sizeof(double) + sizeof(int)) * (size_t)LS_WARPS * topk; }

// ---- score_one_kernel: one query, one launch ----
constexpr int S1_THREADS = 256;
constexpr int S1_STAGES = 3;
constexpr int S1_MAXNV = 8;
PIO_HD inline size_t s1_smem_bytes(int kp, int nvp, int topk) {
  return sizeof(double) * ((size_t)kp * nvp + S1_MAXNV) + sizeof(float) * (size_t)S1_STAGES * S1_THREADS * (kp + 4) +
         (sizeof(double) + sizeof(int)) * (size_t)(S1_THREADS / 32) * topk + 128;
}

}  // namespace pio
