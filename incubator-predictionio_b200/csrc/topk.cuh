// topk.cuh -- top-k scoring over the item factor matrix (serving side of the hot path) and the
// multinomial NaiveBayes reductions of the classification template.
//
// What is scored (reference):
//   dot     : recommendProducts(WithFilter) -- <x_u, y_i> over all candidate items
//             (examples/scala-parallel-recommendation/blacklist-items/src/main/scala/ALSModel.scala:44-60)
//   cosine  : similarproduct predict -- sum_q cosine(y_q, y_i), score > 0 only
//             (examples/scala-parallel-similarproduct/multi-events-multi-algos/src/main/scala/ALSAlgorithm.scala:160-187,220-234)
//   top-k   : getTopN (:200-217); ties by the smaller item index
// Scores are accumulated in fp64 over the fp32 factors in index order, exactly like the reference's blas.ddot / cosine
// loops over Array[Double], so scores and rankings are bit-identical to the oracle -- and the compute bound of every
// kernel here is the fp64 pipe (one DFMA per query vector x item x feature), not HBM.
//
// Kernels, by call shape (the planner in score_plan.h picks, pio_als.cu launches; DESIGN.md 4.6):
//   score_one_kernel                 one query = one launch: lookup, scan, selection, result into mapped host memory
//   score_dot_blocked_kernel         batches of users   (rank <= 64, topk <= 32): two items x eight queries per thread
//   score_cos_blocked_kernel         batches of similar queries (same limits): bins of <= 4 queries / <= 8 vectors per warp
//   score_dot_topk_batched_kernel    first-generation batch kernels (one item per thread): rank 128, topk > 32, and
//   score_cos_topk_multi_kernel        2..16 users / long similar queries on the three-launch serving path
//   score_cos_topk_batched_kernel    one long similar query, its vectors in shared memory
//   score_cos_topk_kernel            fallback for single queries too large for that
//   score_listed_kernel              white-listed queries of a filtered batch: scored over their lists, not the matrix
//   topk_merge_kernel                merges the per-CTA / per-warp candidate lists of a query; multi-pass bounds (topk > 128)
// Block sizes, pool shapes and every kernel's dynamic shared memory (*_smem_bytes) are in topk_geometry.h.
// Pools: WarpPool (entries in shared memory, cooperative worst-entry search) and SortedPool (sorted in the registers of a
// warp: ballot-counted position + shuffle shift).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include "topk_geometry.h"

namespace pio {

__device__ __forceinline__ bool better(double s1, int i1, double s2, int i2) {
  return (s1 > s2) || (s1 == s2 && i1 < i2);
}

// order-preserving map double -> unsigned 64-bit (a < b  <=>  key(a) < key(b)); key 0 is below every score
__device__ __forceinline__ unsigned long long s1_key(double v) {
  v += 0.0;   // -0.0 -> +0.0: the two compare equal as doubles and must share a key
  const unsigned long long b = (unsigned long long)__double_as_longlong(v);
  return (b >> 63) ? ~b : (b | 0x8000000000000000ull);
}

// Multi-pass selection (topk > TK_MAXK): a pass only accepts candidates strictly worse than the last result of the
// previous pass.  bound.i == TK_NO_BOUND: accept everything (first pass); TK_EXHAUSTED: the previous pass ran out of
// candidates, accept nothing.
constexpr int TK_NO_BOUND = -2;
constexpr int TK_EXHAUSTED = -3;
__device__ __forceinline__ bool below_bound(const ScoreIdx& b, double s, int i) {
  return b.i == TK_NO_BOUND || (b.i >= 0 && better(b.s, b.i, s, i));
}

// Per-query filters of a batch call (pio_als_query_filter on the device).  Exclusion entries are 64-bit keys
// (query << 32 | item id), sorted over the whole call, so the list of a query is the ascending range
// ex[ex_ptr[q] .. ex_ptr[q + 1]); ids outside the item range and duplicates stay in the list and match nothing new.  A
// set row is one bit per item.  The batch kernels test a candidate only when it is about to enter a pool (it has passed
// the pool's threshold test): an excluded item never enters a pool, so thresholds are formed from allowed items only
// and the scan itself is the unfiltered one.
struct QueryFilterDev {
  const unsigned long long* ex = nullptr;
  const long long* ex_ptr = nullptr;   // [queries + 1]; nullptr: no exclusion lists
  const int* set_ix = nullptr;         // [queries] row of set_bits, or -1; nullptr: no sets
  const unsigned* set_bits = nullptr;  // [n_sets][set_words]
  int set_words = 0;
  int qbase = 0;                       // the launch's first query in the numbering of ex / ex_ptr / set_ix
};
// is item `ext` (>= 0) no candidate of query q (numbered inside the launch)?
__device__ __forceinline__ bool qf_drop(const QueryFilterDev& f, int q, int ext) {
  q += f.qbase;
  if (f.set_ix) {
    const int r = __ldg(f.set_ix + q);
    if (r >= 0 && ((__ldg(f.set_bits + (size_t)r * f.set_words + (ext >> 5)) >> (ext & 31)) & 1u)) return true;
  }
  if (f.ex_ptr) {
    const unsigned long long key = ((unsigned long long)(unsigned)q << 32) | (unsigned)ext;
    long long lo = __ldg(f.ex_ptr + q);
    const long long end = __ldg(f.ex_ptr + q + 1);
    long long hi = end;
    while (lo < hi) {
      const long long mid = (lo + hi) >> 1;
      if (__ldg(f.ex + mid) < key) lo = mid + 1;
      else hi = mid;
    }
    if (lo < end && __ldg(f.ex + lo) == key) return true;
  }
  return false;
}

// Block-wide selection: every thread holds TK_ITEMS candidates (score, index; index -1 = none).
// Extracts the best `topk` in order and writes them to out[0..topk).
__device__ __forceinline__ void block_select_topk(double (&sc)[TK_ITEMS], int (&ix)[TK_ITEMS], int topk,
                                                  ScoreIdx* out) {
  __shared__ double ws[TK_THREADS / 32];
  __shared__ int wi[TK_THREADS / 32];
  __shared__ int wowner[TK_THREADS / 32];
  __shared__ int s_owner;
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
  for (int t = 0; t < topk; ++t) {
    // local best
    double bs = 0.0;
    int bi = -1, bslot = -1;
#pragma unroll
    for (int j = 0; j < TK_ITEMS; ++j)
      if (ix[j] >= 0 && (bi < 0 || better(sc[j], ix[j], bs, bi))) { bs = sc[j]; bi = ix[j]; bslot = j; }
    double rs = bs;
    int ri = bi, ro = threadIdx.x;
#pragma unroll
    for (int d = 16; d > 0; d >>= 1) {
      const double os = __shfl_xor_sync(0xffffffffu, rs, d);
      const int oi = __shfl_xor_sync(0xffffffffu, ri, d);
      const int oo = __shfl_xor_sync(0xffffffffu, ro, d);
      if (oi >= 0 && (ri < 0 || better(os, oi, rs, ri))) { rs = os; ri = oi; ro = oo; }
    }
    if (lane == 0) { ws[w] = rs; wi[w] = ri; wowner[w] = ro; }
    __syncthreads();
    if (threadIdx.x == 0) {
      double fs = ws[0];
      int fi = wi[0], fo = wowner[0];
      for (int q = 1; q < TK_THREADS / 32; ++q)
        if (wi[q] >= 0 && (fi < 0 || better(ws[q], wi[q], fs, fi))) { fs = ws[q]; fi = wi[q]; fo = wowner[q]; }
      out[t].s = fs;
      out[t].i = fi;
      s_owner = fi >= 0 ? fo : -1;
    }
    __syncthreads();
    if (s_owner == (int)threadIdx.x && bslot >= 0) ix[bslot] = -1;
    __syncthreads();
  }
}

// ---- batched dot-product scoring -------------------------------------------------------------------------------
// grid: (GX persistent CTAs striding over 256-item tiles, query groups of SB_QB queries).  A tile of the item factor
// matrix is staged once (coalesced cp.async, padded rows -> conflict-free LDS.128) and scored against all SB_QB queries
// of the group from registers: the matrix is read n_queries / SB_QB times instead of n_queries times.  Each query
// keeps a top-k pool in shared memory for the whole scan; an item is offered to it only if it beats the pool's current
// worst entry (rare after the first tiles), under a per-query lock - no per-tile block-wide selection rounds.
// xq: [n_queries][kp] (zero padded), qvalid[q] == 0 -> no candidates.  cand: [n_queries][GX][topk], unsorted, i = -1 = empty.

__device__ __forceinline__ void sb_cp_async16(void* smem_dst, const void* gsrc) {
  const unsigned d = (unsigned)__cvta_generic_to_shared(smem_dst);
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16;\n" ::"r"(d), "l"(gsrc));
}

// A top-k pool owned by ONE warp (entries in shared memory, bookkeeping in warp-uniform registers): no lock, no atomics.
// All 32 lanes call; candidates are taken in lane order.  The worst entry is found cooperatively (each lane scans the
// entries lane, lane+32, ..., then a butterfly reduction), so an insertion costs ~100 cycles instead of a serial scan.
struct WarpPool {
  double thr;   // score of the worst entry (valid once cnt == topk)
  int wid;      // its external id
  int worst;    // its slot
  int cnt;
};
__device__ __forceinline__ void wpool_find_worst(WarpPool& wp, int topk, const double* ps, const int* pi) {
  const int lane = threadIdx.x & 31;
  double ws = 0.0;
  int wi = -1, wslot = -1;
  for (int t = lane; t < topk; t += 32) {
    const double s = ps[t];
    const int i = pi[t];
    if (wslot < 0 || better(ws, wi, s, i)) { ws = s; wi = i; wslot = t; }
  }
#pragma unroll
  for (int d = 16; d > 0; d >>= 1) {
    const double os = __shfl_xor_sync(0xffffffffu, ws, d);
    const int oi = __shfl_xor_sync(0xffffffffu, wi, d);
    const int oslot = __shfl_xor_sync(0xffffffffu, wslot, d);
    if (oslot >= 0 && (wslot < 0 || better(ws, wi, os, oi))) { ws = os; wi = oi; wslot = oslot; }
  }
  wp.thr = ws;
  wp.wid = wi;
  wp.worst = wslot;
  __syncwarp();   // the entries have been read by every lane before lane 0 overwrites one (the shuffles above already
                  // converge the warp; this makes the ordering explicit for the memory model and for racecheck)
}
__device__ __forceinline__ void wpool_offer(WarpPool& wp, bool want, double s, int ext, int topk, double* ps, int* pi) {
  const int lane = threadIdx.x & 31;
  want = want && (wp.cnt < topk || s >= wp.thr);
  unsigned m = __ballot_sync(0xffffffffu, want);
  while (m) {
    const int leader = __ffs(m) - 1;
    m &= m - 1;
    const double cs = __shfl_sync(0xffffffffu, s, leader);
    const int ce = __shfl_sync(0xffffffffu, ext, leader);
    if (wp.cnt < topk) {
      if (lane == 0) { ps[wp.cnt] = cs; pi[wp.cnt] = ce; }
      ++wp.cnt;
      __syncwarp();
      if (wp.cnt == topk) wpool_find_worst(wp, topk, ps, pi);
    } else if (better(cs, ce, wp.thr, wp.wid)) {
      if (lane == 0) { ps[wp.worst] = cs; pi[wp.worst] = ce; }
      __syncwarp();
      wpool_find_worst(wp, topk, ps, pi);
    }
  }
}

template <bool FILT>
__global__ void __launch_bounds__(SB_THREADS, 2)
score_dot_topk_batched_kernel(const float* __restrict__ Y, int n_items, int kp,
                              const float* __restrict__ xq, const uint8_t* __restrict__ qvalid, int n_queries,
                              const int* __restrict__ cand_ext, const uint8_t* __restrict__ mask,
                              const double* __restrict__ weight, const ScoreIdx* __restrict__ bound,
                              int topk, ScoreIdx* __restrict__ cand, const QueryFilterDev flt) {
  extern __shared__ __align__(16) unsigned char sb_smem[];
  const int row = kp + 4;                                         // floats per staged row (16-byte skew per row)
  double* xd = reinterpret_cast<double*>(sb_smem);                // [kp][SB_QB]
  float* tile = reinterpret_cast<float*>(xd + (size_t)kp * SB_QB);   // [SB_THREADS][row]; reused for the score exchange
  const size_t tile_bytes = sb_tile_bytes(kp);
  double* hs = reinterpret_cast<double*>(reinterpret_cast<unsigned char*>(tile) + tile_bytes);   // [SB_QB][topk]
  int* hi = reinterpret_cast<int*>(hs + (size_t)SB_QB * topk);    // [SB_QB][topk]
  double* scs = reinterpret_cast<double*>(tile);                  // [SB_QB][SB_THREADS] scores of the current tile
  int* sext = reinterpret_cast<int*>(scs + (size_t)SB_QB * SB_THREADS);   // [SB_THREADS] their external ids
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int q0 = blockIdx.y * SB_QB;
  for (int o = tid; o < kp * SB_QB; o += SB_THREADS) {
    const int t = o / SB_QB, q = o % SB_QB;
    xd[o] = (q0 + q < n_queries) ? (double)xq[(size_t)(q0 + q) * kp + t] : 0.0;
  }
  // warp w owns the pools of queries w*QPW .. w*QPW+QPW-1 of the group
  constexpr int QPW = SB_QB / (SB_THREADS / 32);
  WarpPool wp[QPW];
  ScoreIdx bnd[QPW];
#pragma unroll
  for (int j = 0; j < QPW; ++j) {
    wp[j].thr = 0.0; wp[j].wid = -1; wp[j].worst = 0; wp[j].cnt = 0;
    const int q = q0 + warp * QPW + j;
    bnd[j].s = 0.0;
    bnd[j].i = TK_NO_BOUND;
    if (bound && q < n_queries) bnd[j] = bound[q];
  }
  unsigned qmask = 0;   // queries of this group that take candidates
  for (int q = 0; q < SB_QB; ++q)
    if (q0 + q < n_queries && qvalid[q0 + q]) qmask |= 1u << q;
  const int ntiles = (n_items + SB_THREADS - 1) / SB_THREADS;
  const int f4row = kp / 4;
  for (int tl = blockIdx.x; tl < ntiles; tl += gridDim.x) {
    const int base = tl * SB_THREADS;
    __syncthreads();   // the previous tile has been consumed (and xd / pools are initialised)
    for (int o = tid; o < SB_THREADS * f4row; o += SB_THREADS) {
      const int r = o / f4row, c4 = o % f4row;
      float* d = tile + (size_t)r * row + c4 * 4;
      if (base + r < n_items) sb_cp_async16(d, Y + (size_t)(base + r) * kp + c4 * 4);
      else *reinterpret_cast<float4*>(d) = make_float4(0.f, 0.f, 0.f, 0.f);
    }
    asm volatile("cp.async.commit_group;\n" ::);
    asm volatile("cp.async.wait_group 0;\n" ::);
    __syncthreads();
    const int i = base + tid;
    int ext = (i < n_items) ? cand_ext[i] : -1;    // external id, -1 = owns no factor
    if (ext >= 0 && mask && mask[ext]) ext = -1;
    double acc[SB_QB];
#pragma unroll
    for (int q = 0; q < SB_QB; ++q) acc[q] = 0.0;
    if (ext >= 0 && qmask) {
      const float4* yrow = reinterpret_cast<const float4*>(tile + (size_t)tid * row);
      for (int c4 = 0; c4 < f4row; ++c4) {
        const float4 y4 = yrow[c4];
        const float ye[4] = {y4.x, y4.y, y4.z, y4.w};
#pragma unroll
        for (int e = 0; e < 4; ++e) {
          const double yd = (double)ye[e];
          const double2* xr = reinterpret_cast<const double2*>(xd + (size_t)(c4 * 4 + e) * SB_QB);
#pragma unroll
          for (int q = 0; q < SB_QB; q += 2) {
            const double2 x2 = xr[q / 2];
            acc[q] = fma(x2.x, yd, acc[q]);       // index order t = 0..k-1, like blas.ddot over Array[Double]
            acc[q + 1] = fma(x2.y, yd, acc[q + 1]);
          }
        }
      }
    }
    if (weight && ext >= 0) {   // per-item score weight (ecommerce adjust-score): adjustedScore = s * weights(i)
      const double w = weight[ext];
#pragma unroll
      for (int q = 0; q < SB_QB; ++q) acc[q] = acc[q] * w;
    }
    // exchange: every thread publishes its SB_QB scores, then each warp feeds the pools it owns (no locks)
    __syncthreads();   // the staged rows are dead
#pragma unroll
    for (int q = 0; q < SB_QB; ++q) scs[q * SB_THREADS + tid] = acc[q];
    sext[tid] = ext;
    __syncthreads();
#pragma unroll
    for (int j = 0; j < QPW; ++j) {
      const int q = warp * QPW + j;
      if ((qmask >> q) & 1u) {
        for (int it = lane; it < SB_THREADS; it += 32) {
          const int e = sext[it];
          const double sv = scs[q * SB_THREADS + it];
          bool want = e >= 0 && below_bound(bnd[j], sv, e);
          if (FILT) want = want && (wp[j].cnt < topk || sv >= wp[j].thr) && !qf_drop(flt, q0 + q, e);
          wpool_offer(wp[j], want, sv, e, topk, hs + (size_t)q * topk, hi + (size_t)q * topk);
        }
      }
    }
  }
  __syncwarp();
#pragma unroll
  for (int j = 0; j < QPW; ++j) {
    const int q = warp * QPW + j;
    if (q0 + q < n_queries) {
      for (int t = lane; t < topk; t += 32) {
        ScoreIdx e;
        e.s = t < wp[j].cnt ? hs[(size_t)q * topk + t] : 0.0;
        e.i = t < wp[j].cnt ? hi[(size_t)q * topk + t] : -1;
        cand[((size_t)(q0 + q) * gridDim.x + blockIdx.x) * topk + t] = e;
      }
    }
  }
}

// A top-k pool kept SORTED in the registers of one warp: entry g (0 = best) lives in lane g % 32, slot g / 32.  An
// insertion is one position count (ballots) and one shift (shuffles) -- no search for the worst entry; the threshold is
// entry topk - 1.  Warp-uniform: cnt.  All 32 lanes call offer(); candidates are taken in lane order.
struct SortedPool {
  static constexpr int SLOTS = TK_MAXK / 32;
  double s[SLOTS];
  int i[SLOTS];
  int cnt;
  double thr;   // score and id of entry topk - 1 once cnt == topk
  int tid_;
  __device__ __forceinline__ void init() {
#pragma unroll
    for (int q = 0; q < SLOTS; ++q) { s[q] = 0.0; i[q] = -1; }
    cnt = 0; thr = 0.0; tid_ = -1;
  }
  __device__ __forceinline__ void insert(double cs, int ce, int topk) {
    const int lane = threadIdx.x & 31;
    const int nslot = (topk + 31) >> 5;
    int p = 0;   // entries better than the candidate = its position
#pragma unroll
    for (int q = 0; q < SLOTS; ++q)
      if (q < nslot) p += __popc(__ballot_sync(0xffffffffu, q * 32 + lane < cnt && better(s[q], i[q], cs, ce)));
    double carry_s = 0.0;   // lane 31 of the previous slot (moves into lane 0 of this one)
    int carry_i = -1;
#pragma unroll
    for (int q = 0; q < SLOTS; ++q)
      if (q < nslot) {
        double us = __shfl_up_sync(0xffffffffu, s[q], 1);
        int ui = __shfl_up_sync(0xffffffffu, i[q], 1);
        const double last_s = __shfl_sync(0xffffffffu, s[q], 31);
        const int last_i = __shfl_sync(0xffffffffu, i[q], 31);
        if (lane == 0) { us = carry_s; ui = carry_i; }
        const int g = q * 32 + lane;
        if (g == p) { s[q] = cs; i[q] = ce; }
        else if (g > p) { s[q] = us; i[q] = ui; }
        carry_s = last_s;
        carry_i = last_i;
      }
    if (cnt < topk) ++cnt;
    if (cnt == topk) {
      const int q = (topk - 1) >> 5, l = (topk - 1) & 31;
      double ts = 0.0;
      int ti = -1;
#pragma unroll
      for (int qq = 0; qq < SLOTS; ++qq)
        if (qq == q) { ts = s[qq]; ti = i[qq]; }
      thr = __shfl_sync(0xffffffffu, ts, l);
      tid_ = __shfl_sync(0xffffffffu, ti, l);
    }
  }
  // empty pool: the 32 candidates of a step are sorted by a bitonic network (15 exchange stages) instead of being
  // inserted one after the other; lane g ends up with the g-th best, which IS slot 0 of the pool
  __device__ __forceinline__ void fill_sorted(bool want, double sc, int ext, int topk) {
    const int lane = threadIdx.x & 31;
    double ms = want ? sc : 0.0;
    int mi = want ? ext : -1;
#pragma unroll
    for (int kk = 2; kk <= 32; kk <<= 1) {
#pragma unroll
      for (int j = kk >> 1; j > 0; j >>= 1) {
        const double os = __shfl_xor_sync(0xffffffffu, ms, j);
        const int oi = __shfl_xor_sync(0xffffffffu, mi, j);
        const bool mine_better = mi >= 0 && (oi < 0 || better(ms, mi, os, oi));
        const bool want_better = ((lane & j) == 0) == ((lane & kk) == 0);   // this lane keeps the better one of the pair
        if (mine_better != want_better) { ms = os; mi = oi; }
      }
    }
    const int nvalid = __popc(__ballot_sync(0xffffffffu, want));
    s[0] = ms;
    i[0] = mi;
    cnt = nvalid < topk ? nvalid : topk;
    if (cnt == topk) {      // only possible for topk <= 32: the threshold is entry topk - 1 of slot 0
      thr = __shfl_sync(0xffffffffu, ms, (topk - 1) & 31);
      tid_ = __shfl_sync(0xffffffffu, mi, (topk - 1) & 31);
    }
  }
  __device__ __forceinline__ void offer(bool want, double sc, int ext, int topk) {
    want = want && (cnt < topk || sc >= thr);
    unsigned m = __ballot_sync(0xffffffffu, want);
    if (cnt == 0 && (m & (m - 1))) {   // nothing pooled yet and more than one candidate
      fill_sorted(want, sc, ext, topk);
      return;
    }
    while (m) {
      const int leader = __ffs(m) - 1;
      m &= m - 1;
      const double cs = __shfl_sync(0xffffffffu, sc, leader);
      const int ce = __shfl_sync(0xffffffffu, ext, leader);
      if (cnt < topk || better(cs, ce, thr, tid_)) insert(cs, ce, topk);
    }
  }
  // entries to shared memory ([topk] each), best first
  __device__ __forceinline__ void dump(int topk, double* ps, int* pi) const {
    const int lane = threadIdx.x & 31;
#pragma unroll
    for (int q = 0; q < SLOTS; ++q) {
      const int g = q * 32 + lane;
      if (g < cnt) { ps[g] = s[q]; pi[g] = i[q]; }
    }
  }
};

// ---- blocked dot-product scoring: two items x eight queries per thread, sixteen warps per SM ------------------------
// The batched kernel above issues one broadcast LDS.128 of query values per two DFMAs: the shared-memory pipe and the
// fp64 pipe saturate together.  Here every lane scores TWO items against DB_QW = 8 queries, so one LDS.128 feeds four
// DFMAs.  A CTA is eight independent "rings" of two warps: the warps of a ring share 64 staged rows per step (each copies
// half with cp.async; two named barriers of 64 threads per step -- never a CTA barrier in the scan; a ring waits for its
// own rows while the other seven compute) and split the 16 queries of the group between them; every warp owns the top-k
// pools of its eight queries (entries and bookkeeping in shared memory; almost every score fails the threshold test, the
// insertion is an out-of-line call).  Measured on the way: one warp per scheduler with 2 x 16 accumulators keeps the fp64
// pipe 31 % busy; rings of four warps (4 queries each) convert every row four times and the conversion pipe (F2F: 15.7
// lanes/clk/SM) becomes co-critical (fp64 45 %, XU 44 %).  Same arithmetic and order as above -> bit-identical results.
// For kp <= 64 and topk <= DB_MAXK; cand: [n_queries][gridDim.x * DB_RINGS][topk], unsorted, i = -1 = empty.

// The rare path of the scan (a score passed the threshold test): NOT inlined -- unrolled copies of the pool insertion
// between the threshold tests of a step are tens of KB of code on the hot path (ncu on a first version: "no
// instruction" 2.5 stalls per issued instruction).
__device__ __noinline__ void db_insert(DbPoolHdr* hd, double* ps, int* pi, unsigned long long* cthr, bool w0, double s0,
                                       int e0, bool w1, double s1, int e1, int topk) {
  // the pool is kept sorted in shared memory (topk <= 32: entry g belongs to lane g); an insertion happens in registers
  // (SortedPool: ballot-counted position + shuffle shift) between one load and one store of the 32 entries
  const int lane = threadIdx.x & 31;
  SortedPool sp;
  sp.init();
  sp.cnt = hd->cnt;
  sp.thr = hd->thr;
  sp.tid_ = hd->wid;
  if (lane < sp.cnt) { sp.s[0] = ps[lane]; sp.i[0] = pi[lane]; }
  sp.offer(w0, s0, e0, topk);
  sp.offer(w1, s1, e1, topk);
  if (lane < sp.cnt) { ps[lane] = sp.s[0]; pi[lane] = sp.i[0]; }
  __syncwarp();   // every lane has read the header before lane 0 rewrites it
  if (lane == 0) {
    hd->thr = sp.thr; hd->cnt = sp.cnt; hd->wid = sp.tid_;
    if (sp.cnt == topk) atomicMax(cthr, s1_key(sp.thr));   // the smallest entry of a FULL pool bounds the query's topk-th score
  }
  __syncwarp();
}

// the same with the query's filter: a lane's candidate that its query excludes is withdrawn before the insertion
__device__ __noinline__ void dbf_insert(DbPoolHdr* hd, double* ps, int* pi, unsigned long long* cthr, bool w0, double s0,
                                        int e0, bool w1, double s1, int e1, int topk, const QueryFilterDev& flt, int q) {
  if (w0 && qf_drop(flt, q, e0)) w0 = false;
  if (w1 && qf_drop(flt, q, e1)) w1 = false;
  if (!__any_sync(0xffffffffu, w0 || w1)) return;
  db_insert(hd, ps, pi, cthr, w0, s0, e0, w1, s1, e1, topk);
}

template <int KP, bool FILT>
__global__ void __launch_bounds__(32 * DB_WARPS, 1)
score_dot_blocked_kernel(const float* __restrict__ Y, int n_items, const float* __restrict__ xq,
                         const uint8_t* __restrict__ qvalid, int n_queries, const int* __restrict__ cand_ext,
                         const uint8_t* __restrict__ mask, const double* __restrict__ weight, int topk,
                         ScoreIdx* __restrict__ cand, const QueryFilterDev flt) {
  constexpr int ROW = KP + 4, F4 = KP / 4;
  constexpr int RPI = 32 / F4;                 // rows per warp-wide copy instruction (512 contiguous bytes)
  constexpr int CPW = DB_ROWS / RPI / DB_WPR;  // copy instructions per warp and step
  extern __shared__ __align__(16) unsigned char db_smem[];
  double* xd = reinterpret_cast<double*>(db_smem);                                   // [KP][SB_QB]
  float* rings = reinterpret_cast<float*>(xd + (size_t)KP * SB_QB);                  // [DB_RINGS][DB_STAGES][DB_ROWS][ROW]
  DbPoolHdr* hdrs = reinterpret_cast<DbPoolHdr*>(rings + (size_t)DB_RINGS * DB_STAGES * DB_ROWS * ROW);   // [DB_RINGS][SB_QB]
  double* pss = reinterpret_cast<double*>(hdrs + DB_RINGS * SB_QB);                  // [DB_RINGS][SB_QB][topk]
  int* pis = reinterpret_cast<int*>(pss + (size_t)DB_RINGS * SB_QB * topk);          // [DB_RINGS][SB_QB][topk]
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int rg = warp / DB_WPR, sub = warp % DB_WPR;      // ring, and which four queries of the group
  const int q0 = blockIdx.y * SB_QB;
  for (int o = tid; o < KP * SB_QB; o += 32 * DB_WARPS) {
    const int t = o / SB_QB, q = o % SB_QB;
    xd[o] = (q0 + q < n_queries) ? (double)xq[(size_t)(q0 + q) * KP + t] : 0.0;
  }
  for (int o = tid; o < DB_RINGS * SB_QB; o += 32 * DB_WARPS) {
    hdrs[o].thr = 0.0; hdrs[o].cnt = 0; hdrs[o].wid = -1; hdrs[o].worst = 0;
  }
  // per query: key of the best threshold any ring of this CTA has reached -- scores strictly below it are dropped before
  // they are offered to this ring's pool (eight pools per query would otherwise each warm up on an eighth of the items)
  __shared__ unsigned long long cthr[SB_QB];
  if (tid < SB_QB) cthr[tid] = 0ull;
  unsigned qmask = 0;   // my queries that take candidates
  for (int q = 0; q < DB_QW; ++q)
    if (q0 + sub * DB_QW + q < n_queries && qvalid[q0 + sub * DB_QW + q]) qmask |= 1u << q;
  __syncthreads();
  float* ring = rings + (size_t)rg * DB_STAGES * DB_ROWS * ROW;
  DbPoolHdr* hdr = hdrs + rg * SB_QB + sub * DB_QW;
  double* ps = pss + ((size_t)rg * SB_QB + sub * DB_QW) * topk;
  int* pi = pis + ((size_t)rg * SB_QB + sub * DB_QW) * topk;
  const double* xw = xd + sub * DB_QW;
  auto ring_bar = [&]() { asm volatile("bar.sync %0, %1;" ::"r"(1 + rg), "r"(32 * DB_WPR) : "memory"); };
  const int nsteps = (n_items + DB_RINGS * DB_ROWS - 1) / (DB_RINGS * DB_ROWS);
  const int my_steps = (int)blockIdx.x < nsteps ? (nsteps - 1 - (int)blockIdx.x) / (int)gridDim.x + 1 : 0;
  auto base_of = [&](int j) { return (((int)blockIdx.x + j * (int)gridDim.x) * DB_RINGS + rg) * DB_ROWS; };
  auto fetch = [&](int j) {   // this warp's quarter of the ring's step j
    if (j < my_steps) {
      const int base = base_of(j);
      const int r0 = sub * CPW * RPI + lane / F4;
      float* dst = ring + (size_t)(j % DB_STAGES) * DB_ROWS * ROW + (size_t)r0 * ROW + (lane % F4) * 4;
      const float* src = Y + (size_t)(base + r0) * KP + (lane % F4) * 4;
      if (base + DB_ROWS <= n_items) {
#pragma unroll
        for (int m = 0; m < CPW; ++m) sb_cp_async16(dst + (size_t)m * RPI * ROW, src + (size_t)m * RPI * KP);
      } else {
#pragma unroll
        for (int m = 0; m < CPW; ++m)
          if (base + r0 + m * RPI < n_items) sb_cp_async16(dst + (size_t)m * RPI * ROW, src + (size_t)m * RPI * KP);
      }
    }
    asm volatile("cp.async.commit_group;\n" ::);
  };
  if (DB_STAGES > 1) fetch(0);
  int ext_n[2] = {-1, -1};
  if (my_steps > 0) {
#pragma unroll
    for (int u = 0; u < 2; ++u) {
      const int i = base_of(0) + u * 32 + lane;
      ext_n[u] = i < n_items ? __ldg(cand_ext + i) : -1;
    }
  }
  for (int j = 0; j < my_steps; ++j) {
    int ext[2] = {ext_n[0], ext_n[1]};
    if (j + 1 < my_steps) {
#pragma unroll
      for (int u = 0; u < 2; ++u) {
        const int i = base_of(j + 1) + u * 32 + lane;
        ext_n[u] = i < n_items ? __ldg(cand_ext + i) : -1;
      }
    }
#pragma unroll
    for (int u = 0; u < 2; ++u)
      if (ext[u] >= 0 && mask && mask[ext[u]]) ext[u] = -1;
    ring_bar();                // the slot about to be refilled has been read by every warp of the ring
    fetch(j + DB_STAGES - 1);
    asm volatile("cp.async.wait_group %0;\n" ::"n"(DB_STAGES - 1));
    ring_bar();                // step j has landed for the whole ring
    double acc[2][DB_QW];
#pragma unroll
    for (int u = 0; u < 2; ++u)
#pragma unroll
      for (int q = 0; q < DB_QW; ++q) acc[u][q] = 0.0;
    if (qmask) {
      const float4* r0 = reinterpret_cast<const float4*>(ring + ((size_t)(j % DB_STAGES) * DB_ROWS + lane) * ROW);
      const float4* r1 = reinterpret_cast<const float4*>(ring + ((size_t)(j % DB_STAGES) * DB_ROWS + 32 + lane) * ROW);
#pragma unroll 2
      for (int c4 = 0; c4 < F4; ++c4) {
        const float4 a4 = r0[c4], b4 = r1[c4];
        const double ya[4] = {(double)a4.x, (double)a4.y, (double)a4.z, (double)a4.w};
        const double yb[4] = {(double)b4.x, (double)b4.y, (double)b4.z, (double)b4.w};
#pragma unroll
        for (int e = 0; e < 4; ++e) {
          const double2* xr = reinterpret_cast<const double2*>(xw + (size_t)(c4 * 4 + e) * SB_QB);
#pragma unroll
          for (int q = 0; q < DB_QW; q += 2) {
            const double2 x2 = xr[q / 2];
            acc[0][q] = fma(x2.x, ya[e], acc[0][q]);          // index order t = 0..k-1, like blas.ddot over Array[Double]
            acc[0][q + 1] = fma(x2.y, ya[e], acc[0][q + 1]);
            acc[1][q] = fma(x2.x, yb[e], acc[1][q]);
            acc[1][q + 1] = fma(x2.y, yb[e], acc[1][q + 1]);
          }
        }
      }
    }
    if (weight) {   // per-item score weight (ecommerce adjust-score): adjustedScore = s * weights(i)
#pragma unroll
      for (int u = 0; u < 2; ++u)
        if (ext[u] >= 0) {
          const double w = weight[ext[u]];
#pragma unroll
          for (int q = 0; q < DB_QW; ++q) acc[u][q] = acc[u][q] * w;
        }
    }
#pragma unroll
    for (int q = 0; q < DB_QW; ++q) {
      if (!((qmask >> q) & 1u)) continue;
      const int4 h4 = *reinterpret_cast<const int4*>(&hdr[q]);       // thr (8 bytes), cnt, wid
      const double thr = __hiloint2double(h4.y, h4.x);
      const int cnt = h4.z;
      const unsigned long long ck = *reinterpret_cast<volatile unsigned long long*>(&cthr[sub * DB_QW + q]);
      const bool w0 = ext[0] >= 0 && (cnt < topk || acc[0][q] >= thr) && s1_key(acc[0][q]) >= ck;
      const bool w1 = ext[1] >= 0 && (cnt < topk || acc[1][q] >= thr) && s1_key(acc[1][q]) >= ck;
      if (!__any_sync(0xffffffffu, w0 || w1)) continue;
      if (FILT)
        dbf_insert(&hdr[q], ps + (size_t)q * topk, pi + (size_t)q * topk, &cthr[sub * DB_QW + q], w0, acc[0][q], ext[0], w1,
                   acc[1][q], ext[1], topk, flt, q0 + sub * DB_QW + q);
      else
        db_insert(&hdr[q], ps + (size_t)q * topk, pi + (size_t)q * topk, &cthr[sub * DB_QW + q], w0, acc[0][q], ext[0], w1,
                  acc[1][q], ext[1], topk);
    }
  }
  asm volatile("cp.async.wait_group 0;\n" ::);
  __syncwarp();
#pragma unroll 1
  for (int q = 0; q < DB_QW; ++q) {
    const int qq = q0 + sub * DB_QW + q;
    if (qq >= n_queries) break;
    const int cnt = hdr[q].cnt;
    ScoreIdx* out = cand + (((size_t)qq * gridDim.x + blockIdx.x) * DB_RINGS + rg) * topk;
    for (int t = lane; t < topk; t += 32) {
      ScoreIdx e;
      e.s = t < cnt ? ps[(size_t)q * topk + t] : 0.0;
      e.i = t < cnt ? pi[(size_t)q * topk + t] : -1;
      out[t] = e;
    }
  }
}

// ---- blocked cosine scoring (similarproduct batches): the same rings, eight query VECTORS per warp ------------------
// The host packs consecutive queries into bins of <= CB_QPW queries and <= DB_QW query vectors (a query never spans two
// bins); a warp scores two items per lane against the vectors of its bin, turns them into per-query cosine sums (in
// query-vector order, fp64 -- bit-identical to the kernels below) and keeps the pools of its queries.  blockIdx.y = a pair
// of bins (the two warps of every ring).  bin_q0 / bin_v0: first query / first vector of every bin (+ one end entry);
// qf: the query vectors [n_vec][KP]; vq: global query of every vector; qid_ptr / qid: the id list of every query (all
// of them are excluded from its results unless keep_query).  cand: [n_queries][gridDim.x * DB_RINGS][topk].

__device__ __noinline__ void cb_insert(DbPoolHdr* hd, double* ps, int* pi, unsigned long long* cthr, bool w0, double s0,
                                       int e0, bool w1, double s1, int e1, int topk, const int* __restrict__ qid, int nid) {
  // (rare path) the query's own items are no candidates (ALSAlgorithm.scala:243-245 `!queryList.contains(i)`); nid = 0
  // when they are kept
  for (int t = 0; t < nid; ++t) {
    const int id = __ldg(qid + t);
    if (id == e0) w0 = false;
    if (id == e1) w1 = false;
  }
  if (!__any_sync(0xffffffffu, w0 || w1)) return;
  db_insert(hd, ps, pi, cthr, w0, s0, e0, w1, s1, e1, topk);
}

__device__ __noinline__ void cbf_insert(DbPoolHdr* hd, double* ps, int* pi, unsigned long long* cthr, bool w0, double s0,
                                        int e0, bool w1, double s1, int e1, int topk, const int* __restrict__ qid, int nid,
                                        const QueryFilterDev& flt, int q) {
  if (w0 && qf_drop(flt, q, e0)) w0 = false;
  if (w1 && qf_drop(flt, q, e1)) w1 = false;
  if (!__any_sync(0xffffffffu, w0 || w1)) return;
  cb_insert(hd, ps, pi, cthr, w0, s0, e0, w1, s1, e1, topk, qid, nid);
}

template <int KP, bool FILT>
__global__ void __launch_bounds__(32 * DB_WARPS, 1)
score_cos_blocked_kernel(const float* __restrict__ Y, int n_items, int k, const float* __restrict__ qf,
                         const int* __restrict__ bin_q0, const int* __restrict__ bin_v0, int n_bins,
                         const int* __restrict__ vq, const long long* __restrict__ qid_ptr, const int* __restrict__ qid,
                         const int* __restrict__ cand_ext, const uint8_t* __restrict__ mask,
                         const double* __restrict__ weight, int keep_query, int topk, ScoreIdx* __restrict__ cand,
                         const QueryFilterDev flt) {
  constexpr int ROW = KP + 4, F4 = KP / 4;
  constexpr int RPI = 32 / F4;
  constexpr int CPW = DB_ROWS / RPI / DB_WPR;
  constexpr int NV = DB_QW;                    // vectors per warp
  constexpr int GQ = DB_WPR * CB_QPW;          // pools per ring
  extern __shared__ __align__(16) unsigned char db_smem[];
  double* xd = reinterpret_cast<double*>(db_smem);                                   // [KP][DB_WPR * NV]
  float* rings = reinterpret_cast<float*>(xd + (size_t)KP * SB_QB);                  // [DB_RINGS][DB_STAGES][DB_ROWS][ROW]
  DbPoolHdr* hdrs = reinterpret_cast<DbPoolHdr*>(rings + (size_t)DB_RINGS * DB_STAGES * DB_ROWS * ROW);   // [DB_RINGS][GQ]
  double* pss = reinterpret_cast<double*>(hdrs + DB_RINGS * SB_QB);                  // [DB_RINGS][GQ][topk]
  int* pis = reinterpret_cast<int*>(pss + (size_t)DB_RINGS * SB_QB * topk);
  __shared__ double s1[DB_WPR * NV];
  __shared__ int svq[DB_WPR * NV];             // local query (0 .. CB_QPW - 1) of every vector
  __shared__ unsigned long long cthr[GQ];
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int rg = warp / DB_WPR, sub = warp % DB_WPR;
  const int bin = blockIdx.y * DB_WPR + sub;
  const bool have_bin = bin < n_bins;
  const int bq0 = have_bin ? bin_q0[bin] : 0, nqw = have_bin ? bin_q0[bin + 1] - bq0 : 0;
  const int bv0 = have_bin ? bin_v0[bin] : 0, nvw = have_bin ? bin_v0[bin + 1] - bv0 : 0;
  static_assert(DB_WPR * NV == SB_QB, "xd is laid out [KP][SB_QB]");
  for (int o = tid; o < KP * SB_QB; o += 32 * DB_WARPS) {
    const int c = o / SB_QB, col = o % SB_QB, sb = col / NV, v = col % NV;
    const int b = blockIdx.y * DB_WPR + sb;
    double x = 0.0;
    if (b < n_bins) {
      const int v0 = bin_v0[b];
      if (v < bin_v0[b + 1] - v0) x = (double)qf[(size_t)(v0 + v) * KP + c];
    }
    xd[o] = x;
  }
  if (tid < SB_QB) {
    const int sb = tid / NV, v = tid % NV, b = blockIdx.y * DB_WPR + sb;
    double n1 = 0.0;
    int lq = 0;
    if (b < n_bins) {
      const int v0 = bin_v0[b];
      if (v < bin_v0[b + 1] - v0) {
        for (int c = 0; c < k; ++c) {
          const double a = (double)qf[(size_t)(v0 + v) * KP + c];
          n1 += a * a;
        }
        lq = vq[v0 + v] - bin_q0[b];
      }
    }
    s1[tid] = sqrt(n1);
    svq[tid] = lq;
  }
  for (int o = tid; o < DB_RINGS * GQ; o += 32 * DB_WARPS) {
    hdrs[o].thr = 0.0; hdrs[o].cnt = 0; hdrs[o].wid = -1; hdrs[o].worst = 0;
  }
  if (tid < GQ) cthr[tid] = 0ull;
  __syncthreads();
  float* ring = rings + (size_t)rg * DB_STAGES * DB_ROWS * ROW;
  DbPoolHdr* hdr = hdrs + rg * GQ + sub * CB_QPW;
  double* ps = pss + ((size_t)rg * GQ + sub * CB_QPW) * topk;
  int* pi = pis + ((size_t)rg * GQ + sub * CB_QPW) * topk;
  const double* xw = xd + sub * NV;
  double s1r[NV];
  int vqr[NV];
#pragma unroll
  for (int v = 0; v < NV; ++v) { s1r[v] = s1[sub * NV + v]; vqr[v] = svq[sub * NV + v]; }
  const int* qid_of[CB_QPW];
  int nid_of[CB_QPW];
#pragma unroll
  for (int q = 0; q < CB_QPW; ++q) {
    qid_of[q] = qid;
    nid_of[q] = 0;
    if (q < nqw && !keep_query) {
      qid_of[q] = qid + qid_ptr[bq0 + q];
      nid_of[q] = (int)(qid_ptr[bq0 + q + 1] - qid_ptr[bq0 + q]);
    }
  }
  auto ring_bar = [&]() { asm volatile("bar.sync %0, %1;" ::"r"(1 + rg), "r"(32 * DB_WPR) : "memory"); };
  const int nsteps = (n_items + DB_RINGS * DB_ROWS - 1) / (DB_RINGS * DB_ROWS);
  const int my_steps = (int)blockIdx.x < nsteps ? (nsteps - 1 - (int)blockIdx.x) / (int)gridDim.x + 1 : 0;
  auto base_of = [&](int j) { return (((int)blockIdx.x + j * (int)gridDim.x) * DB_RINGS + rg) * DB_ROWS; };
  auto fetch = [&](int j) {
    if (j < my_steps) {
      const int base = base_of(j);
      const int r0 = sub * CPW * RPI + lane / F4;
      float* dst = ring + (size_t)(j % DB_STAGES) * DB_ROWS * ROW + (size_t)r0 * ROW + (lane % F4) * 4;
      const float* src = Y + (size_t)(base + r0) * KP + (lane % F4) * 4;
      if (base + DB_ROWS <= n_items) {
#pragma unroll
        for (int m = 0; m < CPW; ++m) sb_cp_async16(dst + (size_t)m * RPI * ROW, src + (size_t)m * RPI * KP);
      } else {
#pragma unroll
        for (int m = 0; m < CPW; ++m)
          if (base + r0 + m * RPI < n_items) sb_cp_async16(dst + (size_t)m * RPI * ROW, src + (size_t)m * RPI * KP);
      }
    }
    asm volatile("cp.async.commit_group;\n" ::);
  };
  if (DB_STAGES > 1) fetch(0);
  int ext_n[2] = {-1, -1};
  if (my_steps > 0) {
#pragma unroll
    for (int u = 0; u < 2; ++u) {
      const int i = base_of(0) + u * 32 + lane;
      ext_n[u] = i < n_items ? __ldg(cand_ext + i) : -1;
    }
  }
  for (int j = 0; j < my_steps; ++j) {
    int ext[2] = {ext_n[0], ext_n[1]};
    if (j + 1 < my_steps) {
#pragma unroll
      for (int u = 0; u < 2; ++u) {
        const int i = base_of(j + 1) + u * 32 + lane;
        ext_n[u] = i < n_items ? __ldg(cand_ext + i) : -1;
      }
    }
#pragma unroll
    for (int u = 0; u < 2; ++u)
      if (ext[u] >= 0 && mask && mask[ext[u]]) ext[u] = -1;
    ring_bar();
    fetch(j + DB_STAGES - 1);
    asm volatile("cp.async.wait_group %0;\n" ::"n"(DB_STAGES - 1));
    ring_bar();
    if (nvw == 0) continue;     // (uniform per warp) nothing to score: the barriers above keep the ring in step
    double d[2][NV], n2[2] = {0.0, 0.0};
#pragma unroll
    for (int u = 0; u < 2; ++u)
#pragma unroll
      for (int v = 0; v < NV; ++v) d[u][v] = 0.0;
    {
      const float4* r0 = reinterpret_cast<const float4*>(ring + ((size_t)(j % DB_STAGES) * DB_ROWS + lane) * ROW);
      const float4* r1 = reinterpret_cast<const float4*>(ring + ((size_t)(j % DB_STAGES) * DB_ROWS + 32 + lane) * ROW);
#pragma unroll 2
      for (int c4 = 0; c4 < F4; ++c4) {
        const float4 a4 = r0[c4], b4 = r1[c4];
        const double ya[4] = {(double)a4.x, (double)a4.y, (double)a4.z, (double)a4.w};
        const double yb[4] = {(double)b4.x, (double)b4.y, (double)b4.z, (double)b4.w};
#pragma unroll
        for (int e = 0; e < 4; ++e) {
          n2[0] = fma(ya[e], ya[e], n2[0]);
          n2[1] = fma(yb[e], yb[e], n2[1]);
          const double2* xr = reinterpret_cast<const double2*>(xw + (size_t)(c4 * 4 + e) * SB_QB);
#pragma unroll
          for (int v = 0; v < NV; v += 2) {
            const double2 x2 = xr[v / 2];
            d[0][v] = fma(x2.x, ya[e], d[0][v]);
            d[0][v + 1] = fma(x2.y, ya[e], d[0][v + 1]);
            d[1][v] = fma(x2.x, yb[e], d[1][v]);
            d[1][v + 1] = fma(x2.y, yb[e], d[1][v + 1]);
          }
        }
      }
    }
    double sc[2][CB_QPW];
#pragma unroll
    for (int u = 0; u < 2; ++u) {
#pragma unroll
      for (int q = 0; q < CB_QPW; ++q) sc[u][q] = 0.0;
      const double s2 = sqrt(n2[u]);
#pragma unroll
      for (int v = 0; v < NV; ++v)
        if (v < nvw) {
          const double n1n2 = s1r[v] * s2;
          const double term = (n1n2 == 0.0) ? 0.0 : d[u][v] / n1n2;
#pragma unroll
          for (int q = 0; q < CB_QPW; ++q)
            if (vqr[v] == q) sc[u][q] += term;      // the vectors of a query are consecutive: the sum runs in query order
        }
      if (weight && ext[u] >= 0) {
        const double w = weight[ext[u]];
#pragma unroll
        for (int q = 0; q < CB_QPW; ++q) sc[u][q] = sc[u][q] * w;
      }
    }
#pragma unroll
    for (int q = 0; q < CB_QPW; ++q) {
      if (q >= nqw) continue;
      const int4 h4 = *reinterpret_cast<const int4*>(&hdr[q]);
      const double thr = __hiloint2double(h4.y, h4.x);
      const int cnt = h4.z;
      const unsigned long long ck = *reinterpret_cast<volatile unsigned long long*>(&cthr[sub * CB_QPW + q]);
      const bool w0 = ext[0] >= 0 && sc[0][q] > 0.0 && (cnt < topk || sc[0][q] >= thr) && s1_key(sc[0][q]) >= ck;
      const bool w1 = ext[1] >= 0 && sc[1][q] > 0.0 && (cnt < topk || sc[1][q] >= thr) && s1_key(sc[1][q]) >= ck;
      if (!__any_sync(0xffffffffu, w0 || w1)) continue;
      if (FILT)
        cbf_insert(&hdr[q], ps + (size_t)q * topk, pi + (size_t)q * topk, &cthr[sub * CB_QPW + q], w0, sc[0][q], ext[0], w1,
                   sc[1][q], ext[1], topk, qid_of[q], nid_of[q], flt, bq0 + q);
      else
        cb_insert(&hdr[q], ps + (size_t)q * topk, pi + (size_t)q * topk, &cthr[sub * CB_QPW + q], w0, sc[0][q], ext[0], w1,
                  sc[1][q], ext[1], topk, qid_of[q], nid_of[q]);
    }
  }
  asm volatile("cp.async.wait_group 0;\n" ::);
  __syncwarp();
#pragma unroll 1
  for (int q = 0; q < nqw; ++q) {
    const int cnt = hdr[q].cnt;
    ScoreIdx* out = cand + (((size_t)(bq0 + q) * gridDim.x + blockIdx.x) * DB_RINGS + rg) * topk;
    for (int t = lane; t < topk; t += 32) {
      ScoreIdx e;
      e.s = t < cnt ? ps[(size_t)q * topk + t] : 0.0;
      e.i = t < cnt ? pi[(size_t)q * topk + t] : -1;
      out[t] = e;
    }
  }
}

// ---- similarproduct scoring, same structure: one query = nqv item vectors -------------------------------------
// qf: [nqv][kp] vectors of the query items that own a factor (query order kept); qid: all nq_all query item ids
// (external) - every one of them is excluded from the candidates (ALSAlgorithm.scala:243-245).  score_i = sum over the
// query vectors, in query order, of d / (sqrt(n1) * sqrt(n2)) with d, n1, n2 accumulated in fp64 in index order
// (ALSAlgorithm.scala:220-234), kept only if > 0.  cand: [gridDim.x][warps][topk].

__global__ void __launch_bounds__(SB_THREADS, 2)
score_cos_topk_batched_kernel(const float* __restrict__ Y, int n_items, int kp, int k,
                              const float* __restrict__ qf, const int* __restrict__ qid, int nq_all, int nqv,
                              const int* __restrict__ cand_ext, const uint8_t* __restrict__ mask,
                              const double* __restrict__ weight, const ScoreIdx* __restrict__ bound, int keep_query,
                              int topk, ScoreIdx* __restrict__ cand) {
  extern __shared__ __align__(16) unsigned char sb_smem[];
  const int row = kp + 4;
  const int nqp = (nqv + SC_G - 1) / SC_G * SC_G;
  ScoreIdx bnd;
  bnd.s = 0.0;
  bnd.i = TK_NO_BOUND;
  if (bound) bnd = *bound;
  double* xd = reinterpret_cast<double*>(sb_smem);                     // [kp][nqp]
  double* s1 = xd + (size_t)kp * nqp;                                   // [nqp] sqrt(n1) of every query vector
  float* tile = reinterpret_cast<float*>(s1 + nqp);                    // [SB_THREADS][row]
  double* hs = reinterpret_cast<double*>(tile + (size_t)SB_THREADS * row);   // [warps][topk] one pool per warp
  int* hi = reinterpret_cast<int*>(hs + (size_t)(SB_THREADS / 32) * topk);   // [warps][topk]
  int* sq = hi + (size_t)(SB_THREADS / 32) * topk;                      // [nq_all] excluded ids
  const int tid = threadIdx.x;
  for (int o = tid; o < kp * nqp; o += SB_THREADS) {
    const int c = o / nqp, t = o % nqp;
    xd[o] = (t < nqv) ? (double)qf[(size_t)t * kp + c] : 0.0;
  }
  for (int t = tid; t < nqp; t += SB_THREADS) {
    double n1 = 0.0;
    if (t < nqv)
      for (int c = 0; c < k; ++c) {
        const double a = (double)qf[(size_t)t * kp + c];
        n1 += a * a;
      }
    s1[t] = sqrt(n1);
  }
  for (int t = tid; t < nq_all; t += SB_THREADS) sq[t] = qid[t];
  const int lane = tid & 31, warp = tid >> 5;
  WarpPool wp;
  wp.thr = 0.0; wp.wid = -1; wp.worst = 0; wp.cnt = 0;
  double* ps = hs + (size_t)warp * topk;
  int* pi = hi + (size_t)warp * topk;
  const int ntiles = (n_items + SB_THREADS - 1) / SB_THREADS;
  const int f4row = kp / 4;
  for (int tl = blockIdx.x; tl < ntiles; tl += gridDim.x) {
    const int base = tl * SB_THREADS;
    __syncthreads();
    for (int o = tid; o < SB_THREADS * f4row; o += SB_THREADS) {
      const int r = o / f4row, c4 = o % f4row;
      float* d = tile + (size_t)r * row + c4 * 4;
      if (base + r < n_items) sb_cp_async16(d, Y + (size_t)(base + r) * kp + c4 * 4);
      else *reinterpret_cast<float4*>(d) = make_float4(0.f, 0.f, 0.f, 0.f);
    }
    asm volatile("cp.async.commit_group;\n" ::);
    asm volatile("cp.async.wait_group 0;\n" ::);
    __syncthreads();
    const int i = base + tid;
    int ext = (i < n_items) ? cand_ext[i] : -1;
    if (ext >= 0 && mask && mask[ext]) ext = -1;
    if (ext >= 0 && !keep_query)
      for (int t = 0; t < nq_all; ++t)
        if (sq[t] == ext) { ext = -1; break; }
    double score = 0.0;
    if (ext >= 0) {
      const float4* yrow = reinterpret_cast<const float4*>(tile + (size_t)tid * row);
      double n2 = 0.0;
      for (int c4 = 0; c4 < f4row; ++c4) {
        const float4 y4 = yrow[c4];
        const double b0 = (double)y4.x, b1 = (double)y4.y, b2 = (double)y4.z, b3 = (double)y4.w;
        n2 = fma(b0, b0, n2);   // padded columns are zero; b * b is exact in fp64, so fma == the reference's n2 += b * b
        n2 = fma(b1, b1, n2);
        n2 = fma(b2, b2, n2);
        n2 = fma(b3, b3, n2);
      }
      const double s2 = sqrt(n2);
      for (int g = 0; g < nqp; g += SC_G) {
        double d[SC_G];
#pragma unroll
        for (int j = 0; j < SC_G; ++j) d[j] = 0.0;
        for (int c4 = 0; c4 < f4row; ++c4) {
          const float4 y4 = yrow[c4];
          const float ye[4] = {y4.x, y4.y, y4.z, y4.w};
#pragma unroll
          for (int e = 0; e < 4; ++e) {
            const double yd = (double)ye[e];
            const double2* xr = reinterpret_cast<const double2*>(xd + (size_t)(c4 * 4 + e) * nqp + g);
#pragma unroll
            for (int j = 0; j < SC_G; j += 2) {
              const double2 x2 = xr[j / 2];
              d[j] = fma(x2.x, yd, d[j]);
              d[j + 1] = fma(x2.y, yd, d[j + 1]);
            }
          }
        }
#pragma unroll
        for (int j = 0; j < SC_G; ++j)
          if (g + j < nqv) {
            const double n1n2 = s1[g + j] * s2;
            score += (n1n2 == 0.0) ? 0.0 : d[j] / n1n2;
          }
      }
    }
    if (weight && ext >= 0) score = score * weight[ext];
    wpool_offer(wp, ext >= 0 && score > 0.0 && below_bound(bnd, score, ext), score, ext, topk, ps, pi);   // each warp pools the items it scored
  }
  __syncwarp();
  for (int t = lane; t < topk; t += 32) {
    ScoreIdx e;
    e.s = t < wp.cnt ? ps[t] : 0.0;
    e.i = t < wp.cnt ? pi[t] : -1;
    cand[((size_t)blockIdx.x * (SB_THREADS / 32) + warp) * topk + t] = e;
  }
}

// ---- similarproduct scoring for MANY queries (batchPredict, pio_als_similar_batch) ---------------------------------
// grid: (GX persistent CTAs striding over 256-item tiles, groups of SM_QG queries).  A staged tile is scored against
// every query vector of the group (<= SM_NV vectors: xd), the per-query sums go through shared memory (scs[q][item]),
// then warp q feeds the pool of query q (query items excluded unless keep_query, weights, score > 0, pass bound).
// Same arithmetic, in the same order, as score_cos_topk_batched_kernel -> bit-identical results.
//   gvec0[g] .. gvec0[g+1] : vectors of group g in qf ([total vectors][kp], query order inside a query)
//   vq[v]                  : query (0..SM_QG-1 inside the group) of vector v
//   qid_ptr / qid          : all query item ids (external) of every query, for the exclusion rule

template <bool FILT>
__global__ void __launch_bounds__(SB_THREADS, 2)
score_cos_topk_multi_kernel(const float* __restrict__ Y, int n_items, int kp, int k, const float* __restrict__ qf,
                            const int* __restrict__ gvec0, const int* __restrict__ vq, const long long* __restrict__ qid_ptr,
                            const int* __restrict__ qid, int n_queries, const int* __restrict__ cand_ext,
                            const uint8_t* __restrict__ mask, const double* __restrict__ weight,
                            const ScoreIdx* __restrict__ bound, int keep_query, int topk, ScoreIdx* __restrict__ cand,
                            const QueryFilterDev flt) {
  extern __shared__ __align__(16) unsigned char sb_smem[];
  const int row = kp + 4;
  double* xd = reinterpret_cast<double*>(sb_smem);                          // [kp][SM_NV]
  double* s1 = xd + (size_t)kp * SM_NV;                                      // [SM_NV]
  float* tile = reinterpret_cast<float*>(s1 + SM_NV);                       // [SB_THREADS][row]; reused for scs / sext
  const size_t tile_bytes = sb_tile_bytes(kp);
  double* hs = reinterpret_cast<double*>(reinterpret_cast<unsigned char*>(tile) + tile_bytes);   // [SM_QG][topk]
  int* hi = reinterpret_cast<int*>(hs + (size_t)SM_QG * topk);              // [SM_QG][topk]
  int* svq = hi + (size_t)SM_QG * topk;                                      // [SM_NV]
  int* sqid = svq + SM_NV;                                                   // [SM_QG][SM_QIDS] excluded ids of each query
  double* scs = reinterpret_cast<double*>(tile);                            // [SM_QG][SB_THREADS]
  int* sext = reinterpret_cast<int*>(scs + (size_t)SM_QG * SB_THREADS);     // [SB_THREADS]
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int grp = blockIdx.y, q0 = grp * SM_QG;
  const int v0 = gvec0[grp], nv = gvec0[grp + 1] - v0;
  for (int o = tid; o < kp * SM_NV; o += SB_THREADS) {
    const int c = o / SM_NV, t = o % SM_NV;
    xd[o] = (t < nv) ? (double)qf[(size_t)(v0 + t) * kp + c] : 0.0;
  }
  for (int t = tid; t < SM_NV; t += SB_THREADS) {
    double n1 = 0.0;
    if (t < nv)
      for (int c = 0; c < k; ++c) {
        const double a = (double)qf[(size_t)(v0 + t) * kp + c];
        n1 += a * a;
      }
    s1[t] = sqrt(n1);
    svq[t] = t < nv ? vq[v0 + t] : 0;
  }
  // warp w owns the pool of query q0 + w
  const int myq = q0 + warp;
  WarpPool wp;
  wp.thr = 0.0; wp.wid = -1; wp.worst = 0; wp.cnt = 0;
  ScoreIdx bnd;
  bnd.s = 0.0;
  bnd.i = TK_NO_BOUND;
  if (bound && myq < n_queries) bnd = bound[myq];
  long long ib = 0, ie = 0;
  if (myq < n_queries) { ib = qid_ptr[myq]; ie = qid_ptr[myq + 1]; }
  const bool ids_in_smem = ie - ib <= SM_QIDS;      // the usual case: the exclusion list is read from shared memory
  if (ids_in_smem)
    for (int t = lane; t < (int)(ie - ib); t += 32) sqid[warp * SM_QIDS + t] = qid[ib + t];
  __syncwarp();
  double* ps = hs + (size_t)warp * topk;
  int* pi = hi + (size_t)warp * topk;
  const int ntiles = (n_items + SB_THREADS - 1) / SB_THREADS;
  const int f4row = kp / 4;
  for (int tl = blockIdx.x; tl < ntiles; tl += gridDim.x) {
    const int base = tl * SB_THREADS;
    __syncthreads();
    for (int o = tid; o < SB_THREADS * f4row; o += SB_THREADS) {
      const int r = o / f4row, c4 = o % f4row;
      float* d = tile + (size_t)r * row + c4 * 4;
      if (base + r < n_items) sb_cp_async16(d, Y + (size_t)(base + r) * kp + c4 * 4);
      else *reinterpret_cast<float4*>(d) = make_float4(0.f, 0.f, 0.f, 0.f);
    }
    asm volatile("cp.async.commit_group;\n" ::);
    asm volatile("cp.async.wait_group 0;\n" ::);
    __syncthreads();
    const int i = base + tid;
    int ext = (i < n_items) ? cand_ext[i] : -1;
    if (ext >= 0 && mask && mask[ext]) ext = -1;
    double sc[SM_QG];
#pragma unroll
    for (int q = 0; q < SM_QG; ++q) sc[q] = 0.0;
    if (ext >= 0 && nv > 0) {
      const float4* yrow = reinterpret_cast<const float4*>(tile + (size_t)tid * row);
      double n2 = 0.0;
      for (int c4 = 0; c4 < f4row; ++c4) {
        const float4 y4 = yrow[c4];
        const double b0 = (double)y4.x, b1 = (double)y4.y, b2 = (double)y4.z, b3 = (double)y4.w;
        n2 = fma(b0, b0, n2);
        n2 = fma(b1, b1, n2);
        n2 = fma(b2, b2, n2);
        n2 = fma(b3, b3, n2);
      }
      const double s2 = sqrt(n2);
      for (int g = 0; g < nv; g += SC_G) {
        double d[SC_G];
#pragma unroll
        for (int j = 0; j < SC_G; ++j) d[j] = 0.0;
        for (int c4 = 0; c4 < f4row; ++c4) {
          const float4 y4 = yrow[c4];
          const float ye[4] = {y4.x, y4.y, y4.z, y4.w};
#pragma unroll
          for (int e = 0; e < 4; ++e) {
            const double yd = (double)ye[e];
            const double2* xr = reinterpret_cast<const double2*>(xd + (size_t)(c4 * 4 + e) * SM_NV + g);
#pragma unroll
            for (int j = 0; j < SC_G; j += 2) {
              const double2 x2 = xr[j / 2];
              d[j] = fma(x2.x, yd, d[j]);
              d[j + 1] = fma(x2.y, yd, d[j + 1]);
            }
          }
        }
#pragma unroll
        for (int j = 0; j < SC_G; ++j)
          if (g + j < nv) {
            const double n1n2 = s1[g + j] * s2;
            const double term = (n1n2 == 0.0) ? 0.0 : d[j] / n1n2;
            const int q = svq[g + j];
#pragma unroll
            for (int qq = 0; qq < SM_QG; ++qq)
              if (qq == q) sc[qq] += term;      // vectors of a query are consecutive: the sum runs in query order
          }
      }
      if (weight) {
        const double w = weight[ext];
#pragma unroll
        for (int q = 0; q < SM_QG; ++q) sc[q] = sc[q] * w;
      }
    }
    __syncthreads();   // the staged rows are dead
#pragma unroll
    for (int q = 0; q < SM_QG; ++q) scs[q * SB_THREADS + tid] = sc[q];
    sext[tid] = ext;
    __syncthreads();
    if (myq < n_queries) {
      for (int it = lane; it < SB_THREADS; it += 32) {
        const int e = sext[it];
        const double sv = scs[warp * SB_THREADS + it];
        bool want = e >= 0 && sv > 0.0 && below_bound(bnd, sv, e);
        if (FILT) want = want && (wp.cnt < topk || sv >= wp.thr) && !qf_drop(flt, myq, e);
        if (want && !keep_query) {
          if (ids_in_smem) {
            for (int t = 0; t < (int)(ie - ib); ++t)
              if (sqid[warp * SM_QIDS + t] == e) { want = false; break; }
          } else {
            for (long long t = ib; t < ie; ++t)
              if (qid[t] == e) { want = false; break; }
          }
        }
        wpool_offer(wp, want, sv, e, topk, ps, pi);
      }
    }
  }
  __syncwarp();
  if (myq < n_queries) {
    for (int t = lane; t < topk; t += 32) {
      ScoreIdx e;
      e.s = t < wp.cnt ? ps[t] : 0.0;
      e.i = t < wp.cnt ? pi[t] : -1;
      cand[((size_t)myq * gridDim.x + blockIdx.x) * topk + t] = e;
    }
  }
}

// (fallback for very large queries) one query = a set of item vectors. qf: [nqv][KP] vectors of the query items that own a factor
// (query order kept); qid: all nq_all query item ids (external) -- every one of them is excluded
// from the candidates (ALSAlgorithm.scala:243-245 `!queryList.contains(i)`).
__global__ void __launch_bounds__(TK_THREADS)
score_cos_topk_kernel(const float* __restrict__ Y, int n_items, int kp, int k,
                      const float* __restrict__ qf, const int* __restrict__ qid, int nq_all, int nqv,
                      const int* __restrict__ cand_ext, const uint8_t* __restrict__ mask,
                      const double* __restrict__ weight, const ScoreIdx* __restrict__ bound, int keep_query,
                      int topk, ScoreIdx* __restrict__ cand) {
  ScoreIdx bnd;
  bnd.s = 0.0;
  bnd.i = TK_NO_BOUND;
  if (bound) bnd = *bound;
  double sc[TK_ITEMS];
  int ix[TK_ITEMS];
#pragma unroll
  for (int j = 0; j < TK_ITEMS; ++j) {
    const int i = blockIdx.x * TK_TILE + j * TK_THREADS + threadIdx.x;
    sc[j] = 0.0;
    ix[j] = -1;
    const int ext = i < n_items ? cand_ext[i] : -1;
    if (ext >= 0 && !(mask && mask[ext])) {
      bool isq = false;
      if (!keep_query)
        for (int t = 0; t < nq_all; ++t) isq |= (qid[t] == ext);
      if (!isq) {
        const float* f = Y + (size_t)i * kp;
        double score = 0.0;
        for (int t = 0; t < nqv; ++t) {
          const float* v1 = qf + (size_t)t * kp;
          double n1 = 0.0, n2 = 0.0, d = 0.0;
          for (int c = 0; c < k; ++c) {
            const double a = (double)v1[c], b = (double)f[c];
            n1 += a * a;
            n2 += b * b;
            d += a * b;
          }
          const double n1n2 = sqrt(n1) * sqrt(n2);
          score += (n1n2 == 0.0) ? 0.0 : d / n1n2;
        }
        if (weight) score = score * weight[ext];
        if (score > 0.0 && below_bound(bnd, score, ext)) { sc[j] = score; ix[j] = ext; }
      }
    }
  }
  block_select_topk(sc, ix, topk, cand + (size_t)blockIdx.x * topk);
}

// ---- white-listed queries: scored over their lists ------------------------------------------------------------------
// A query with a white list has few candidates: scanning the item matrix for it would leave its pool unfilled for the
// whole scan (every item takes the insertion path).  Here one CTA takes one query and walks its sorted white list
// (wl: keys query << 32 | item id, like the exclusion lists; duplicates are adjacent and taken once, ids outside the
// item range skipped), one entry per lane: the item's row is read from the factor matrix and scored with the
// arithmetic of the scan kernels (fp64, index order; cosine terms in query order) -> the same bits.  Every rule of the
// scan applies: owns a factor, item_mask, set row, exclusion list, the query's own items (COS, unless keep_query),
// score > 0 (COS), weights, pass bound.  Each warp pools what it scored; the merge orders the LS_WARPS lists.
//   DOT: xq [queries][kp] user vectors, qvalid[q] == 0 -> no candidates
//   COS: xq [all query ids][kp] the gathered vector of every query id (zeros for an id without a factor: its cosine
//        terms are exactly 0), qid_ptr / qid the id list of every query
// grid: (1, queries of the launch); cand: [queries][LS_WARPS][topk]; bound: per query of the launch, or nullptr.
template <bool COS>
__global__ void __launch_bounds__(LS_THREADS)
score_listed_kernel(const float* __restrict__ Y, int kp, const int* __restrict__ perm, const unsigned* __restrict__ deg,
                    int n_ext, const float* __restrict__ xq, const uint8_t* __restrict__ qvalid,
                    const long long* __restrict__ qid_ptr, const int* __restrict__ qid,
                    const unsigned long long* __restrict__ wl, const long long* __restrict__ wl_ptr,
                    const uint8_t* __restrict__ mask, const double* __restrict__ weight,
                    const ScoreIdx* __restrict__ bound, int keep_query, int topk, ScoreIdx* __restrict__ cand,
                    const QueryFilterDev flt) {
  extern __shared__ __align__(16) unsigned char ls_smem[];
  double* hs = reinterpret_cast<double*>(ls_smem);            // [LS_WARPS][topk]
  int* hi = reinterpret_cast<int*>(hs + (size_t)LS_WARPS * topk);
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int q = flt.qbase + blockIdx.y;
  double* ps = hs + (size_t)warp * topk;
  int* pi = hi + (size_t)warp * topk;
  WarpPool wp;
  wp.thr = 0.0; wp.wid = -1; wp.worst = 0; wp.cnt = 0;
  ScoreIdx bnd;
  bnd.s = 0.0;
  bnd.i = TK_NO_BOUND;
  if (bound) bnd = bound[blockIdx.y];
  const long long wb = wl_ptr[q], we = wl_ptr[q + 1];
  long long ib = 0, ie = 0;
  if (COS) { ib = qid_ptr[q]; ie = qid_ptr[q + 1]; }
  const bool live = COS ? ie > ib : qvalid[q] != 0;
  const int f4row = kp / 4;
  for (long long base = wb + warp * 32; live && base < we; base += LS_THREADS) {
    const long long t = base + lane;
    int ext = -1;
    if (t < we) {
      const unsigned long long key = wl[t];
      const unsigned id = (unsigned)key;
      if (id < (unsigned)n_ext && !(t > wb && wl[t - 1] == key)) ext = (int)id;
    }
    if (ext >= 0 && deg[ext] == 0) ext = -1;
    if (ext >= 0 && mask && mask[ext]) ext = -1;
    if (ext >= 0 && qf_drop(flt, blockIdx.y, ext)) ext = -1;
    if (COS && ext >= 0 && !keep_query)
      for (long long v = ib; v < ie; ++v)
        if (qid[v] == ext) { ext = -1; break; }
    double score = 0.0;
    if (ext >= 0) {
      const float4* yrow = reinterpret_cast<const float4*>(Y + (size_t)perm[ext] * kp);
      if (COS) {
        double n2 = 0.0;
        for (int c4 = 0; c4 < f4row; ++c4) {
          const float4 y4 = __ldg(yrow + c4);
          const double b0 = (double)y4.x, b1 = (double)y4.y, b2 = (double)y4.z, b3 = (double)y4.w;
          n2 = fma(b0, b0, n2);
          n2 = fma(b1, b1, n2);
          n2 = fma(b2, b2, n2);
          n2 = fma(b3, b3, n2);
        }
        const double s2 = sqrt(n2);
        for (long long v = ib; v < ie; ++v) {
          const float4* xrow = reinterpret_cast<const float4*>(xq + (size_t)v * kp);
          double n1 = 0.0, d = 0.0;
          for (int c4 = 0; c4 < f4row; ++c4) {
            const float4 y4 = __ldg(yrow + c4), x4 = __ldg(xrow + c4);
            const double ye[4] = {(double)y4.x, (double)y4.y, (double)y4.z, (double)y4.w};
            const double xe[4] = {(double)x4.x, (double)x4.y, (double)x4.z, (double)x4.w};
#pragma unroll
            for (int e = 0; e < 4; ++e) {
              n1 = fma(xe[e], xe[e], n1);     // squares of fp32 values are exact in fp64: fma == n1 += a * a
              d = fma(xe[e], ye[e], d);
            }
          }
          const double n1n2 = sqrt(n1) * s2;
          score += (n1n2 == 0.0) ? 0.0 : d / n1n2;
        }
      } else {
        const float4* xrow = reinterpret_cast<const float4*>(xq + (size_t)q * kp);
        for (int c4 = 0; c4 < f4row; ++c4) {
          const float4 y4 = __ldg(yrow + c4), x4 = __ldg(xrow + c4);
          score = fma((double)x4.x, (double)y4.x, score);   // index order t = 0..k-1, like blas.ddot over Array[Double]
          score = fma((double)x4.y, (double)y4.y, score);
          score = fma((double)x4.z, (double)y4.z, score);
          score = fma((double)x4.w, (double)y4.w, score);
        }
      }
      if (weight) score = score * weight[ext];
    }
    wpool_offer(wp, ext >= 0 && (!COS || score > 0.0) && below_bound(bnd, score, ext), score, ext, topk, ps, pi);
  }
  __syncwarp();
  for (int t = lane; t < topk; t += 32) {
    ScoreIdx e;
    e.s = t < wp.cnt ? ps[t] : 0.0;
    e.i = t < wp.cnt ? pi[t] : -1;
    cand[((size_t)blockIdx.y * LS_WARPS + warp) * topk + t] = e;
  }
}

// grid: n_queries. Merges n_cand unsorted candidates per query (i = -1: empty) -> final topk, best first.
// Lock-free: every warp folds a strided share of the candidates into its own pool (wpool_offer: almost everything is
// rejected by the threshold once the pool is full), then the <= 8 x topk survivors are ordered by rank counting (ids are
// distinct, so better() is a total order).  A single-query call (serving latency) no longer serialises on a lock.
__global__ void __launch_bounds__(TK_THREADS)
topk_merge_kernel(const ScoreIdx* __restrict__ cand, int n_cand, int topk, int out_stride, int out_off,
                  int* __restrict__ out_items, float* __restrict__ out_scores, int* __restrict__ out_count,
                  ScoreIdx* __restrict__ bound_out) {
  constexpr int NW = TK_THREADS / 32;
  __shared__ double hs[NW * TK_MAXK];
  __shared__ int hi[NW * TK_MAXK];
  __shared__ int wcnt[NW];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const ScoreIdx* c = cand + (size_t)blockIdx.x * n_cand;
  WarpPool wp;
  wp.thr = 0.0; wp.wid = -1; wp.worst = 0; wp.cnt = 0;
  double* ps = hs + warp * topk;
  int* pi = hi + warp * topk;
  for (int base = warp * 32; base < n_cand; base += TK_THREADS) {
    const int o = base + lane;
    ScoreIdx e;
    e.s = 0.0;
    e.i = -1;
    if (o < n_cand) e = c[o];
    wpool_offer(wp, e.i >= 0, e.s, e.i, topk, ps, pi);
  }
  if (lane == 0) wcnt[warp] = wp.cnt;
  __syncthreads();
  int total = 0;
#pragma unroll
  for (int w = 0; w < NW; ++w) total += wcnt[w];
  const int cnt = total < topk ? total : topk;
  int* oi = out_items + (size_t)blockIdx.x * out_stride + out_off;
  float* os = out_scores + (size_t)blockIdx.x * out_stride + out_off;
  for (int t = threadIdx.x; t < topk; t += TK_THREADS)
    if (t >= cnt) {   // fewer candidates than topk: the tail stays empty
      oi[t] = -1;
      os[t] = 0.f;
    }
  // rank of every survivor among all survivors
  for (int t = threadIdx.x; t < NW * topk; t += TK_THREADS) {
    const int w = t / topk, j = t % topk;
    if (j >= wcnt[w]) continue;
    const double s = hs[t];
    const int id = hi[t];
    int rank = 0;
    for (int w2 = 0; w2 < NW; ++w2)
      for (int u = 0; u < wcnt[w2]; ++u) rank += better(hs[w2 * topk + u], hi[w2 * topk + u], s, id) ? 1 : 0;
    if (rank < topk) {
      oi[rank] = id;
      os[rank] = (float)s;
      if (bound_out && rank == topk - 1) {   // the last result of a full pass bounds the next pass
        bound_out[blockIdx.x].s = s;
        bound_out[blockIdx.x].i = id;
      }
    }
  }
  if (threadIdx.x == 0) {
    if (out_count && (out_off == 0 || cnt > 0)) out_count[blockIdx.x] = out_off + cnt;
    if (bound_out && cnt < topk) bound_out[blockIdx.x].i = TK_EXHAUSTED;
  }
}

// ---- one query, one launch (serving latency) -----------------------------------------------------------------------
// The whole predict call of a deployed engine for ONE query (ALSModel.recommendProducts for a user; the similarproduct
// cosine scan for <= S1_MAXNV query items) as a single kernel: the query rows are looked up by the CTAs themselves (ids
// travel in the kernel parameters); one persistent CTA per SM streams its share of the item matrix; inside the CTA every
// warp is independent -- it stages its own 32 rows per step through its own three-stage cp.async ring (padded rows,
// conflict-free LDS.128 per thread), scores them and keeps its own top-k pool, with no CTA barrier in the scan; a score
// below the smallest entry of ANY full pool (shared through shared / global memory) never reaches a pool; the eight
// pools of a CTA are merged by rank counting; the last CTA to finish (device counter) merges the per-CTA lists and
// writes the result straight into mapped host memory, followed by a sequence flag the host polls.  Arithmetic and
// tie-breaking are those of the batched kernels above (fp64 in index order, better()): results are bit-identical.
struct OneQuery {
  int nq;
  int ids[S1_MAXNV];   // external ids (COS: the query items; dot: ids[0] = the user)
};
// n_lists lists of topk candidates each, every list best first and padded with i = -1 -> the best topk overall.
// Only candidates at least as good as the topk-th best list head can make it: those few are collected in `surv` (shared
// memory, capacity cap) and ordered by rank counting.  All S1_THREADS threads call; returns the number of results.
template <typename Emit>
__device__ __forceinline__ int s1_merge_lists(const ScoreIdx* c, int n_lists, int topk, ScoreIdx* surv, int cap, int* s_int,
                                              double* s_dbl, Emit emit) {
  const int tid = threadIdx.x;
  // s_int[0] = survivors, s_int[1] = id of the threshold head (or -1: keep everything), s_dbl[0] = its score
  if (tid == 0) { s_int[0] = 0; s_int[1] = -1; }
  __syncthreads();
  double hs_ = 0.0;
  int hi_ = -1;
  if (tid < n_lists) {
    hs_ = __ldcg(&c[(size_t)tid * topk].s);
    hi_ = __ldcg(&c[(size_t)tid * topk].i);
  }
  surv[tid].s = hs_;      // heads, exchanged through the survivor buffer (cap >= S1_THREADS)
  surv[tid].i = hi_;
  __syncthreads();
  if (hi_ >= 0) {
    int rank = 0;
#pragma unroll 4
    for (int l = 0; l < n_lists; ++l) {
      const int oi = surv[l].i;
      rank += (oi >= 0 && better(surv[l].s, oi, hs_, hi_)) ? 1 : 0;
    }
    if (rank == topk - 1) { s_int[1] = hi_; s_dbl[0] = hs_; }
  }
  __syncthreads();
  const int ti = s_int[1];
  const double ts = s_dbl[0];
  __syncthreads();          // the heads have been read: the buffer now collects survivors
  const int n_cand = n_lists * topk;
  for (int o0 = tid; o0 < n_cand; o0 += 8 * S1_THREADS) {   // eight loads in flight per thread
    double sv[8];
    int id[8];
#pragma unroll
    for (int u = 0; u < 8; ++u) {
      const int o = o0 + u * S1_THREADS;
      id[u] = -1;
      sv[u] = 0.0;
      if (o < n_cand) {
        sv[u] = __ldcg(&c[o].s);
        id[u] = __ldcg(&c[o].i);
      }
    }
#pragma unroll
    for (int u = 0; u < 8; ++u)
      if (id[u] >= 0 && (ti < 0 || !better(ts, ti, sv[u], id[u]))) {
        const int at = atomicAdd(&s_int[0], 1);
        if (at < cap) { surv[at].s = sv[u]; surv[at].i = id[u]; }
      }
  }
  __syncthreads();
  const int m = s_int[0];
  if (m > cap) return -1;   // (adversarial input) the caller takes the pool path
  for (int t = tid; t < m; t += S1_THREADS) {
    const double sv = surv[t].s;
    const int id = surv[t].i;
    int rank = 0;
#pragma unroll 4
    for (int u = 0; u < m; ++u) rank += better(surv[u].s, surv[u].i, sv, id) ? 1 : 0;
    if (rank < topk) emit(rank, sv, id);
  }
  return m < topk ? m : topk;
}

// merge through per-warp pools (the CTA's own eight pools when c == nullptr: wcnt[] is already set)
template <typename Emit>
__device__ __forceinline__ int s1_merge(const ScoreIdx* c, int n_cand, int topk, double* hs, int* hi, int* wcnt, Emit emit) {
  constexpr int NW = S1_THREADS / 32;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  if (c) {
    WarpPool wp;
    wp.thr = 0.0; wp.wid = -1; wp.worst = 0; wp.cnt = 0;
    for (int base = warp * 32; base < n_cand; base += S1_THREADS) {
      const int o = base + lane;
      double s = 0.0;
      int i = -1;
      if (o < n_cand) {
        s = __ldcg(&c[o].s);
        i = __ldcg(&c[o].i);
      }
      wpool_offer(wp, i >= 0, s, i, topk, hs + warp * topk, hi + warp * topk);
    }
    if (lane == 0) wcnt[warp] = wp.cnt;
  }
  __syncthreads();
  int total = 0;
#pragma unroll
  for (int w = 0; w < NW; ++w) total += wcnt[w];
  for (int t = threadIdx.x; t < NW * topk; t += S1_THREADS) {
    const int w = t / topk, j = t % topk;
    if (j >= wcnt[w]) continue;
    const double s = hs[t];
    const int id = hi[t];
    int rank = 0;
    if (c) {
      for (int w2 = 0; w2 < NW; ++w2)
        for (int u = 0; u < wcnt[w2]; ++u) rank += better(hs[w2 * topk + u], hi[w2 * topk + u], s, id) ? 1 : 0;
    } else {
      // the CTA's own pools are sorted best first: entries better than (s, id) in a pool = a lower bound by bisection
      for (int w2 = 0; w2 < NW; ++w2) {
        int lo = 0, hi2 = wcnt[w2];
        while (lo < hi2) {
          const int mid = (lo + hi2) >> 1;
          if (better(hs[w2 * topk + mid], hi[w2 * topk + mid], s, id)) lo = mid + 1;
          else hi2 = mid;
        }
        rank += lo;
      }
    }
    if (rank < topk) emit(rank, s, id);
  }
  return total < topk ? total : topk;
}

// streaming copy: the scanned matrix is marked evict-first in L2, so that what the NEXT query needs again (this kernel's
// code, the id maps, the query rows) is not pushed out of the 126 MB L2 by a 256 MB scan
__device__ __forceinline__ void s1_cp_async16_stream(void* smem_dst, const void* gsrc, unsigned long long policy) {
  const unsigned d = (unsigned)__cvta_generic_to_shared(smem_dst);
  asm volatile("cp.async.cg.shared.global.L2::cache_hint [%0], [%1], 16, %2;\n" ::"r"(d), "l"(gsrc), "l"(policy));
}

template <bool COS, int NVP, int KP>
__global__ void __launch_bounds__(S1_THREADS, 1)
score_one_kernel(const float* __restrict__ Y, int n_items, int k, const float* __restrict__ Q,
                 const int* __restrict__ q_perm, const uint32_t* __restrict__ q_deg, int q_n_ext, const OneQuery qry,
                 const int* __restrict__ cand_ext, const uint8_t* __restrict__ mask, const double* __restrict__ weight,
                 int keep_query, int topk, ScoreIdx* __restrict__ cand, unsigned* __restrict__ counter,
                 unsigned long long* __restrict__ g_thr,
                 int* __restrict__ out_items, float* __restrict__ out_scores, int* __restrict__ out_count,
                 volatile unsigned* __restrict__ done_flag, unsigned seq, unsigned long long* __restrict__ trace) {
  constexpr int NW = S1_THREADS / 32;
  constexpr int ROW = KP + 4;                 // floats per staged row: 16 bytes of skew -> conflict-free LDS.128 per thread
  constexpr int F4 = KP / 4;                  // 16-byte chunks per row
  unsigned long long t_begin = 0ull;          // PIO_ALS_SERVE_TRACE: %globaltimer stamps of the CTA that publishes the result
  auto now = [&]() {
    unsigned long long t;
    asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
    return t;
  };
  if (trace && threadIdx.x == 0) t_begin = now();
  extern __shared__ __align__(16) unsigned char s1_smem[];
  double* xd = reinterpret_cast<double*>(s1_smem);                       // [KP][NVP]
  double* s1 = xd + (size_t)KP * NVP;                                     // [S1_MAXNV]
  float* tiles = reinterpret_cast<float*>(s1 + S1_MAXNV);                // [NW][S1_STAGES][32][ROW]
  double* hs = reinterpret_cast<double*>(tiles + (size_t)S1_STAGES * S1_THREADS * ROW);   // [NW][topk]
  int* hi = reinterpret_cast<int*>(hs + (size_t)NW * topk);              // [NW][topk]
  int* wcnt = hi + (size_t)NW * topk;                                     // [NW]
  int* s_int = wcnt + NW;                                                 // [4]
  double* s_dbl = reinterpret_cast<double*>(s_int + 4);                  // [1]
  __shared__ unsigned long long s_thr;        // key of the CTA's pruning threshold (0 = none yet)
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int ntiles = (n_items + S1_THREADS - 1) / S1_THREADS;
  const int my_tiles = (int)blockIdx.x < ntiles ? (ntiles - 1 - (int)blockIdx.x) / (int)gridDim.x + 1 : 0;
  float* ring = tiles + (size_t)warp * S1_STAGES * 32 * ROW;
  unsigned long long l2_stream;
  asm volatile("createpolicy.fractional.L2::evict_first.b64 %0, 1.0;" : "=l"(l2_stream));
  // step j of this warp: rows base(j) .. base(j) + 31 -> ring slot j % S1_STAGES; one commit group per step (empty past the end)
  auto base_of = [&](int j) { return (((int)blockIdx.x + j * (int)gridDim.x) * NW + warp) * 32; };
  auto fetch = [&](int j) {
    if (j < my_tiles) {
      const int base = base_of(j);
      // a warp copies 512 contiguous bytes per instruction: lane -> (row lane / F4, chunk lane % F4), + 32 / F4 rows per copy
      float* dst = ring + (size_t)(j % S1_STAGES) * 32 * ROW + (size_t)(lane / F4) * ROW + (lane % F4) * 4;
      const float* src = Y + (size_t)(base + lane / F4) * KP + (lane % F4) * 4;
      if (base + 32 <= n_items) {
#pragma unroll
        for (int m = 0; m < F4; ++m) s1_cp_async16_stream(dst + (size_t)m * (32 / F4) * ROW, src + (size_t)m * (32 / F4) * KP, l2_stream);
      } else {
#pragma unroll
        for (int m = 0; m < F4; ++m)
          if (base + lane / F4 + m * (32 / F4) < n_items)
            s1_cp_async16_stream(dst + (size_t)m * (32 / F4) * ROW, src + (size_t)m * (32 / F4) * KP, l2_stream);
      }
    }
    asm volatile("cp.async.commit_group;\n" ::);
  };
#pragma unroll
  for (int s = 0; s < S1_STAGES - 1; ++s) fetch(s);
  if (tid == 0) s_thr = 0ull;
  // the query: rows looked up by external id; an id without a factor enters as a zero vector (its cosine terms are 0)
  for (int o = tid; o < KP * NVP; o += S1_THREADS) {
    const int c = o / NVP, t = o % NVP;
    const int id = t < qry.nq ? qry.ids[t] : -1;
    const bool ok = id >= 0 && id < q_n_ext && q_deg[id] > 0;
    xd[o] = ok ? (double)Q[(size_t)q_perm[id] * KP + c] : 0.0;
  }
  bool qvalid;
  {
    const int id = qry.ids[0];
    qvalid = qry.nq > 0 && id >= 0 && id < q_n_ext && q_deg[id] > 0;   // dot: an unknown user has no recommendations
  }
  __syncthreads();
  // one query vector: it lives in registers for the whole scan (one CTA per SM: 255 registers per thread are free)
  constexpr bool XREG = NVP == 1 && !COS;
  double xreg[XREG ? KP : 1];
  double s1r[NVP];
  if (XREG) {
#pragma unroll
    for (int c = 0; c < KP; ++c) xreg[c] = xd[c];
    s1r[0] = 0.0;
  } else {
    if (COS && tid < NVP) {
      double n1 = 0.0;      // index order; columns >= k hold zeros: + 0.0 is exact
#pragma unroll 8
      for (int c = 0; c < KP; ++c) {
        const double a = xd[(size_t)c * NVP + tid];
        n1 += a * a;
      }
      s1[tid] = sqrt(n1);
    }
    __syncthreads();
#pragma unroll
    for (int t = 0; t < NVP; ++t) s1r[t] = COS ? s1[t] : 0.0;
  }
  unsigned long long t_query = 0ull, t_step0 = 0ull;
  if (trace && tid == 0) t_query = now();
  SortedPool wp;
  wp.init();
  int ext_next = -1;
  if (my_tiles > 0) {
    const int i0 = base_of(0) + lane;
    ext_next = i0 < n_items ? __ldg(cand_ext + i0) : -1;
  }
  for (int j = 0; j < my_tiles; ++j) {
    int ext = ext_next;
    if (j + 1 < my_tiles) {
      const int in = base_of(j + 1) + lane;
      ext_next = in < n_items ? __ldg(cand_ext + in) : -1;
    }
    if (ext >= 0 && mask && mask[ext]) ext = -1;
    unsigned long long gthr = 0ull;
    if (lane == 0) gthr = __ldcg(g_thr);   // consumed after the row has been scored: the load latency hides behind it
    asm volatile("cp.async.wait_group %0;\n" ::"n"(S1_STAGES - 2));
    __syncwarp();               // step j has landed for the whole warp; slot (j - 1) % S1_STAGES has been consumed
    fetch(j + S1_STAGES - 1);
    double score = 0.0;
    if (ext >= 0) {
      const float4* yrow = reinterpret_cast<const float4*>(ring + ((size_t)(j % S1_STAGES) * 32 + lane) * ROW);
      double d[NVP];
#pragma unroll
      for (int t = 0; t < NVP; ++t) d[t] = 0.0;
      double n2 = 0.0;
      if (XREG) {
#pragma unroll
        for (int c4 = 0; c4 < F4; ++c4) {
          const float4 y4 = yrow[c4];
          const double yd[4] = {(double)y4.x, (double)y4.y, (double)y4.z, (double)y4.w};
#pragma unroll
          for (int e = 0; e < 4; ++e) {
            if (COS) n2 = fma(yd[e], yd[e], n2);
            d[0] = fma(xreg[(XREG ? c4 * 4 + e : 0)], yd[e], d[0]);   // index order, like blas.ddot over Array[Double]
          }
        }
      } else {
#pragma unroll 4
        for (int c4 = 0; c4 < F4; ++c4) {
          const float4 y4 = yrow[c4];
          const double yd[4] = {(double)y4.x, (double)y4.y, (double)y4.z, (double)y4.w};
#pragma unroll
          for (int e = 0; e < 4; ++e) {
            if (COS) n2 = fma(yd[e], yd[e], n2);
            if (NVP == 1) {
              d[0] = fma(xd[c4 * 4 + e], yd[e], d[0]);
            } else {
              const double2* xr = reinterpret_cast<const double2*>(xd + (size_t)(c4 * 4 + e) * NVP);
#pragma unroll
              for (int t = 0; t < NVP; t += 2) {
                const double2 x2 = xr[t / 2];
                d[t] = fma(x2.x, yd[e], d[t]);
                d[t + (NVP > 1 ? 1 : 0)] = fma(x2.y, yd[e], d[t + (NVP > 1 ? 1 : 0)]);
              }
            }
          }
        }
      }
      if (COS) {
        const double s2 = sqrt(n2);
#pragma unroll
        for (int t = 0; t < NVP; ++t)
          if (t < qry.nq) {
            const double n1n2 = s1r[t] * s2;
            score += (n1n2 == 0.0) ? 0.0 : d[t] / n1n2;   // query order
          }
      } else {
        score = d[0];
      }
      if (weight) score = score * weight[ext];
    }
    bool want = ext >= 0 && (COS ? score > 0.0 : qvalid);
    if (COS && want && !keep_query) {
#pragma unroll
      for (int t = 0; t < S1_MAXNV; ++t)
        if (t < qry.nq && qry.ids[t] == ext) want = false;
    }
    if (lane == 0 && gthr) atomicMax(&s_thr, gthr);
    want = want && s1_key(score) >= *reinterpret_cast<volatile unsigned long long*>(&s_thr);
    if (__any_sync(0xffffffffu, want)) {
      const double thr0 = wp.thr;
      const int cnt0 = wp.cnt;
      wp.offer(want, score, ext, topk);
      if (lane == 0 && wp.cnt == topk && (cnt0 < topk || wp.thr != thr0)) {
        const unsigned long long key = s1_key(wp.thr);
        if (atomicMax(&s_thr, key) < key) atomicMax(g_thr, key);
      }
    }
    if (trace && tid == 0 && j == 0) t_step0 = now();
  }
  asm volatile("cp.async.wait_group 0;\n" ::);
  unsigned long long t_scan = 0ull;
  if (trace && tid == 0) t_scan = now();
  wp.dump(topk, hs + (size_t)warp * topk, hi + (size_t)warp * topk);
  if (lane == 0) wcnt[warp] = wp.cnt;
  // the CTA's own list: topk entries best first, empty slots marked
  ScoreIdx* mine = cand + (size_t)blockIdx.x * topk;
  const int got = s1_merge(nullptr, 0, topk, hs, hi, wcnt, [&](int rank, double s, int id) {
    mine[rank].s = s;
    mine[rank].i = id;
  });
  for (int t = got + tid; t < topk; t += S1_THREADS) {
    mine[t].s = 0.0;
    mine[t].i = -1;
  }
  __syncthreads();          // the CTA's list is written; thread 0 publishes it (its fence is cumulative over the barrier)
  if (tid == 0) {
    __threadfence();
    s_int[2] = atomicAdd(counter, 1u) == gridDim.x - 1 ? 1 : 0;
    __threadfence();        // the last CTA reads the other lists after this
  }
  __syncthreads();
  if (!s_int[2]) return;    // the scan is over everywhere: the staging rings are free to hold the survivors
  unsigned long long t_last = 0ull;
  if (trace && tid == 0) t_last = now();
  auto publish = [&](int rank, double s, int id) {
    out_items[rank] = id;
    out_scores[rank] = (float)s;
  };
  constexpr int CAP = (int)(sizeof(float) * S1_STAGES * S1_THREADS * ROW / sizeof(ScoreIdx));
  int cnt = s1_merge_lists(cand, (int)gridDim.x, topk, reinterpret_cast<ScoreIdx*>(tiles), CAP, s_int, s_dbl, publish);
  if (cnt < 0) {
    __syncthreads();
    cnt = s1_merge(cand, (int)gridDim.x * topk, topk, hs, hi, wcnt, publish);
  }
  for (int t = cnt + tid; t < topk; t += S1_THREADS) {
    out_items[t] = -1;
    out_scores[t] = 0.f;
  }
  if (tid == 0) {
    *out_count = cnt;
    *counter = 0u;
    *g_thr = 0ull;
    if (trace) {
      trace[0] = t_begin; trace[1] = t_scan; trace[2] = t_last; trace[3] = now(); trace[5] = t_query; trace[6] = t_step0;
    }
  }
  __threadfence_system();
  __syncthreads();
  if (tid == 0) {
    if (trace) trace[4] = now();
    *done_flag = seq;
  }
}

// ------------------------------------------------------------------------------------------
// NaiveBayes: per-class counts and feature sums (fp64), deterministic two-stage reduction.
// partial: [gridDim.x][n_class * (n_feat + 1)]  (slot n_feat = count)
// ------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256)
nb_partial_kernel(const int* __restrict__ label, const float* __restrict__ x, long long n, int n_feat,
                  int n_class, double* __restrict__ partial) {
  extern __shared__ double acc[];  // [warps][n_class*(n_feat+1)]
  const int w = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int width = n_class * (n_feat + 1);
  double* my = acc + w * width;
  for (int o = lane; o < width; o += 32) my[o] = 0.0;
  __syncwarp();
  const long long per = (n + gridDim.x - 1) / gridDim.x;
  const long long r0 = (long long)blockIdx.x * per;
  const long long r1 = r0 + per < n ? r0 + per : n;
  // each warp walks its strided rows; lanes serialise their updates in lane order so the
  // summation order is fixed (values are typically small integers, sums exact in fp64).
  // Slot f (the count at f == n_feat) belongs to lane f % 32 at every width.
  for (long long base = r0 + (long long)w * 32; base < r1; base += 8 * 32) {
    const long long r = base + lane;
    int c = -1;
    if (r < r1) c = label[r];
    for (int src = 0; src < 32; ++src) {
      const int cc = __shfl_sync(0xffffffffu, c, src);
      if (cc < 0) continue;
      const long long rr = base + src;
      for (int f = lane; f <= n_feat; f += 32)
        my[cc * (n_feat + 1) + f] += f < n_feat ? (double)x[rr * n_feat + f] : 1.0;
    }
  }
  __syncthreads();
  for (int o = threadIdx.x; o < width; o += blockDim.x) {
    double s = 0.0;
    for (int q = 0; q < (int)(blockDim.x >> 5); ++q) s += acc[q * width + o];
    partial[(size_t)blockIdx.x * width + o] = s;
  }
}

__global__ void nb_reduce_kernel(const double* __restrict__ partial, int nparts, int width,
                                 double* __restrict__ out) {
  const int o = blockIdx.x * blockDim.x + threadIdx.x;
  if (o >= width) return;
  double s = 0.0;
  for (int q = 0; q < nparts; ++q) s += partial[(size_t)q * width + o];
  out[o] = s;
}

__global__ void __launch_bounds__(256)
nb_predict_kernel(const float* __restrict__ x, long long n, int n_feat, int n_class,
                  const double* __restrict__ pi, const double* __restrict__ theta, int* __restrict__ out) {
  const long long r = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (r >= n) return;
  int bestc = 0;
  double bests = -INFINITY;
  for (int c = 0; c < n_class; ++c) {
    double s = pi[c];
    // separate multiply and add (no FMA contraction) so the result is bit-identical to the
    // reference-order host arithmetic
    for (int j = 0; j < n_feat; ++j) s = __dadd_rn(s, __dmul_rn(theta[c * n_feat + j], (double)x[r * n_feat + j]));
    if (s > bests) { bests = s; bestc = c; }
  }
  out[r] = bestc;
}

}  // namespace pio
