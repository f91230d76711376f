// popular.cuh -- batch top-N of one fixed per-item score under per-query filters: the ecommerce template's
// predictDefault (examples/scala-parallel-ecommercerecommendation/adjust-score/src/main/scala/ECommAlgorithm.scala:
// 508-538) for a batch of cold users (DESIGN.md 4.14).
//   once per model: descending order keys of the scores -> stable radix sort -> the ranked order (item, score) and
//   each item's rank position;
//   per part of a call: a warp per query walks the ranked order (no white list) or its white list re-keyed by rank
//   position and sorted, 32 entries at a time, keeping the entries qf_drop does not drop, until it has topk.
// No arithmetic on the scores: every output score is a copy of the caller's.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include "sort_scan.cuh"
#include "topk.cuh"

namespace pio {

// a white-list entry whose id is outside [0, n_items): sorts after every rank position of its query
constexpr uint32_t PP_NO_RANK = 0xffffffffu;

// (key, payload) = (descending order key of scores[i], i): an ascending stable sort ranks the items by score
// descending, -0.0 with +0.0 (s1_key), equal scores by item index
__global__ void pp_rank_keys_kernel(const double* __restrict__ scores, int n, uint64_t* __restrict__ key,
                                    uint32_t* __restrict__ val) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  key[i] = ~s1_key(scores[i]);
  val[i] = (uint32_t)i;
}

// the sorted payloads -> the ranked order: order[p] / sorted[p] = item / score at rank position p, rank[item] = p
__global__ void pp_ranked_kernel(const uint32_t* __restrict__ perm, const double* __restrict__ scores, int n,
                                 int* __restrict__ order, double* __restrict__ sorted, int* __restrict__ rank) {
  const int p = blockIdx.x * blockDim.x + threadIdx.x;
  if (p >= n) return;
  const int i = (int)perm[p];
  order[p] = i;
  sorted[p] = scores[i];
  rank[i] = p;
}

// white-list keys (query << 32 | item), as upload_lists sorts them -> (query << 32 | rank position of item), or
// PP_NO_RANK for an id outside the item range; no payload
__global__ void pp_list_keys_kernel(const unsigned long long* __restrict__ wl, long long n, const int* __restrict__ rank,
                                    int n_items, uint64_t* __restrict__ key, uint32_t* __restrict__ val) {
  const long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= n) return;
  const unsigned long long k = wl[t];
  const unsigned item = (unsigned)k;
  key[t] = (k & 0xffffffff00000000ull) | (item < (unsigned)n_items ? (uint32_t)__ldg(rank + item) : PP_NO_RANK);
  val[t] = 0u;
}

// the ranked order of a model on the device
struct PopularRanked {
  const int* order = nullptr;      // [n_items] item at rank position p
  const double* sorted = nullptr;  // [n_items] its score
  int n_items = 0;
};

// the white lists of one part: sorted (query << 32 | rank position) keys, query q's in keys[ptr[q] .. ptr[q + 1])
struct PopularLists {
  const uint8_t* has_wl = nullptr;   // [queries]; nullptr: no query of the part has a white list
  const uint64_t* keys = nullptr;
  const long long* ptr = nullptr;
};

// One warp per query q of a part.  Its source is the ranked order [0, n_items) or, when it has a white list, its
// re-keyed list; both are in rank order.  Each round the warp reads 32 entries, keeps those that are a first
// occurrence of a valid rank position and that qf_drop keeps, and places them by ballot prefix counts until topk are
// placed.  The rest of the row is padded with -1 / 0.  *walked adds the ranked-order entries the walks read.
__global__ void __launch_bounds__(256) pp_take_kernel(PopularRanked R, int nq, int topk, QueryFilterDev f, PopularLists L,
                                                      int* __restrict__ out_items, double* __restrict__ out_scores,
                                                      int* __restrict__ out_count,
                                                      unsigned long long* __restrict__ walked) {
  const int q = (int)(((long long)blockIdx.x * blockDim.x + threadIdx.x) >> 5);
  const int lane = threadIdx.x & 31;
  if (q >= nq) return;
  const bool listed = L.has_wl && L.has_wl[q];
  const long long lo = listed ? L.ptr[q] : 0, hi = listed ? L.ptr[q + 1] : R.n_items;
  const size_t row = (size_t)q * topk;
  const unsigned below = (1u << lane) - 1u;
  int got = 0;
  long long b = lo;
  for (; b < hi && got < topk; b += 32) {
    const long long e = b + lane;
    int item = -1;
    double s = 0.0;
    if (e < hi) {
      uint32_t p = (uint32_t)e;
      if (listed) {
        const uint64_t k = L.keys[e];
        p = (uint32_t)k;
        if (e > lo && L.keys[e - 1] == k) p = PP_NO_RANK;   // a repeat of the entry before it
      }
      if (p != PP_NO_RANK) {
        item = __ldg(R.order + p);
        if (qf_drop(f, q, item)) item = -1;
        else s = __ldg(R.sorted + p);
      }
    }
    const unsigned keep = __ballot_sync(0xffffffffu, item >= 0);
    const int pos = got + __popc(keep & below);
    if (item >= 0 && pos < topk) {
      out_items[row + pos] = item;
      out_scores[row + pos] = s;
    }
    got += __popc(keep);
  }
  const int cnt = min(got, topk);
  for (int r = cnt + lane; r < topk; r += 32) {
    out_items[row + r] = -1;
    out_scores[row + r] = 0.0;
  }
  if (lane == 0) {
    out_count[q] = cnt;
    if (!listed) atomicAdd(walked, (unsigned long long)min(b, hi));
  }
}

}  // namespace pio
