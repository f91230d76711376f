// cooc_predict.cuh -- batch scoring of the similarproduct template's CooccurrenceAlgorithm.predict
// (examples/scala-parallel-similarproduct/multi-events-multi-algos/src/main/scala/CooccurrenceAlgorithm.scala:107-175)
// over a device copy of the trained top lists (DESIGN.md 4.9).  Per part of a batch:
//   query lists as sorted (query << 32 | item) keys -> expansion of each distinct known query item into its top list,
//   keyed (query << bits_i | candidate) with the count as payload -> radix sort -> one int64 sum per run of equal keys
//   whose (query, candidate) passes the filters -> two stable sorts, by inverted score then by query -> first topk.
// Integer work only: every output is exact.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include "sort_scan.cuh"
#include "topk.cuh"

namespace pio {

// is key in the ascending keys[lo .. hi)?
__device__ __forceinline__ bool cp_sorted_has(const unsigned long long* __restrict__ keys, long long lo, long long hi,
                                              unsigned long long key) {
  const long long end = hi;
  while (lo < hi) {
    const long long mid = (lo + hi) >> 1;
    if (__ldg(keys + mid) < key) lo = mid + 1;
    else hi = mid;
  }
  return lo < end && __ldg(keys + lo) == key;
}

// size[t] = top_n of the item of query-list entry t, or 0 for an id outside [0, n_items) and for a repeat of the entry
// before it (the keys are sorted, so a query's repeats are adjacent): each distinct known query item expands once
__global__ void cp_size_kernel(const unsigned long long* __restrict__ qk, long long n, int n_items,
                               const int* __restrict__ top_n, uint32_t* __restrict__ size) {
  const long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= n) return;
  const unsigned long long k = qk[t];
  const unsigned item = (unsigned)k;
  const bool keep = item < (unsigned)n_items && (t == 0 || qk[t - 1] != k);
  size[t] = keep ? (uint32_t)__ldg(top_n + item) : 0u;
}

// one warp per query-list entry: its size[t] top-list entries go to off[t] .. as (query << bits_i | candidate, count)
__global__ void cp_expand_kernel(const unsigned long long* __restrict__ qk, const uint32_t* __restrict__ size,
                                 const uint32_t* __restrict__ off, long long n, const int* __restrict__ top_items,
                                 const int* __restrict__ top_counts, int topn, int bits_i, uint64_t* __restrict__ keys,
                                 uint32_t* __restrict__ pay) {
  const int lane = threadIdx.x & 31;
  const long long warps = (long long)gridDim.x * (blockDim.x >> 5);
  for (long long t = ((long long)blockIdx.x * blockDim.x + threadIdx.x) >> 5; t < n; t += warps) {
    const uint32_t m = size[t];
    if (m == 0) continue;
    const unsigned long long k = qk[t];
    const uint64_t q = (uint64_t)(k >> 32) << bits_i;
    const size_t row = (size_t)(unsigned)k * topn;
    const size_t o = off[t];
    for (uint32_t r = lane; r < m; r += 32) {
      keys[o + r] = q | (uint32_t)__ldg(top_items + row + r);
      pay[o + r] = (uint32_t)__ldg(top_counts + row + r);
    }
  }
}

// the lists of one part that rule 3 reads besides QueryFilterDev: the query lists themselves and the white lists
struct CoocLists {
  const unsigned long long* q = nullptr;   // sorted (query << 32 | item) keys of the query lists
  const long long* q_ptr = nullptr;        // [queries + 1]
  const uint8_t* has_wl = nullptr;         // [queries]; nullptr: no query has a white list
  const unsigned long long* wl = nullptr;  // sorted keys of the white lists
  const long long* wl_ptr = nullptr;
};

// pass[e] = 1 at the first entry of each run of equal (query, candidate) keys whose candidate is one of the query's:
// in its white list (if it has one), not in its exclusion list, not one of its own items, and not in its set row
__global__ void cp_pass_kernel(const uint64_t* __restrict__ keys, long long n, int bits_i, CoocLists L, QueryFilterDev f,
                               uint32_t* __restrict__ pass) {
  const long long e = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (e >= n) return;
  const uint64_t k = keys[e];
  bool ok = e == 0 || keys[e - 1] != k;
  if (ok) {
    const int q = (int)(k >> bits_i);
    const unsigned item = (unsigned)(k & ((1ull << bits_i) - 1));
    const unsigned long long qi = ((unsigned long long)(unsigned)q << 32) | item;
    if (L.has_wl && L.has_wl[q]) ok = cp_sorted_has(L.wl, L.wl_ptr[q], L.wl_ptr[q + 1], qi);
    ok = ok && !cp_sorted_has(L.q, L.q_ptr[q], L.q_ptr[q + 1], qi) && !qf_drop(f, q, (int)item);
  }
  pass[e] = ok ? 1u : 0u;
}

// row pos[e] of each passing run head e: the run's summed count in int64, its query and item, and the first sort's
// (key, payload) = (bound - score, row): ascending keys are descending scores
__global__ void cp_rows_kernel(const uint64_t* __restrict__ keys, const uint32_t* __restrict__ pay, long long n, int bits_i,
                               const uint32_t* __restrict__ pass, const uint32_t* __restrict__ pos, uint64_t bound,
                               int* __restrict__ row_q, int* __restrict__ row_item, long long* __restrict__ row_score,
                               uint64_t* __restrict__ skey, uint32_t* __restrict__ sval) {
  const long long e = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (e >= n || !pass[e]) return;
  const uint64_t k = keys[e];
  unsigned long long s = 0;
  for (long long x = e; x < n && keys[x] == k; ++x) s += pay[x];
  const uint32_t r = pos[e];
  row_q[r] = (int)(k >> bits_i);
  row_item[r] = (int)(k & ((1ull << bits_i) - 1));
  row_score[r] = (long long)s;
  skey[r] = bound - s;
  sval[r] = r;
}

// the second sort's (key, payload): the query of each row, in the order of the first sort
__global__ void cp_query_keys_kernel(const uint32_t* __restrict__ perm, long long n, const int* __restrict__ row_q,
                                     uint64_t* __restrict__ key, uint32_t* __restrict__ val) {
  const long long k = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (k >= n) return;
  const uint32_t r = perm[k];
  key[k] = (uint64_t)(unsigned)row_q[r];
  val[k] = r;
}

// one block per query q: its rows are qkey[lo .. hi) of the final order; the first min(topk, hi - lo) are its result,
// the rest of its topk slots are padded with -1 / 0
__global__ void cp_take_kernel(const uint64_t* __restrict__ qkey, const uint32_t* __restrict__ perm, long long n_rows,
                               int topk, const int* __restrict__ row_item, const long long* __restrict__ row_score,
                               int* __restrict__ out_items, long long* __restrict__ out_scores, int* __restrict__ out_count) {
  const int q = blockIdx.x;
  long long lo = 0, hi = n_rows;
  while (lo < hi) {   // first row of q
    const long long mid = (lo + hi) >> 1;
    if (qkey[mid] < (uint64_t)q) lo = mid + 1;
    else hi = mid;
  }
  const long long first = lo;
  hi = n_rows;
  while (lo < hi) {   // first row after q
    const long long mid = (lo + hi) >> 1;
    if (qkey[mid] <= (uint64_t)q) lo = mid + 1;
    else hi = mid;
  }
  const int cnt = (int)min((long long)topk, lo - first);
  for (int r = threadIdx.x; r < topk; r += blockDim.x) {
    const size_t o = (size_t)q * topk + r;
    if (r < cnt) {
      const uint32_t row = perm[first + r];
      out_items[o] = row_item[row];
      out_scores[o] = row_score[row];
    } else {
      out_items[o] = -1;
      out_scores[o] = 0;
    }
  }
  if (threadIdx.x == 0) out_count[q] = cnt;
}

}  // namespace pio
