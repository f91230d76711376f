// cooc.cuh -- item co-occurrence counts of the similarproduct template's CooccurrenceAlgorithm
// (examples/scala-parallel-similarproduct/multi-events-multi-algos/src/main/scala/CooccurrenceAlgorithm.scala:72-105):
//   userItem = (user, item).distinct;  cooccurrences = userItem.join(userItem).filter(item1 < item2) -> count per pair;
//   per item the n co-occurring items with the largest counts.
// Integer work, HBM-bound: radix sorts, scans and run-length counts over (user, item) and (item1, item2) keys.  Ties in the
// per-item ranking are unspecified in the reference (sortBy on a groupByKey order); here: larger count first, then the
// smaller item index.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include "sort_scan.cuh"

namespace pio {

__global__ void cooc_keys_kernel(const int* __restrict__ u, const int* __restrict__ it, long long n, int bits_i,
                                 uint64_t* __restrict__ keys, uint32_t* __restrict__ pay) {
  const long long e = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (e < n) {
    keys[e] = ((uint64_t)(uint32_t)u[e] << bits_i) | (uint64_t)(uint32_t)it[e];
    pay[e] = (uint32_t)e;
  }
}
// flag = 1 at the first element of every run of equal keys
__global__ void cooc_head_kernel(const uint64_t* __restrict__ keys, long long n, uint32_t* __restrict__ flag) {
  const long long e = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (e < n) flag[e] = (e == 0 || keys[e] != keys[e - 1]) ? 1u : 0u;
}
// compact the distinct (user, item) keys
__global__ void cooc_compact_kernel(const uint64_t* __restrict__ keys, const uint32_t* __restrict__ flag,
                                    const uint32_t* __restrict__ pos, long long n, uint64_t* __restrict__ out) {
  const long long e = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (e < n && flag[e]) out[pos[e]] = keys[e];
}
// per distinct element: is it the first of its user?  (user = key >> bits_i)
__global__ void cooc_user_head_kernel(const uint64_t* __restrict__ dk, long long m, int bits_i, uint32_t* __restrict__ uflag) {
  const long long e = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (e < m) uflag[e] = (e == 0 || (dk[e] >> bits_i) != (dk[e - 1] >> bits_i)) ? 1u : 0u;
}
// element e (rank r inside its user's sorted item list) pairs with the r earlier items of the user: npairs[e] = r.
// *total (zeroed by the caller) receives the sum of the ranks in 64 bits: the uint32 scan of the ranks wraps once a
// user has more than ~92 700 distinct items, so the pair count must not be read back from it.
__global__ void cooc_rank_kernel(const uint64_t* __restrict__ dk, long long m, int bits_i, uint32_t* __restrict__ rank,
                                 unsigned long long* __restrict__ total) {
  const long long e = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  unsigned long long r = 0;
  if (e < m) {
    const uint64_t usr = dk[e] >> bits_i;
    long long s = e;
    while (s > 0 && (dk[s - 1] >> bits_i) == usr) --s;   // users' lists are short next to m; templates view <= 1e3 items
    r = (unsigned long long)(e - s);
    rank[e] = (uint32_t)r;
  }
#pragma unroll
  for (int d = 16; d > 0; d >>= 1) r += __shfl_down_sync(0xffffffffu, r, d);
  if ((threadIdx.x & 31) == 0 && r) atomicAdd(total, r);
}
__global__ void cooc_pairs_kernel(const uint64_t* __restrict__ dk, const uint32_t* __restrict__ rank,
                                  const uint32_t* __restrict__ off, long long m, int bits_i, uint64_t* __restrict__ pk,
                                  uint32_t* __restrict__ pp) {
  const long long e = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (e >= m) return;
  const uint64_t imask = (1ull << bits_i) - 1ull;
  const uint64_t hi_item = dk[e] & imask;               // the list is sorted: earlier items are smaller
  const uint32_t r = rank[e];
  for (uint32_t t = 0; t < r; ++t) {
    const uint64_t lo_item = dk[e - r + t] & imask;
    pk[off[e] + t] = (lo_item << bits_i) | hi_item;     // item1 < item2
    pp[off[e] + t] = 0;
  }
}
// runs of equal pair keys -> (pair, count); both directions as ranking keys: item | (CMAX - count) | other
__global__ void cooc_runs_kernel(const uint64_t* __restrict__ pk, const uint32_t* __restrict__ flag,
                                 const uint32_t* __restrict__ pos, long long np, int bits_i, int bits_c,
                                 uint64_t* __restrict__ rk, uint32_t* __restrict__ rp) {
  const long long e = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (e >= np || !flag[e]) return;
  long long t = e + 1;
  while (t < np && !flag[t]) ++t;
  const uint64_t cnt = (uint64_t)(t - e);
  const uint64_t imask = (1ull << bits_i) - 1ull, cmax = (1ull << bits_c) - 1ull;
  const uint64_t a = pk[e] >> bits_i, b = pk[e] & imask;
  const uint64_t inv = cmax - (cnt > cmax ? cmax : cnt);
  const uint32_t o = pos[e];
  rk[2 * (size_t)o] = (a << (bits_c + bits_i)) | (inv << bits_i) | b;
  rk[2 * (size_t)o + 1] = (b << (bits_c + bits_i)) | (inv << bits_i) | a;
  rp[2 * (size_t)o] = (uint32_t)cnt;
  rp[2 * (size_t)o + 1] = (uint32_t)cnt;
}
// sorted ranking keys -> the first topn entries of every item
__global__ void cooc_take_kernel(const uint64_t* __restrict__ rk, const uint32_t* __restrict__ rp, long long n2, int bits_i,
                                 int bits_c, int topn, int* __restrict__ out_item, int* __restrict__ out_count,
                                 int* __restrict__ out_n) {
  const long long e = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (e >= n2) return;
  const uint64_t item = rk[e] >> (bits_c + bits_i);
  long long s = e;
  int r = 0;
  while (s > 0 && (rk[s - 1] >> (bits_c + bits_i)) == item && r < topn) { --s; ++r; }
  if (r >= topn) return;
  out_item[(size_t)item * topn + r] = (int)(rk[e] & ((1ull << bits_i) - 1ull));
  out_count[(size_t)item * topn + r] = (int)rp[e];
  atomicMax(&out_n[item], r + 1);
}

}  // namespace pio
