// assoc_predict.cuh -- the complementary purchase template's predict for a batch of queries (DESIGN.md 4.15.1).
//
// The model's frequent sets form a prefix trie: set s is (set_prefix[s], set_item[s]) with set_item[s] its largest
// item, sets by length and then in lexicographic order of their items.  A condition of a query is a frequent set whose
// items are all in the query, so the walk is bounded by the frequent sets inside each query, not by C(n, k):
//   level 1       the query's distinct frequent items (L: per query, its items sorted by item, each with its first
//                 position in the query), each with its level-1 set
//   level k       every found (k-1)-set s at list index t is extended by its trie children whose item is in L after t,
//                 probing whichever side is shorter with binary searches in the other (ap_count / ap_fill)
//   output        the found sets that have rules: positions rebuilt from the prefix chain (ap_cond), then ordered by
//                 (query, positions ascending) with stable radix passes over exact keys (ap_key + radix_sort_pairs)
// A frontier entry is (set id, index into L); L's index names the query.  Everything is numbered in 32 bits within a
// part: the caller bounds a part's entries below 2^32.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

namespace pio {

// child range [child_lo[p], child_hi[p]) of every set p that is a prefix: the sets with prefix p are contiguous, since
// prefix ids are non-decreasing within a level (checked on the host); s runs over the sets of level >= 2
__global__ void ap_children_kernel(const long long* __restrict__ prefix, long long s0, long long n_sets,
                                   int* __restrict__ child_lo, int* __restrict__ child_hi) {
  const long long s = s0 + (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (s >= n_sets) return;
  const long long p = prefix[s];
  if (s == s0 || prefix[s - 1] != p) child_lo[p] = (int)s;
  if (s + 1 == n_sets || prefix[s + 1] != p) child_hi[p] = (int)(s + 1);
}

// rule range [rule_lo[c], rule_hi[c]) of every cond c (rules grouped by cond, checked on the host)
__global__ void ap_rules_kernel(const long long* __restrict__ rule_cond, long long n_rules, long long* __restrict__ rule_lo,
                                long long* __restrict__ rule_hi) {
  const long long r = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (r >= n_rules) return;
  const long long c = rule_cond[r];
  if (r == 0 || rule_cond[r - 1] != c) rule_lo[c] = r;
  if (r + 1 == n_rules || rule_cond[r + 1] != c) rule_hi[c] = r + 1;
}

// item_set[i] = the level-1 set of item i (-1 before this kernel: not frequent)
__global__ void ap_item_set_kernel(const int* __restrict__ set_item, long long n1, int* __restrict__ item_set) {
  const long long s = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (s < n1) item_set[set_item[s]] = (int)s;
}

// the query of entry e of a part: the last q with q_ptr[q] <= e
__device__ __forceinline__ int ap_query_of(const long long* __restrict__ q_ptr, int nq, long long e) {
  int lo = 0, hi = nq - 1;
  while (lo < hi) {
    const int mid = (lo + hi + 1) >> 1;
    if (q_ptr[mid] <= e) lo = mid;
    else hi = mid - 1;
  }
  return lo;
}

// flag[e] = 1 when entry e names a frequent item (ids outside [0, n_items) are unknown)
__global__ void ap_known_kernel(const int* __restrict__ items, long long n, int n_items,
                                const int* __restrict__ item_set, uint32_t* __restrict__ flag) {
  const long long e = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (e >= n) return;
  const int it = items[e];
  flag[e] = (it >= 0 && it < n_items && item_set[it] >= 0) ? 1u : 0u;
}

// the flagged entries as (query << bits_i | item, position in the query), in entry order
__global__ void ap_entry_keys_kernel(const int* __restrict__ items, const long long* __restrict__ q_ptr, int nq,
                                     long long n, const uint32_t* __restrict__ flag, const uint32_t* __restrict__ at,
                                     int bits_i, uint64_t* __restrict__ key, uint32_t* __restrict__ pos) {
  const long long e = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (e >= n || !flag[e]) return;
  const int q = ap_query_of(q_ptr, nq, e);
  key[at[e]] = ((uint64_t)q << bits_i) | (uint64_t)items[e];
  pos[at[e]] = (uint32_t)(e - q_ptr[q]);
}

// first[u] = 1 where sorted key u starts a run: the first position of a repeated item
__global__ void ap_first_kernel(const uint64_t* __restrict__ key, long long n, uint32_t* __restrict__ first) {
  const long long u = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (u < n) first[u] = (u == 0 || key[u - 1] != key[u]) ? 1u : 0u;
}

// L and the level-1 frontier: one entry per distinct frequent item of a query, sorted by (query, item)
__global__ void ap_list_kernel(const uint64_t* __restrict__ key, const uint32_t* __restrict__ pos, long long n,
                               const uint32_t* __restrict__ first, const uint32_t* __restrict__ at, int bits_i,
                               const int* __restrict__ item_set, int* __restrict__ L_q, int* __restrict__ L_item,
                               uint32_t* __restrict__ L_pos, int* __restrict__ f_set, uint32_t* __restrict__ f_t) {
  const long long u = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (u >= n || !first[u]) return;
  const uint32_t v = at[u];
  const int it = (int)(key[u] & ((1ull << bits_i) - 1));
  L_q[v] = (int)(key[u] >> bits_i);
  L_item[v] = it;
  L_pos[v] = pos[u];
  f_set[v] = item_set[it];
  f_t[v] = v;
}

// [L_start[q], L_end[q]) = query q's entries of L (both zeroed before: a query without frequent items is empty)
__global__ void ap_list_ranges_kernel(const int* __restrict__ L_q, long long n, uint32_t* __restrict__ L_start,
                                      uint32_t* __restrict__ L_end) {
  const long long u = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (u >= n) return;
  const int q = L_q[u];
  if (u == 0 || L_q[u - 1] != q) L_start[q] = (uint32_t)u;
  if (u + 1 == n || L_q[u + 1] != q) L_end[q] = (uint32_t)(u + 1);
}

// first index in a[lo, hi) whose value is >= x
__device__ __forceinline__ uint32_t ap_lower(const int* __restrict__ a, uint32_t lo, uint32_t hi, int x) {
  while (lo < hi) {
    const uint32_t mid = lo + ((hi - lo) >> 1);
    if (a[mid] < x) lo = mid + 1;
    else hi = mid;
  }
  return lo;
}

// The extensions of frontier entry (s, t): the children c of s whose item is in L(t, L_end[q]).  Both sides are sorted
// by item; the shorter one is walked and each of its items looked up in what is left of the other.  emit(c, u) is
// called in ascending item order.
template <class Emit>
__device__ __forceinline__ void ap_extend(int s, uint32_t t, const int* __restrict__ L_q, const int* __restrict__ L_item,
                                          const uint32_t* __restrict__ L_end, const int* __restrict__ child_lo,
                                          const int* __restrict__ child_hi, const int* __restrict__ set_item, Emit emit) {
  uint32_t lo = t + 1;
  const uint32_t hi = L_end[L_q[t]];
  uint32_t c = (uint32_t)child_lo[s];
  const uint32_t c_hi = (uint32_t)child_hi[s];
  if (c_hi - c <= hi - lo) {
    for (; c < c_hi && lo < hi; ++c) {
      const int it = set_item[c];
      lo = ap_lower(L_item, lo, hi, it);
      if (lo < hi && L_item[lo] == it) emit((int)c, lo++);
    }
  } else {
    for (; lo < hi && c < c_hi; ++lo) {
      const int it = L_item[lo];
      c = ap_lower(set_item, c, c_hi, it);
      if (c < c_hi && set_item[c] == it) emit((int)c++, lo);
    }
  }
}

__global__ void ap_count_kernel(const int* __restrict__ f_set, const uint32_t* __restrict__ f_t, long long n,
                                const int* __restrict__ L_q, const int* __restrict__ L_item,
                                const uint32_t* __restrict__ L_end, const int* __restrict__ child_lo,
                                const int* __restrict__ child_hi, const int* __restrict__ set_item,
                                uint32_t* __restrict__ cnt) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  uint32_t k = 0;
  ap_extend(f_set[i], f_t[i], L_q, L_item, L_end, child_lo, child_hi, set_item, [&](int, uint32_t) { ++k; });
  cnt[i] = k;
}

__global__ void ap_fill_kernel(const int* __restrict__ f_set, const uint32_t* __restrict__ f_t, long long n,
                               const int* __restrict__ L_q, const int* __restrict__ L_item,
                               const uint32_t* __restrict__ L_end, const int* __restrict__ child_lo,
                               const int* __restrict__ child_hi, const int* __restrict__ set_item,
                               const uint32_t* __restrict__ off, int* __restrict__ g_set, uint32_t* __restrict__ g_t) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  uint32_t o = off[i];
  ap_extend(f_set[i], f_t[i], L_q, L_item, L_end, child_lo, child_hi, set_item, [&](int c, uint32_t u) {
    g_set[o] = c;
    g_t[o] = u;
    ++o;
  });
}

// has[i] = 1 when frontier entry i's set has rules
__global__ void ap_has_rules_kernel(const int* __restrict__ f_set, long long n, const long long* __restrict__ rule_lo,
                                    const long long* __restrict__ rule_hi, uint32_t* __restrict__ has) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) has[i] = rule_hi[f_set[i]] > rule_lo[f_set[i]] ? 1u : 0u;
}

// Cond at[i] of the level-k entries that have rules: its set and list index, and its k (position, item) pairs in
// ascending position (query order), rebuilt from the prefix chain: each item is found in the query's part of L that
// precedes the entry's own (the items of a set ascend along L).
__global__ void ap_cond_kernel(const int* __restrict__ f_set, const uint32_t* __restrict__ f_t, long long n, int k,
                               const uint32_t* __restrict__ has, const uint32_t* __restrict__ at,
                               const long long* __restrict__ prefix, const int* __restrict__ set_item,
                               const int* __restrict__ L_q, const int* __restrict__ L_item,
                               const uint32_t* __restrict__ L_pos, const uint32_t* __restrict__ L_start,
                               int* __restrict__ c_set, uint32_t* __restrict__ c_t, uint32_t* __restrict__ c_pos,
                               int* __restrict__ c_item) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n || !has[i]) return;
  const uint32_t c = at[i], t = f_t[i];
  const int s = f_set[i];
  c_set[c] = s;
  c_t[c] = t;
  uint32_t* pos = c_pos + (size_t)c * k;
  int* its = c_item + (size_t)c * k;
  const uint32_t lo = L_start[L_q[t]];
  uint32_t u = t;
  long long p = s;
  for (int j = 0; j < k; ++j) {   // insertion in ascending position as the chain is walked (largest item first)
    if (j > 0) u = ap_lower(L_item, lo, u, set_item[p]);
    const uint32_t ps = L_pos[u];
    const int it = L_item[u];
    int m = j;
    for (; m > 0 && pos[m - 1] > ps; --m) {
      pos[m] = pos[m - 1];
      its[m] = its[m - 1];
    }
    pos[m] = ps;
    its[m] = it;
    p = prefix[p];
  }
}

__global__ void ap_iota_kernel(uint32_t* __restrict__ v, long long n) {
  const long long r = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (r < n) v[r] = (uint32_t)r;
}

// key[r] of the cond perm[r] for one LSD pass: fields f0 .. f1 (0 = the query, j >= 1 = the cond's j-th position),
// f0 most significant, bits_q / bits_p wide
__global__ void ap_key_kernel(const uint32_t* __restrict__ perm, long long n, int k, int f0, int f1, int bits_q,
                              int bits_p, const uint32_t* __restrict__ c_t, const int* __restrict__ L_q,
                              const uint32_t* __restrict__ c_pos, uint64_t* __restrict__ key) {
  const long long r = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (r >= n) return;
  const uint32_t c = perm[r];
  uint64_t v = 0;
  for (int f = f0; f <= f1; ++f)
    v = f == 0 ? (uint64_t)L_q[c_t[c]] : (v << bits_p) | c_pos[(size_t)c * k + f - 1];
  key[r] = v;
}

// the level's conds in sorted order: query, items in query order, first rule and rule count min(range, max(num, 0))
__global__ void ap_emit_kernel(const uint32_t* __restrict__ perm, long long n, int k, const int* __restrict__ c_set,
                               const uint32_t* __restrict__ c_t, const int* __restrict__ c_item,
                               const int* __restrict__ L_q, const long long* __restrict__ rule_lo,
                               const long long* __restrict__ rule_hi, const int* __restrict__ num,
                               int* __restrict__ o_q, int* __restrict__ o_item, long long* __restrict__ o_rule,
                               int* __restrict__ o_n) {
  const long long r = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (r >= n) return;
  const uint32_t c = perm[r];
  const int s = c_set[c], q = L_q[c_t[c]];
  o_q[r] = q;
  for (int j = 0; j < k; ++j) o_item[(size_t)r * k + j] = c_item[(size_t)c * k + j];
  const long long lo = rule_lo[s], range = rule_hi[s] - lo;
  const long long want = num[q] > 0 ? num[q] : 0;
  o_rule[r] = lo;
  o_n[r] = (int)(range < want ? range : want);
}

}  // namespace pio
