// assoc.cuh -- association rules of the complementary purchase template (docs/manual/source/templates/
// complementarypurchase/dase.html.md.erb:241-314): buy events -> time-window baskets -> frequent item sets up to
// maxRuleLength -> rules scored by support, confidence and lift, the top maxNumRulesPerCond per condition.
// The rules are stated in tests/assoc_ref.py and DESIGN.md 4.15.  Integer work, HBM-bound: radix sorts, scans and
// run-length counts over (basket, item) and (set, item) keys.
//
//   fold_time_key_kernel, fold_entity_key_kernel (events_fold.cuh) + radix_sort_pairs
//                              stable sort by time (sign bit flipped), then by user: the order is (user, t, event)
//   assoc_basket_head_kernel   a basket starts at a user's first buy and after every gap > basketWindow * 1000 ms
//   assoc_bi_key_kernel        (basket, item) keys; sort + cooc_head / cooc_compact make them distinct
//   assoc_basket_size_kernel   basket sizes; baskets of fewer than minBasketSize items are dropped
//   assoc_kept_kernel          the kept baskets' items (ascending in each basket) and the item counts (level 1)
//   level k >= 2               every occurrence of a frequent (k-1)-set in a basket -- (position of its last item, set
//                              id) -- is extended by each later (larger) frequent item of its basket: key = (set id <<
//                              bits_i) | item.  A sort and a run-length count give each candidate's count; the frequent
//                              ones are numbered in key order, which is the lexicographic order of their items, and
//                              their occurrences feed level k + 1.  A set is counted only when its prefix is frequent,
//                              which drops nothing that could be frequent (count(S) <= count(prefix)).
//   assoc_rule_kernel          per frequent set S, |S| >= 2, and c in S: count(S \ {c}) by binary search in the keys of
//                              level |S| - 1 (from the prefix ids of S when c is not its last item); scores in fp64
//   ranking                    stable sorts by conseq, then -lift, then condition; the first maxNumRulesPerCond of each
//                              condition are kept
// Every count is an integer and every order is a key order: the result is the same from run to run.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include "sort_scan.cuh"

namespace pio {

constexpr int ASSOC_MAX_LEN = 32;    // longest frequent set the rule kernel decodes (the candidate limit keeps sets shorter)
constexpr int ASSOC_RULE_THREADS = 64;

// head[s] = 1 where sorted event s starts a basket: the first buy of its user, or a gap over the window
__global__ void assoc_basket_head_kernel(const uint64_t* __restrict__ ukey, const uint32_t* __restrict__ pay,
                                         const long long* __restrict__ t_ms, long long n, long long window_ms,
                                         uint32_t* __restrict__ head) {
  const long long s = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (s >= n) return;
  head[s] = (s == 0 || ukey[s] != ukey[s - 1] || t_ms[pay[s]] - t_ms[pay[s - 1]] > window_ms) ? 1u : 0u;
}

// (basket, item) of sorted event s; basket = inclusive count of heads - 1
__global__ void assoc_bi_key_kernel(const uint32_t* __restrict__ head, const uint32_t* __restrict__ bscan,
                                    const uint32_t* __restrict__ pay, const int* __restrict__ item, long long n,
                                    int bits_i, uint64_t* __restrict__ key, uint32_t* __restrict__ kpay) {
  const long long s = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (s >= n) return;
  const uint64_t b = (uint64_t)(bscan[s] + head[s] - 1u);
  key[s] = (b << bits_i) | (uint64_t)(uint32_t)item[pay[s]];
  kpay[s] = 0;
}

// at the first distinct entry of every basket: its size, and whether it has at least min_size items
__global__ void assoc_basket_size_kernel(const uint64_t* __restrict__ dk, const uint32_t* __restrict__ bh,
                                         const uint32_t* __restrict__ bord, long long m, int bits_i, int min_size,
                                         uint32_t* __restrict__ keep) {
  const long long e = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (e >= m || !bh[e]) return;
  const uint64_t b = dk[e] >> bits_i;
  long long t = e + 1;
  while (t < m && (dk[t] >> bits_i) == b) ++t;
  keep[bord[e]] = (t - e) >= (long long)min_size ? 1u : 0u;
}

// entries of kept baskets: flag (then scanned into the kept positions) ...
__global__ void assoc_kept_flag_kernel(const uint32_t* __restrict__ bh, const uint32_t* __restrict__ bord,
                                       const uint32_t* __restrict__ keep, long long m, uint32_t* __restrict__ flag) {
  const long long e = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (e < m) flag[e] = keep[bord[e] + bh[e] - 1u];
}
// ... their items and kept-basket numbers, and the item counts of level 1
__global__ void assoc_kept_kernel(const uint64_t* __restrict__ dk, const uint32_t* __restrict__ bh,
                                  const uint32_t* __restrict__ bord, const uint32_t* __restrict__ kord,
                                  const uint32_t* __restrict__ flag, const uint32_t* __restrict__ pos, long long m,
                                  int bits_i, int* __restrict__ k_item, uint32_t* __restrict__ k_basket,
                                  uint32_t* __restrict__ cnt1) {
  const long long e = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (e >= m || !flag[e]) return;
  const int it = (int)(dk[e] & ((1ull << bits_i) - 1ull));
  k_item[pos[e]] = it;
  k_basket[pos[e]] = kord[bord[e] + bh[e] - 1u];
  atomicAdd(cnt1 + it, 1u);
}

// level 1: an item is frequent when it occurs and its count reaches thr (fp64 compare)
__global__ void assoc_l1_flag_kernel(const uint32_t* __restrict__ cnt1, int n_items, double thr,
                                     uint32_t* __restrict__ f1) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n_items) f1[i] = (cnt1[i] > 0u && (double)cnt1[i] >= thr) ? 1u : 0u;
}
__global__ void assoc_l1_emit_kernel(const uint32_t* __restrict__ cnt1, const uint32_t* __restrict__ f1,
                                     const uint32_t* __restrict__ id1, int n_items, uint64_t* __restrict__ keys,
                                     uint32_t* __restrict__ count) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n_items || !f1[i]) return;
  keys[id1[i]] = (uint64_t)i;
  count[id1[i]] = cnt1[i];
}

// the kept entries whose item is frequent: flag, then (after the scan) the pruned baskets and level-1 occurrences
__global__ void assoc_prune_flag_kernel(const int* __restrict__ k_item, const uint32_t* __restrict__ f1, long long m,
                                        uint32_t* __restrict__ flag) {
  const long long e = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (e < m) flag[e] = f1[k_item[e]];
}
__global__ void assoc_prune_kernel(const int* __restrict__ k_item, const uint32_t* __restrict__ k_basket,
                                   const uint32_t* __restrict__ flag, const uint32_t* __restrict__ pos,
                                   const uint32_t* __restrict__ id1, long long m, int* __restrict__ p_item,
                                   uint32_t* __restrict__ p_basket, uint32_t* __restrict__ occ_pos,
                                   uint32_t* __restrict__ occ_id) {
  const long long e = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (e >= m || !flag[e]) return;
  const uint32_t p = pos[e];
  p_item[p] = k_item[e];
  p_basket[p] = k_basket[e];
  occ_pos[p] = p;
  occ_id[p] = id1[k_item[e]];
}
// end[g] = one past the last pruned entry of g's basket (entries of a basket are contiguous)
__global__ void assoc_seg_start_kernel(const uint32_t* __restrict__ p_basket, long long np, uint32_t* __restrict__ hd) {
  const long long g = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (g < np) hd[g] = (g == 0 || p_basket[g] != p_basket[g - 1]) ? 1u : 0u;
}
__global__ void assoc_seg_pos_kernel(const uint32_t* __restrict__ hd, const uint32_t* __restrict__ sidx, long long np,
                                     uint32_t* __restrict__ seg_start) {
  const long long g = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (g < np && hd[g]) seg_start[sidx[g]] = (uint32_t)g;
}
__global__ void assoc_seg_end_kernel(const uint32_t* __restrict__ hd, const uint32_t* __restrict__ sidx,
                                     const uint32_t* __restrict__ seg_start, long long np, uint32_t* __restrict__ end) {
  const long long g = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (g < np) end[g] = seg_start[sidx[g] + hd[g]];   // seg_start[n_seg] = np
}

// level k: occurrence o extends by the entries after its last item in its basket; *total (zeroed by the caller) gets
// their sum in 64 bits, so that the uint32 scan of ext is used only once the total is known to fit
__global__ void assoc_ext_kernel(const uint32_t* __restrict__ occ_pos, const uint32_t* __restrict__ end, long long no,
                                 uint32_t* __restrict__ ext, unsigned long long* __restrict__ total) {
  const long long o = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  unsigned long long r = 0;
  if (o < no) {
    const uint32_t g = occ_pos[o];
    r = end[g] - g - 1u;
    ext[o] = (uint32_t)r;
  }
#pragma unroll
  for (int d = 16; d > 0; d >>= 1) r += __shfl_down_sync(0xffffffffu, r, d);
  if ((threadIdx.x & 31) == 0 && r) atomicAdd(total, r);
}
__global__ void assoc_expand_kernel(const uint32_t* __restrict__ occ_pos, const uint32_t* __restrict__ occ_id,
                                    const uint32_t* __restrict__ ext, const uint32_t* __restrict__ off, long long no,
                                    const int* __restrict__ p_item, int bits_i, uint64_t* __restrict__ key,
                                    uint32_t* __restrict__ pay, uint32_t* __restrict__ cand_pos) {
  const long long o = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (o >= no) return;
  const uint32_t g = occ_pos[o], r = ext[o], base = off[o];
  const uint64_t hi = (uint64_t)occ_id[o] << bits_i;
  for (uint32_t t = 0; t < r; ++t) {
    key[base + t] = hi | (uint64_t)(uint32_t)p_item[g + 1u + t];
    pay[base + t] = base + t;
    cand_pos[base + t] = g + 1u + t;
  }
}
// at the head of every run of equal candidate keys: its count, and whether it is frequent
__global__ void assoc_runs_kernel(const uint64_t* __restrict__ key, const uint32_t* __restrict__ hf,
                                  const uint32_t* __restrict__ rix, long long nc, double thr,
                                  uint64_t* __restrict__ rkey, uint32_t* __restrict__ rcnt, uint32_t* __restrict__ rf) {
  const long long s = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (s >= nc || !hf[s]) return;
  long long t = s + 1;
  while (t < nc && !hf[t]) ++t;
  const uint32_t r = rix[s];
  rkey[r] = key[s];
  rcnt[r] = (uint32_t)(t - s);
  rf[r] = (double)(t - s) >= thr ? 1u : 0u;
}
__global__ void assoc_level_emit_kernel(const uint64_t* __restrict__ rkey, const uint32_t* __restrict__ rcnt,
                                        const uint32_t* __restrict__ rf, const uint32_t* __restrict__ rid, long long nr,
                                        uint64_t* __restrict__ keys, uint32_t* __restrict__ count) {
  const long long r = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (r >= nr || !rf[r]) return;
  keys[rid[r]] = rkey[r];
  count[rid[r]] = rcnt[r];
}
// sorted candidate s: flag = its set is frequent (scanned into the next occurrence list), then the occurrence
__global__ void assoc_occ_flag_kernel(const uint32_t* __restrict__ hf, const uint32_t* __restrict__ rix,
                                      const uint32_t* __restrict__ rf, long long nc, uint32_t* __restrict__ flag) {
  const long long s = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (s < nc) flag[s] = rf[rix[s] + hf[s] - 1u];
}
__global__ void assoc_occ_kernel(const uint32_t* __restrict__ pay, const uint32_t* __restrict__ cand_pos,
                                 const uint32_t* __restrict__ hf, const uint32_t* __restrict__ rix,
                                 const uint32_t* __restrict__ rid, const uint32_t* __restrict__ flag,
                                 const uint32_t* __restrict__ pos, long long nc, uint32_t* __restrict__ occ_pos,
                                 uint32_t* __restrict__ occ_id) {
  const long long s = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (s >= nc || !flag[s]) return;
  occ_pos[pos[s]] = cand_pos[pay[s]];
  occ_id[pos[s]] = rid[rix[s] + hf[s] - 1u];
}

// ---- rules ----------------------------------------------------------------------------------------------------------
// The frequent sets of every level, on the device: keys[l] (ascending; level 1: the item, level l > 1: (id of the
// prefix at level l - 1) << bits_i | last item), count[l], n[l], and base[l] = global id of the first set of level l.
struct AssocLevels {
  const uint64_t* keys[ASSOC_MAX_LEN + 1];
  const uint32_t* count[ASSOC_MAX_LEN + 1];
  uint32_t n[ASSOC_MAX_LEN + 1];
  uint32_t base[ASSOC_MAX_LEN + 1];
};

// index of key x in keys[0, n) (present by construction)
__device__ __forceinline__ uint32_t assoc_find(const uint64_t* __restrict__ keys, uint32_t n, uint64_t x) {
  uint32_t lo = 0, hi = n;
  while (hi - lo > 1u) {
    const uint32_t mid = lo + (hi - lo) / 2u;
    if (keys[mid] <= x) lo = mid; else hi = mid;
  }
  return lo;
}

struct AssocRuleArgs {
  int k, bits_i;
  double t;                    // T, the number of transactions
  double min_conf, min_lift;
};

// Per frequent set of level k (thread): its items a[0..k) (ascending) and prefix ids pid[l] (id of a[0..l) at level
// l), decoded into shared memory.  For c = a[j]: the condition's id comes from pid[j] extended by a[j+1..k) through
// levels j+1 .. k-1 (level 1 looked up by item when j = 0).  Mode 0 counts the passing rules of each set (and their
// 64-bit total), mode 1 writes them at off[set].
template <int MODE>
__global__ void __launch_bounds__(ASSOC_RULE_THREADS)
assoc_rule_kernel(AssocLevels L, AssocRuleArgs a, uint32_t* __restrict__ npass, unsigned long long* __restrict__ total,
                  const uint32_t* __restrict__ off, uint32_t* __restrict__ r_cond, int* __restrict__ r_conseq,
                  double* __restrict__ r_sup, double* __restrict__ r_conf, double* __restrict__ r_lift) {
  __shared__ uint32_t s_item[ASSOC_MAX_LEN][ASSOC_RULE_THREADS];
  __shared__ uint32_t s_pid[ASSOC_MAX_LEN + 1][ASSOC_RULE_THREADS];
  const int tx = threadIdx.x, k = a.k;
  const long long set = (long long)blockIdx.x * blockDim.x + tx;
  const uint32_t imask = (1u << a.bits_i) - 1u;
  unsigned long long passed = 0;
  if (set < L.n[k]) {
    uint32_t id = (uint32_t)set;
    s_pid[k][tx] = id;
    for (int l = k; l >= 2; --l) {
      const uint64_t key = L.keys[l][id];
      s_item[l - 1][tx] = (uint32_t)(key & imask);
      id = (uint32_t)(key >> a.bits_i);
      s_pid[l - 1][tx] = id;
    }
    s_item[0][tx] = (uint32_t)L.keys[1][id];
    const uint32_t cs = L.count[k][set];
    const double sup = (double)cs / a.t;
    uint32_t w = off ? off[set] : 0u;
    for (int j = 0; j < k; ++j) {
      uint32_t cid;
      int l;
      if (j == 0) {
        cid = assoc_find(L.keys[1], L.n[1], s_item[1][tx]);
        l = 2;
      } else {
        cid = s_pid[j][tx];
        l = j + 1;
      }
      for (int t = (j == 0 ? 2 : j + 1); t < k; ++t, ++l)
        cid = assoc_find(L.keys[l], L.n[l], ((uint64_t)cid << a.bits_i) | s_item[t][tx]);
      const uint32_t c = s_item[j][tx];
      const uint32_t cc = L.count[k - 1][cid];
      const uint32_t c1 = L.count[1][assoc_find(L.keys[1], L.n[1], c)];
      const double conf = (double)cs / (double)cc;
      const double lift = conf / ((double)c1 / a.t);
      if (conf >= a.min_conf && lift >= a.min_lift) {
        if (MODE == 1) {
          r_cond[w] = L.base[k - 1] + cid;
          r_conseq[w] = (int)c;
          r_sup[w] = sup;
          r_conf[w] = conf;
          r_lift[w] = lift;
          ++w;
        }
        ++passed;
      }
    }
    if (MODE == 0) npass[set] = (uint32_t)passed;
  }
  if (MODE == 0) {
#pragma unroll
    for (int d = 16; d > 0; d >>= 1) passed += __shfl_down_sync(0xffffffffu, passed, d);
    if ((tx & 31) == 0 && passed) atomicAdd(total, passed);
  }
}

// ranking keys of the rules (payload: rule index), one stable pass each: conseq, then -lift, then condition
__global__ void assoc_rank_key_kernel(const uint32_t* __restrict__ pay, long long nr, int which,
                                      const uint32_t* __restrict__ r_cond, const int* __restrict__ r_conseq,
                                      const double* __restrict__ r_lift, uint64_t* __restrict__ key,
                                      uint32_t* __restrict__ kpay) {
  const long long s = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (s >= nr) return;
  const uint32_t r = pay ? pay[s] : (uint32_t)s;
  uint64_t k;
  if (which == 0) {
    k = (uint64_t)(uint32_t)r_conseq[r];
  } else if (which == 1) {
    // order-preserving bits of -lift: ascending keys = descending lift
    uint64_t u = (uint64_t)__double_as_longlong(-r_lift[r]);
    k = (u >> 63) ? ~u : (u | (1ull << 63));
  } else {
    k = (uint64_t)r_cond[r];
  }
  key[s] = k;
  kpay[s] = r;
}
// rules per condition (the conditions' rule runs are contiguous once sorted)
__global__ void assoc_cond_count_kernel(const uint64_t* __restrict__ key, long long nr, uint32_t* __restrict__ ccount) {
  const long long s = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (s < nr) atomicAdd(ccount + key[s], 1u);
}
__global__ void assoc_cond_keep_kernel(const uint32_t* __restrict__ ccount, long long ns, uint32_t max_per_cond,
                                       uint32_t* __restrict__ kcount) {
  const long long c = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (c < ns) kcount[c] = min(ccount[c], max_per_cond);
}
__global__ void assoc_take_kernel(const uint64_t* __restrict__ key, const uint32_t* __restrict__ pay, long long nr,
                                  const uint32_t* __restrict__ cstart, const uint32_t* __restrict__ kstart,
                                  uint32_t max_per_cond, const uint32_t* __restrict__ r_cond,
                                  const int* __restrict__ r_conseq, const double* __restrict__ r_sup,
                                  const double* __restrict__ r_conf, const double* __restrict__ r_lift,
                                  uint32_t* __restrict__ o_cond, int* __restrict__ o_conseq, double* __restrict__ o_sup,
                                  double* __restrict__ o_conf, double* __restrict__ o_lift) {
  const long long s = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (s >= nr) return;
  const uint32_t c = (uint32_t)key[s], rank = (uint32_t)s - cstart[c];
  if (rank >= max_per_cond) return;
  const uint32_t o = kstart[c] + rank, r = pay[s];
  o_cond[o] = r_cond[r];
  o_conseq[o] = r_conseq[r];
  o_sup[o] = r_sup[r];
  o_conf[o] = r_conf[r];
  o_lift[o] = r_lift[r];
}

}  // namespace pio
