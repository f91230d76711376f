// serve_merge.cuh -- the similarproduct template's Serving.serve over a batch
// (examples/scala-parallel-similarproduct/multi-events-multi-algos/src/main/scala/Serving.scala:29-69, DESIGN.md 4.13):
// every algorithm's list of a query z-scored with numpy's mean and sample deviation, the values summed per item, the
// items ordered by sum descending (ties: first appearance) and cut at the query's num.  Per part of a batch:
//   one thread per (query, algorithm) list: mean and deviation -> one warp per list: (query << bits_i | item, entry)
//   pairs and the entry's value, in (query, algorithm, position) order -> stable radix sort by (query, item) -> one sum
//   per run, in entry order, kept at the run's first entry -> those entries compacted in entry order (first appearance)
//   -> stable sorts by the sum's descending key, then by query -> first min(num, topk) of each query.
// Every floating-point operation is an explicitly rounded __d*_rn intrinsic, so that nothing is contracted into an FMA
// and each value is the one numpy and Python compute.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include "sort_scan.cuh"

namespace pio {

constexpr int SM_PW_BLOCK = 128;   // numpy's PW_BLOCKSIZE
constexpr int SM_PW_DEPTH = 32;    // splits of a list of fewer than 2^31 values: at most 24 deep

// numpy's pairwise_sum of f(0) .. f(n - 1): a plain loop from 0.0 below 8 values, eight accumulators combined
// ((r0 + r1) + (r2 + r3)) + ((r4 + r5) + (r6 + r7)) plus an in-order tail up to SM_PW_BLOCK values
template <class F>
__device__ __forceinline__ double sm_pw_leaf(const F& f, long long lo, long long n) {
  if (n < 8) {
    double res = 0.0;
    for (long long i = 0; i < n; ++i) res = __dadd_rn(res, f(lo + i));
    return res;
  }
  double r[8];
#pragma unroll
  for (int k = 0; k < 8; ++k) r[k] = f(lo + k);
  long long i = 8;
  for (; i < n - (n % 8); i += 8)
#pragma unroll
    for (int k = 0; k < 8; ++k) r[k] = __dadd_rn(r[k], f(lo + i + k));
  double res = __dadd_rn(__dadd_rn(__dadd_rn(r[0], r[1]), __dadd_rn(r[2], r[3])),
                         __dadd_rn(__dadd_rn(r[4], r[5]), __dadd_rn(r[6], r[7])));
  for (; i < n; ++i) res = __dadd_rn(res, f(lo + i));
  return res;
}

// ... and above SM_PW_BLOCK the sum of its two halves, split at n / 2 rounded down to a multiple of 8: the recursion
// walked with an explicit stack of the pending left halves
__device__ __forceinline__ long long sm_pw_split(long long n) {
  const long long h = n / 2;
  return h - h % 8;
}
template <class F>
__device__ double sm_pairwise(const F& f, long long n) {
  long long node_lo[SM_PW_DEPTH], node_n[SM_PW_DEPTH];
  double left[SM_PW_DEPTH];
  bool right[SM_PW_DEPTH];
  int sp = 0;
  long long lo = 0, m = n;
  for (;;) {
    while (m > SM_PW_BLOCK) {   // descend into the left half
      node_lo[sp] = lo, node_n[sp] = m, right[sp] = false;
      ++sp;
      m = sm_pw_split(m);
    }
    double v = sm_pw_leaf(f, lo, m);
    for (;;) {   // climb: a finished left half starts its right half, a finished right half completes its node
      if (sp == 0) return v;
      const int t = sp - 1;
      if (!right[t]) {
        left[t] = v;
        right[t] = true;
        const long long h = sm_pw_split(node_n[t]);
        lo = node_lo[t] + h, m = node_n[t] - h;
        break;
      }
      v = __dadd_rn(left[t], v);
      --sp;
    }
  }
}

// the algorithms' rows of one part on the device: algorithm a's rows are items[a] / scores[a] with width w[a]
struct MergeLists {
  const int* const* items;
  const double* const* scores;
  const int* w;
  int n_algos;
};

// one thread per list l = query * n_algos + algorithm of cnt[l] entries: Serving.serve's mean and sample deviation,
// or (num == 1: not standardised) mean = 0, sd = -1
__global__ void sm_stats_kernel(MergeLists L, const uint32_t* __restrict__ cnt, long long n_lists,
                                const int* __restrict__ num, double* __restrict__ mean, double* __restrict__ sd) {
  const long long l = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (l >= n_lists) return;
  const int q = (int)(l / L.n_algos), a = (int)(l % L.n_algos);
  if (num[q] == 1) {
    mean[l] = 0.0, sd[l] = -1.0;
    return;
  }
  const long long n = cnt[l];
  const double* s = L.scores[a] + (size_t)q * L.w[a];
  const double mu = n ? __ddiv_rn(__dadd_rn(0.0, sm_pairwise([&](long long i) { return s[i]; }, n)), (double)n) : 0.0;
  double dev = 0.0;
  if (n > 1) {
    const double ss = __dadd_rn(0.0, sm_pairwise([&](long long i) {
      const double x = __dsub_rn(s[i], mu);
      return __dmul_rn(x, x);
    }, n));
    dev = __dsqrt_rn(__ddiv_rn(ss, (double)(n - 1)));
  }
  mean[l] = mu, sd[l] = dev;
}

// one warp per list: entry e = off[l] + p of list l gets the key (query << bits_i | item), the payload e and its value
// z[e] -- the score itself when not standardised, 0 when the deviation is 0, else (score - mean) / deviation
__global__ void sm_entries_kernel(MergeLists L, const uint32_t* __restrict__ cnt, const uint32_t* __restrict__ off,
                                  long long n_lists, const double* __restrict__ mean, const double* __restrict__ sd,
                                  int bits_i, uint64_t* __restrict__ key, uint32_t* __restrict__ val,
                                  double* __restrict__ z) {
  const int lane = threadIdx.x & 31;
  const long long warps = (long long)gridDim.x * (blockDim.x >> 5);
  for (long long l = ((long long)blockIdx.x * blockDim.x + threadIdx.x) >> 5; l < n_lists; l += warps) {
    const uint32_t n = cnt[l];
    if (n == 0) continue;
    const int q = (int)(l / L.n_algos), a = (int)(l % L.n_algos);
    const size_t row = (size_t)q * L.w[a];
    const double mu = mean[l], dev = sd[l];
    const uint64_t qk = (uint64_t)q << bits_i;
    for (uint32_t p = lane; p < n; p += 32) {
      const double s = L.scores[a][row + p];
      const uint32_t e = off[l] + p;
      key[e] = qk | (uint32_t)L.items[a][row + p];
      val[e] = e;
      z[e] = dev < 0.0 ? s : dev == 0.0 ? 0.0 : __ddiv_rn(__dsub_rn(s, mu), dev);
    }
  }
}

// sorted position t heading a run of equal (query, item) keys: the run's values summed 0.0 + z0 + z1 + ... in entry
// (algorithm, position) order, stored at the run's first entry e = val[t], which head[e] marks
__global__ void sm_sum_kernel(const uint64_t* __restrict__ key, const uint32_t* __restrict__ val, long long n,
                              const double* __restrict__ z, uint32_t* __restrict__ head, uint64_t* __restrict__ head_key,
                              double* __restrict__ head_sum) {
  const long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= n) return;
  const uint64_t k = key[t];
  if (t > 0 && key[t - 1] == k) return;
  double s = 0.0;
  for (long long x = t; x < n && key[x] == k; ++x) s = __dadd_rn(s, z[val[x]]);
  const uint32_t e = val[t];
  head[e] = 1u;
  head_key[e] = k;
  head_sum[e] = s;
}

// an fp64 value as a 64-bit key whose ascending order is the value's descending order; -0.0 and +0.0 share a key, as
// they compare equal in Python's sort
__device__ __forceinline__ uint64_t sm_desc_key(double v) {
  uint64_t b = (uint64_t)__double_as_longlong(v == 0.0 ? 0.0 : v);
  b = (b >> 63) ? ~b : (b | 0x8000000000000000ull);
  return ~b;
}

// entry e heading a run becomes row pos[e]: rows are in entry order, which is (query, first appearance) order
__global__ void sm_rows_kernel(const uint32_t* __restrict__ head, const uint32_t* __restrict__ pos, long long n,
                               const uint64_t* __restrict__ head_key, const double* __restrict__ head_sum,
                               uint64_t* __restrict__ row_key, double* __restrict__ row_sum, uint64_t* __restrict__ skey,
                               uint32_t* __restrict__ sval) {
  const long long e = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (e >= n || !head[e]) return;
  const uint32_t r = pos[e];
  row_key[r] = head_key[e];
  row_sum[r] = head_sum[e];
  skey[r] = sm_desc_key(head_sum[e]);
  sval[r] = r;
}

// the second sort's (key, payload): the query of each row, in the order of the first sort
__global__ void sm_query_keys_kernel(const uint32_t* __restrict__ perm, long long n, const uint64_t* __restrict__ row_key,
                                     int bits_i, uint64_t* __restrict__ key, uint32_t* __restrict__ val) {
  const long long k = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (k >= n) return;
  const uint32_t r = perm[k];
  key[k] = row_key[r] >> bits_i;
  val[k] = r;
}

// one block per query q: its rows are qkey[lo .. hi) of the final order; the first min(num[q], topk, hi - lo) are its
// result, the rest of its topk slots are padded with -1 / 0
__global__ void sm_take_kernel(const uint64_t* __restrict__ qkey, const uint32_t* __restrict__ perm, long long n_rows,
                               int topk, const int* __restrict__ num, const uint64_t* __restrict__ row_key, int bits_i,
                               const double* __restrict__ row_sum, int* __restrict__ out_items,
                               double* __restrict__ out_scores, int* __restrict__ out_count) {
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
  const int cnt = (int)min((long long)min(topk, num[q]), lo - first);
  for (int r = threadIdx.x; r < topk; r += blockDim.x) {
    const size_t o = (size_t)q * topk + r;
    if (r < cnt) {
      const uint32_t row = perm[first + r];
      out_items[o] = (int)(row_key[row] & ((1ull << bits_i) - 1));
      out_scores[o] = row_sum[row];
    } else {
      out_items[o] = -1;
      out_scores[o] = 0.0;
    }
  }
  if (threadIdx.x == 0) out_count[q] = cnt;
}

}  // namespace pio
