// eval_folds.cuh -- the k-fold split of the recommendation template's evaluation on the device
// (examples/scala-parallel-recommendation/blacklist-items/src/main/scala/DataSource.scala readEval: rating e goes to the
// test set of fold e % kFold and to the training set of every other fold), and the ranking-metric counts of Evaluation.scala
// (PrecisionAtK, PositiveCount) over a fold's top-N result.
//
// All work is on global indices: the user and item columns of all ratings are encoded once (ids_encode.cuh); a fold's
// BiMap.stringInt is then a renumbering of the global ids that train in it, in order of first training occurrence
// (DESIGN.md 4.11).  Per global id the split keeps e1 = its first position and e2 = its first position in a fold other
// than fold(e1); the first training occurrence in fold f is e1 when fold(e1) != f, else e2 (none when e2 does not exist).
// Positions are int32: the caller guarantees n < 2^31.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include "sort_scan.cuh"

namespace pio {
namespace evf {

constexpr int NONE = 0x7fffffff;   // "no such position"
constexpr int RC_WARPS = 8;        // rank_counts_kernel: queries (warps) per CTA

// e1[g[e]] = min e (e1 preset to NONE)
__global__ void first_pos_kernel(const int* __restrict__ g, long long n, int* __restrict__ e1) {
  const long long e = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (e < n) atomicMin(&e1[g[e]], (int)e);
}

// e2[g[e]] = min e with fold(e) != fold(e1[g[e]]) (e2 preset to NONE)
__global__ void second_pos_kernel(const int* __restrict__ g, long long n, int k_fold, const int* __restrict__ e1,
                                  int* __restrict__ e2) {
  const long long e = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (e >= n) return;
  const int id = g[e];
  if ((int)(e % k_fold) != e1[id] % k_fold) atomicMin(&e2[id], (int)e);
}

__device__ __forceinline__ int first_train_pos(const int* e1, const int* e2, int id, int k_fold, int f) {
  const int a = e1[id];
  return a % k_fold != f ? a : e2[id];
}

// flag[t] = 1 at the first training occurrence t of every id that trains in fold f (flag preset to 0)
__global__ void train_flag_kernel(const int* __restrict__ e1, const int* __restrict__ e2, int n_ids, int k_fold, int f,
                                  uint32_t* __restrict__ flag) {
  const int id = blockIdx.x * blockDim.x + threadIdx.x;
  if (id >= n_ids) return;
  const int t = first_train_pos(e1, e2, id, k_fold, f);
  if (t != NONE) flag[t] = 1u;
}

// scan = exclusive scan of train_flag_kernel's flags: loc[id] = the fold-local index of id (-1: not in the fold's
// training set), l2g[loc] = id
__global__ void train_index_kernel(const int* __restrict__ e1, const int* __restrict__ e2, int n_ids, int k_fold, int f,
                                   const uint32_t* __restrict__ scan, int* __restrict__ loc, int* __restrict__ l2g) {
  const int id = blockIdx.x * blockDim.x + threadIdx.x;
  if (id >= n_ids) return;
  const int t = first_train_pos(e1, e2, id, k_fold, f);
  if (t == NONE) {
    loc[id] = -1;
    return;
  }
  const int l = (int)scan[t];
  loc[id] = l;
  l2g[l] = id;
}

// The training COO of fold f in rating order: rating e (e % k_fold != f) is entry e - |{j < e : j % k_fold == f}|
__global__ void train_coo_kernel(const int* __restrict__ gu, const int* __restrict__ gi, const double* __restrict__ r,
                                 long long n, int k_fold, int f, const int* __restrict__ uloc,
                                 const int* __restrict__ iloc, int* __restrict__ ou, int* __restrict__ oi,
                                 float* __restrict__ ov) {
  const long long e = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (e >= n || (int)(e % k_fold) == f) return;
  const long long p = e - (e + k_fold - 1 - f) / k_fold;
  ou[p] = uloc[gu[e]];
  oi[p] = iloc[gi[e]];
  ov[p] = (float)r[e];   // round to nearest, as numpy's astype(float32)
}

// Test rating t of fold f is rating f + t * k_fold, t < m.  qfirst[u] = the first test rating of user u (preset NONE).
__global__ void query_first_kernel(const int* __restrict__ gu, int k_fold, int f, long long m, int* __restrict__ qfirst) {
  const long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (t < m) atomicMin(&qfirst[gu[f + t * k_fold]], (int)t);
}

// flag[t] = 1 where t is its user's first test rating (m + 1 entries: flag[m] = 0)
__global__ void query_flag_kernel(const int* __restrict__ gu, int k_fold, int f, long long m,
                                  const int* __restrict__ qfirst, uint32_t* __restrict__ flag) {
  const long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (t < m) flag[t] = qfirst[gu[f + t * k_fold]] == (int)t ? 1u : 0u;
  else if (t == m) flag[t] = 0u;
}

// scan = exclusive scan of query_flag_kernel's flags (query index at a query's first test rating).  Per query q:
// q2g[q] = its global user, qtrain[q] = its fold-local training index or -1.  Per test rating t the sort key
// (query << ibits | global item) with payload t.
__global__ void query_index_kernel(const int* __restrict__ gu, const int* __restrict__ gi, int k_fold, int f, long long m,
                                   const int* __restrict__ qfirst, const uint32_t* __restrict__ scan,
                                   const int* __restrict__ uloc, int ibits, int* __restrict__ q2g,
                                   int* __restrict__ qtrain, uint64_t* __restrict__ key, uint32_t* __restrict__ val) {
  const long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= m) return;
  const long long e = f + t * k_fold;
  const int u = gu[e];
  const int t0 = qfirst[u];
  const uint32_t q = scan[t0];
  if (t0 == (int)t) {
    q2g[q] = u;
    qtrain[q] = uloc[u];
  }
  key[t] = ((uint64_t)q << ibits) | (uint32_t)gi[e];
  val[t] = (uint32_t)t;
}

// Over the test ratings sorted by (query, global item), stable: raw[s] = the rating in slot s, qptr[q] = the first slot
// of query q (qptr[nq] = m), dflag[s] = 1 where a (query, item) run starts (m + 1 entries: dflag[m] = 0)
__global__ void test_slots_kernel(const uint64_t* __restrict__ ks, const uint32_t* __restrict__ vs, long long m,
                                  int k_fold, int f, const double* __restrict__ r, int ibits, int nq,
                                  double* __restrict__ raw, int* __restrict__ qptr, uint32_t* __restrict__ dflag) {
  const long long s = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (s > m) return;
  if (s == m) {
    qptr[nq] = (int)m;
    dflag[m] = 0u;
    return;
  }
  raw[s] = r[f + (long long)vs[s] * k_fold];
  const uint64_t q = ks[s] >> ibits;
  if (s == 0 || (ks[s - 1] >> ibits) != q) qptr[q] = (int)s;
  dflag[s] = (s == 0 || ks[s] != ks[s - 1]) ? 1u : 0u;
}

// dscan = exclusive scan of the run flags: distinct (query, item) d = dscan[s] at the head s of its run, ditem[d] = the
// global item, dmax[d] = the largest of its ratings
__global__ void test_distinct_kernel(const uint64_t* __restrict__ ks, long long m, const double* __restrict__ raw,
                                     const uint32_t* __restrict__ dscan, uint64_t imask, int* __restrict__ ditem,
                                     double* __restrict__ dmax) {
  const long long s = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (s >= m || (s > 0 && ks[s] == ks[s - 1])) return;
  const uint32_t d = dscan[s];
  double mx = raw[s];
  for (long long j = s + 1; j < m && ks[j] == ks[s]; ++j) mx = fmax(mx, raw[j]);
  ditem[d] = (int)(ks[s] & imask);
  dmax[d] = mx;
}

// dptr[q] = the first distinct slot of query q (q <= nq; qptr[nq] = m and dscan[m] = number of distinct pairs)
__global__ void test_dptr_kernel(const int* __restrict__ qptr, const uint32_t* __restrict__ dscan, int nq,
                                 int* __restrict__ dptr) {
  const int q = blockIdx.x * blockDim.x + threadIdx.x;
  if (q <= nq) dptr[q] = (int)dscan[qptr[q]];
}

// One warp per query q of a fold's top-N result (items: fold-local indices, nq x num; count[q] valid entries):
//   hits[q] = how many of the first min(k, count[q]) items have a largest test rating >= thr
//   npos[q] = distinct test items with largest rating >= thr;  nraw[q] = test ratings >= thr
// Predicted items are looked up by global id (il2g) in the query's sorted distinct items.
__global__ void __launch_bounds__(32 * RC_WARPS)
rank_counts_kernel(const int* __restrict__ items, const int* __restrict__ count, int num, int nq, int k, double thr,
                   const int* __restrict__ il2g, const int* __restrict__ qptr, const double* __restrict__ raw,
                   const int* __restrict__ dptr, const int* __restrict__ ditem, const double* __restrict__ dmax,
                   int* __restrict__ hits, int* __restrict__ npos, int* __restrict__ nraw) {
  const int q = blockIdx.x * RC_WARPS + (threadIdx.x >> 5);
  const int lane = threadIdx.x & 31;
  if (q >= nq) return;
  int c_raw = 0, c_pos = 0, c_hit = 0;
  for (int s = qptr[q] + lane; s < qptr[q + 1]; s += 32) c_raw += raw[s] >= thr;
  const int d0 = dptr[q], d1 = dptr[q + 1];
  for (int d = d0 + lane; d < d1; d += 32) c_pos += dmax[d] >= thr;
  const int kk = min(k, min(count[q], num));
  for (int j = lane; j < kk; j += 32) {
    const int it = il2g[items[(long long)q * num + j]];
    int lo = d0, hi = d1;   // first slot with ditem >= it
    while (lo < hi) {
      const int mid = (lo + hi) >> 1;
      if (ditem[mid] < it) lo = mid + 1;
      else hi = mid;
    }
    c_hit += lo < d1 && ditem[lo] == it && dmax[lo] >= thr;
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    c_raw += __shfl_xor_sync(0xffffffffu, c_raw, o);
    c_pos += __shfl_xor_sync(0xffffffffu, c_pos, o);
    c_hit += __shfl_xor_sync(0xffffffffu, c_hit, o);
  }
  if (lane == 0) {
    hits[q] = c_hit;
    npos[q] = c_pos;
    nraw[q] = c_raw;
  }
}

}  // namespace evf
}  // namespace pio
