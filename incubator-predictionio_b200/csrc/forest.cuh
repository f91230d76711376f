// forest.cuh -- RandomForest classifier kernels (pio_rf_train / pio_rf_predict; rules: tests/forest_ref.py, DESIGN 4.10):
//   sample_flag_kernel + scan + sample_compact_kernel   the split sample (keyed Bernoulli draw per row)
//   sample_keys_kernel + radix sort + run_head_kernel + scan + run_compact_kernel
//                                                       per feature: the distinct sampled values and where their runs
//                                                       start; only the runs go to the host (forest_splits.h thresholds)
//   bin_kernel<BinT>                                    x (fp64, row-major) -> uint8 / uint16 bin codes
//   hist_kernel<BinT, SMEM>                             per level, the hot path: bootstrap-weighted class counts per
//                                                       (node slot, feature of its subset, bin, class)
//   select_kernel                                       per node slot: the best split over its features and thresholds
//   update_kernel<BinT>                                 each row's node -> its child, or retired at a leaf
//   predict_kernel                                      one thread per row: every tree's walk and the vote
// Counts are integers, so every sum is independent of the order of its atomics: the forest is the same on every run.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include "forest_splits.h"

namespace pio {
namespace rf {

constexpr int THREADS = 256;
constexpr int SEL_WARPS = 8;

struct Cdf {
  double v[RF_POISSON_N];
};

__global__ void sample_flag_kernel(int64_t n, uint64_t base, double frac, uint32_t* __restrict__ flag) {
  const int64_t r = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (r < n) flag[r] = rf_sampled(base, (uint64_t)r, frac) ? 1u : 0u;
}
__global__ void sample_compact_kernel(const uint32_t* __restrict__ flag, const uint32_t* __restrict__ pos, int64_t n,
                                      uint32_t* __restrict__ rows) {
  const int64_t r = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (r < n && flag[r]) rows[pos[r]] = (uint32_t)r;
}

// order-preserving 64-bit key of a double; -0.0 counts as 0.0
__device__ __forceinline__ uint64_t key_of(double v) {
  const uint64_t b = (uint64_t)__double_as_longlong(v == 0.0 ? 0.0 : v);
  return (b >> 63) ? ~b : (b | (1ull << 63));
}
// rows == nullptr: every row
__global__ void sample_keys_kernel(const double* __restrict__ x, int F, int f, const uint32_t* __restrict__ rows,
                                   int64_t m, uint64_t* __restrict__ key, uint32_t* __restrict__ val) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= m) return;
  const int64_t r = rows ? (int64_t)rows[i] : i;
  key[i] = key_of(x[r * F + f]);
  val[i] = (uint32_t)i;
}
__global__ void run_head_kernel(const uint64_t* __restrict__ k, int64_t m, uint32_t* __restrict__ head) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < m) head[i] = (i == 0 || k[i] != k[i - 1]) ? 1u : 0u;
}
__global__ void run_compact_kernel(const uint64_t* __restrict__ k, const uint32_t* __restrict__ head,
                                   const uint32_t* __restrict__ pos, int64_t m, uint64_t* __restrict__ rkey,
                                   uint32_t* __restrict__ rstart) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < m && head[i]) rkey[pos[i]] = k[i], rstart[pos[i]] = (uint32_t)i;
}

// bin code = the number of the feature's thresholds below x (a row goes left of threshold j iff its bin <= j);
// thresholds of feature f are thr[off[f] .. off[f + 1]), staged in shared memory when `staged`
template <typename BinT>
__global__ void __launch_bounds__(THREADS) bin_kernel(const double* __restrict__ x, int64_t n, int F,
                                                      const double* __restrict__ thr, const int* __restrict__ off,
                                                      int staged, BinT* __restrict__ bins) {
  extern __shared__ double s_thr[];
  const double* T = thr;
  if (staged) {
    for (int i = threadIdx.x; i < off[F]; i += blockDim.x) s_thr[i] = thr[i];
    __syncthreads();
    T = s_thr;
  }
  const int64_t total = n * F;
  for (int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; e < total; e += (int64_t)gridDim.x * blockDim.x) {
    const int f = (int)(e % F);
    const double v = x[e];
    const int base = __ldg(off + f);
    int lo = base, hi = __ldg(off + f + 1);
    while (lo < hi) {
      const int mid = (lo + hi) >> 1;
      if (T[mid] < v) lo = mid + 1;
      else hi = mid;
    }
    bins[e] = (BinT)(lo - base);
  }
}

struct HistArgs {
  const uint8_t* cls;          // [n] class of each row
  const void* bins;            // [n][F]
  const int* node;             // [G][n] node slot of each (tree of the group, row), -1 at a leaf
  const uint64_t* bag;         // [G] bag stream base per tree, nullptr: every weight is 1
  const int* sub;              // [S][K] subset features of each slot
  unsigned long long* hist;    // [slots of the chunk][K][NB][C], slot hist_base first
  int64_t n;
  int F, G, K, NB, C;
  int s0, s1, hist_base;       // this pass counts slots [s0, s1) ...
  int g0, g1;                  // ... which belong to trees [g0, g1] of the group (slots are ordered by tree)
  Cdf cdf;
};

// One pass over the rows for the node slots [s0, s1); only the node ids of the trees owning those slots are read.
// SMEM: counts go to a shared-memory histogram of those slots and are flushed with one 64-bit atomic per nonzero entry;
// otherwise straight to the global histogram.
template <typename BinT, bool SMEM>
__global__ void __launch_bounds__(THREADS) hist_kernel(const HistArgs a) {
  extern __shared__ uint32_t sh[];
  const int per_slot = a.K * a.NB * a.C;
  const int size = SMEM ? (a.s1 - a.s0) * per_slot : 0;
  if (SMEM) {
    for (int i = threadIdx.x; i < size; i += blockDim.x) sh[i] = 0u;
    __syncthreads();
  }
  const BinT* bins = static_cast<const BinT*>(a.bins);
  for (int64_t r = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; r < a.n; r += (int64_t)gridDim.x * blockDim.x) {
    const int c = a.cls[r];
    const BinT* br = bins + r * a.F;
    for (int g = a.g0; g <= a.g1; ++g) {
      const int s = a.node[(int64_t)g * a.n + r];
      if (s < a.s0 || s >= a.s1) continue;
      const uint32_t w = a.bag ? (uint32_t)rf_bag_weight(a.cdf.v, a.bag[g], (uint64_t)r) : 1u;
      if (w == 0) continue;
      const int* sf = a.sub + (int64_t)s * a.K;
      for (int kk = 0; kk < a.K; ++kk) {
        const int b = br[__ldg(sf + kk)];
        if (SMEM) atomicAdd(&sh[((s - a.s0) * a.K + kk) * a.NB * a.C + b * a.C + c], w);
        else atomicAdd(&a.hist[(((int64_t)(s - a.hist_base) * a.K + kk) * a.NB + b) * a.C + c], (unsigned long long)w);
      }
    }
  }
  if (SMEM) {
    __syncthreads();
    unsigned long long* dst = a.hist + (int64_t)(a.s0 - a.hist_base) * per_slot;
    for (int i = threadIdx.x; i < size; i += blockDim.x)
      if (sh[i]) atomicAdd(dst + i, (unsigned long long)sh[i]);
  }
}

// gini / entropy of class counts, class by class with explicit roundings (no contraction), as tests/forest_ref.py
// and MLlib's calculate() accumulate them
__device__ __forceinline__ double imp_step(double imp, long long cnt, double n, int kind) {
  const double f = __ddiv_rn((double)cnt, n);
  if (kind == RF_GINI) return __dsub_rn(imp, __dmul_rn(f, f));
  if (cnt == 0) return imp;
  return __dsub_rn(imp, __dmul_rn(f, __ddiv_rn(log(f), 0x1.62e42fefa39efp-1)));
}

__device__ __forceinline__ long long warp_incl_scan64(long long v) {
  const int lane = threadIdx.x & 31;
#pragma unroll
  for (int d = 1; d < 32; d <<= 1) {
    const long long t = __shfl_up_sync(0xffffffffu, v, d);
    if (lane >= d) v += t;
  }
  return v;
}

struct SelArgs {
  const unsigned long long* hist;   // as HistArgs
  const int* sub;                   // [S][K]
  const int* n_thr;                 // [F] thresholds per feature
  double* gain;                     // [S] best gain (-inf: no valid split)
  int* best;                        // [S][2] subset position and threshold index of the best split
  long long* left;                  // [S][C] class counts left of the best split
  long long* total;                 // [S][C] class counts of the node
  int K, NB, C, kind, hist_base, s0;
};

// One block per node slot, one warp per feature of its subset (strided).  A warp walks its feature's thresholds 32 at a
// time: a warp scan over the bins gives each lane's left counts, the gain is fp64 with explicit roundings, and a warp
// argmax keeps the first maximum.  The block then keeps the first maximum over the features (subset order = feature
// order).  A candidate is valid when nL >= 1, nR >= 1 and gain >= 0.
__global__ void __launch_bounds__(SEL_WARPS * 32) select_kernel(const SelArgs a) {
  __shared__ unsigned long long s_tot[RF_MAX_CLASSES];
  __shared__ long long s_carry[SEL_WARPS][RF_MAX_CLASSES];
  __shared__ double s_gain[SEL_WARPS];
  __shared__ int s_kk[SEL_WARPS], s_j[SEL_WARPS];
  const int s = a.s0 + blockIdx.x;
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
  const int C = a.C, NB = a.NB;
  const unsigned long long* H = a.hist + (int64_t)(s - a.hist_base) * a.K * NB * C;
  if (threadIdx.x < C) s_tot[threadIdx.x] = 0ull;
  __syncthreads();
  for (int i = threadIdx.x; i < NB * C; i += blockDim.x) atomicAdd(&s_tot[i % C], H[i]);   // subset feature 0
  __syncthreads();
  long long ntot = 0;
  double ip = RF_GINI == a.kind ? 1.0 : 0.0;
  for (int c = 0; c < C; ++c) ntot += (long long)s_tot[c];
  const double n = (double)(ntot > 0 ? ntot : 1);
  if (ntot > 0)
    for (int c = 0; c < C; ++c) ip = imp_step(ip, (long long)s_tot[c], n, a.kind);
  else ip = 0.0;
  double bg = -INFINITY;
  int bkk = -1, bj = -1;
  for (int kk = w; kk < a.K; kk += SEL_WARPS) {
    const int nthr = a.n_thr[a.sub[(int64_t)s * a.K + kk]];
    const unsigned long long* Hk = H + (int64_t)kk * NB * C;
    for (int c = lane; c < C; c += 32) s_carry[w][c] = 0;
    long long carry_n = 0;
    __syncwarp();
    for (int j0 = 0; j0 < nthr; j0 += 32) {
      const int j = j0 + lane;
      long long vb = 0;
      if (j < NB)
        for (int c = 0; c < C; ++c) vb += (long long)Hk[(int64_t)j * C + c];
      const long long nl = carry_n + warp_incl_scan64(vb);
      carry_n = __shfl_sync(0xffffffffu, nl, 31);
      const long long nr = ntot - nl;
      const double dl = (double)(nl > 0 ? nl : 1), dr = (double)(nr > 0 ? nr : 1);
      double il = RF_GINI == a.kind ? 1.0 : 0.0, ir = il;
      for (int c = 0; c < C; ++c) {
        const long long v = j < NB ? (long long)Hk[(int64_t)j * C + c] : 0;
        const long long lc = s_carry[w][c] + warp_incl_scan64(v);
        __syncwarp();
        if (lane == 31) s_carry[w][c] = lc;
        __syncwarp();
        il = imp_step(il, lc, dl, a.kind);
        ir = imp_step(ir, (long long)s_tot[c] - lc, dr, a.kind);
      }
      const double g = __dsub_rn(__dsub_rn(ip, __dmul_rn(__ddiv_rn((double)nl, n), il)),
                                 __dmul_rn(__ddiv_rn((double)nr, n), ir));
      const bool ok = j < nthr && nl >= 1 && nr >= 1 && g >= 0.0;
      double cg = ok ? g : -INFINITY;
      int cj = ok ? j : -1;
#pragma unroll
      for (int d = 16; d >= 1; d >>= 1) {          // argmax, ties to the smaller threshold index
        const double og = __shfl_xor_sync(0xffffffffu, cg, d);
        const int oj = __shfl_xor_sync(0xffffffffu, cj, d);
        if (og > cg || (og == cg && oj >= 0 && (cj < 0 || oj < cj))) cg = og, cj = oj;
      }
      if (cj >= 0 && cg > bg) bg = cg, bkk = kk, bj = cj;    // earlier thresholds and features win ties
    }
  }
  if (lane == 0) s_gain[w] = bg, s_kk[w] = bkk, s_j[w] = bj;
  __syncthreads();
  if (threadIdx.x == 0) {
    double g = -INFINITY;
    int kk = -1, j = -1;
    for (int q = 0; q < SEL_WARPS; ++q)
      if (s_kk[q] >= 0 && (s_gain[q] > g || (s_gain[q] == g && s_kk[q] < kk))) g = s_gain[q], kk = s_kk[q], j = s_j[q];
    a.gain[s] = g;
    a.best[2 * s] = kk;
    a.best[2 * s + 1] = j;
    s_kk[0] = kk, s_j[0] = j;
  }
  __syncthreads();
  const int kk = s_kk[0], j = s_j[0];
  for (int c = threadIdx.x; c < C; c += blockDim.x) {
    long long lc = 0;
    if (kk >= 0)
      for (int b = 0; b <= j; ++b) lc += (long long)H[((int64_t)kk * NB + b) * C + c];
    a.left[(int64_t)s * C + c] = lc;
    a.total[(int64_t)s * C + c] = (long long)s_tot[c];
  }
}

// upd[s] = (feature, threshold index, left child slot, right child slot) of slot s; feature -1: the node is a leaf;
// a child slot of -1: that child is a leaf
template <typename BinT>
__global__ void update_kernel(int* __restrict__ node, int64_t n, int G, const BinT* __restrict__ bins, int F,
                              const int4* __restrict__ upd) {
  const int64_t total = n * G;
  for (int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; e < total; e += (int64_t)gridDim.x * blockDim.x) {
    const int s = node[e];
    if (s < 0) continue;
    const int4 u = upd[s];
    if (u.x < 0) {
      node[e] = -1;
      continue;
    }
    const int64_t r = e % n;
    node[e] = (int)bins[r * F + u.x] <= u.y ? u.z : u.w;
  }
}

__global__ void root_kernel(int* __restrict__ node, int64_t n, int G) {
  const int64_t total = n * G;
  for (int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; e < total; e += (int64_t)gridDim.x * blockDim.x)
    node[e] = (int)(e / n);
}

// one thread per row: walk every tree (x[f] <= threshold goes left), vote; ties to the smaller class.  Votes live in
// shared memory, [class][thread].
__global__ void __launch_bounds__(128) predict_kernel(const int* __restrict__ tree_off, int T, const int* __restrict__ feat,
                                                      const double* __restrict__ thr, const int* __restrict__ left,
                                                      const int* __restrict__ right, const int* __restrict__ pred, int C,
                                                      const double* __restrict__ x, int64_t n, int F,
                                                      int* __restrict__ out) {
  extern __shared__ int votes[];
  const int64_t r = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  for (int c = 0; c < C; ++c) votes[c * blockDim.x + threadIdx.x] = 0;
  if (r >= n) return;
  const double* xr = x + r * F;
  for (int t = 0; t < T; ++t) {
    int i = __ldg(tree_off + t);
    for (int f = __ldg(feat + i); f >= 0; f = __ldg(feat + i)) i = xr[f] <= __ldg(thr + i) ? __ldg(left + i) : __ldg(right + i);
    ++votes[__ldg(pred + i) * blockDim.x + threadIdx.x];
  }
  int best = 0;
  for (int c = 1; c < C; ++c)
    if (votes[c * blockDim.x + threadIdx.x] > votes[best * blockDim.x + threadIdx.x]) best = c;
  out[r] = best;
}

}  // namespace rf
}  // namespace pio
