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
// The regressor (pio_rf_train_regressor; rules: tests/forest_reg_ref.py, DESIGN 4.16) shares the sample, binning, level
// loop and layout, and differs in two places, each behind one switch:
//   statistics  hist_kernel<BinT, SMEM, true>           per (slot, feature, bin): sum w, sum w yq (int128) and
//                                                       sum w yq^2 (uint128) of the quantised labels yq
//               select_var_kernel                       per (slot, subset feature): variance gains along the bins, or
//                                                       along the categories sorted by centroid
//   split kind  cat_centroid_kernel + cat_rank_kernel   the stable centroid order of categorical features too wide to
//                                                       order inside select_var_kernel
//               update_kernel<BinT, true>               a categorical split moves rows by a bit mask of its left
//                                                       categories
//               predict_reg_kernel                      the mean over trees, with category membership per node
// Counts and label sums are integers, so every sum is independent of the order of its atomics: the forest is the same on
// every run.
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
// thresholds of feature f are thr[off[f] .. off[f + 1]), staged in shared memory when `staged`.  A feature with
// arity[f] > 0 is categorical and its bin is trunc(x).
template <typename BinT>
__global__ void __launch_bounds__(THREADS) bin_kernel(const double* __restrict__ x, int64_t n, int F,
                                                      const double* __restrict__ thr, const int* __restrict__ off,
                                                      int staged, BinT* __restrict__ bins,
                                                      const int* __restrict__ arity = nullptr) {
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
    if (arity && __ldg(arity + f) > 0) {                  // categorical: trunc(v), checked to be in [0, arity)
      bins[e] = (BinT)(int)v;
      continue;
    }
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
  const long long* yq;         // [n] quantised label of each row (hist_kernel<.., true>), else nullptr
};

constexpr int VAR_WORDS = 5;   // a variance entry: sum w, sum w yq (lo, hi), sum w yq^2 (lo, hi), 64-bit words

// 128-bit add with 64-bit atomics: the low word first, its carry (from the returned old value) into the high word
__device__ __forceinline__ void atomic_add128(unsigned long long* p, unsigned long long lo, unsigned long long hi) {
  const unsigned long long old = atomicAdd(p, lo);
  atomicAdd(p + 1, hi + (old + lo < old ? 1ull : 0ull));
}
__device__ __forceinline__ void var_add(unsigned long long* e, unsigned long long w, unsigned long long s_lo,
                                        unsigned long long s_hi, unsigned long long q_lo, unsigned long long q_hi) {
  atomicAdd(e, w);
  atomic_add128(e + 1, s_lo, s_hi);
  atomic_add128(e + 3, q_lo, q_hi);
}

// One pass over the rows for the node slots [s0, s1); only the node ids of the trees owning those slots are read.
// SMEM: counts go to a shared-memory histogram of those slots and are flushed with one 64-bit atomic per nonzero entry;
// otherwise straight to the global histogram.
// VAR: variance entries of VAR_WORDS 64-bit words (shared-memory ones too) from the rows' quantised labels.
template <typename BinT, bool SMEM, bool VAR = false>
__global__ void __launch_bounds__(THREADS) hist_kernel(const HistArgs a) {
  if constexpr (VAR) {
    extern __shared__ unsigned long long shv[];
    const int per_slot = a.K * a.NB * VAR_WORDS;
    const int size = SMEM ? (a.s1 - a.s0) * per_slot : 0;
    if (SMEM) {
      for (int i = threadIdx.x; i < size; i += blockDim.x) shv[i] = 0ull;
      __syncthreads();
    }
    const BinT* bins = static_cast<const BinT*>(a.bins);
    for (int64_t r = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; r < a.n; r += (int64_t)gridDim.x * blockDim.x) {
      const long long y = a.yq[r];
      const unsigned long long ay = (unsigned long long)(y < 0 ? -y : y);
      const unsigned long long sq_lo = ay * ay, sq_hi = __umul64hi(ay, ay);      // yq^2 < 2^89
      const BinT* br = bins + r * a.F;
      for (int g = a.g0; g <= a.g1; ++g) {
        const int s = a.node[(int64_t)g * a.n + r];
        if (s < a.s0 || s >= a.s1) continue;
        const unsigned long long w = a.bag ? (unsigned long long)rf_bag_weight(a.cdf.v, a.bag[g], (uint64_t)r) : 1ull;
        if (w == 0) continue;
        const long long wy = (long long)w * y;                                   // |w yq| <= 2^48
        const unsigned long long s_lo = (unsigned long long)wy, s_hi = wy < 0 ? ~0ull : 0ull;
        const unsigned long long q_lo = sq_lo * w, q_hi = sq_hi * w + __umul64hi(sq_lo, w);
        const int* sf = a.sub + (int64_t)s * a.K;
#pragma unroll 1
        for (int kk = 0; kk < a.K; ++kk) {
          const int b = br[__ldg(sf + kk)];
          if (SMEM) var_add(&shv[(((s - a.s0) * a.K + kk) * a.NB + b) * VAR_WORDS], w, s_lo, s_hi, q_lo, q_hi);
          else var_add(&a.hist[(((int64_t)(s - a.hist_base) * a.K + kk) * a.NB + b) * VAR_WORDS], w, s_lo, s_hi, q_lo,
                       q_hi);
        }
      }
    }
    if (SMEM) {
      __syncthreads();
      unsigned long long* dst = a.hist + (int64_t)(a.s0 - a.hist_base) * per_slot;
      for (int e = threadIdx.x; e < size / VAR_WORDS; e += blockDim.x) {
        const unsigned long long* v = shv + e * VAR_WORDS;
        if (v[0]) var_add(dst + e * VAR_WORDS, v[0], v[1], v[2], v[3], v[4]);
      }
    }
    return;
  }
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
// a child slot of -1: that child is a leaf.  CAT: a slot with mask_off[s] >= 0 splits on categories, and a row goes left
// iff bit `bin` of mask[mask_off[s] ..] is set.
template <typename BinT, bool CAT = false>
__global__ void update_kernel(int* __restrict__ node, int64_t n, int G, const BinT* __restrict__ bins, int F,
                              const int4* __restrict__ upd, const long long* __restrict__ mask_off = nullptr,
                              const uint32_t* __restrict__ mask = nullptr) {
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
    if constexpr (CAT) {
      const int b = (int)bins[r * F + u.x];
      const long long mo = mask_off[s];
      const bool go = mo < 0 ? b <= u.y : ((mask[mo + (b >> 5)] >> (b & 31)) & 1u) != 0u;
      node[e] = go ? u.z : u.w;
    } else {
      node[e] = (int)bins[r * F + u.x] <= u.y ? u.z : u.w;
    }
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

// ---- regressor: variance statistics and categorical splits (tests/forest_reg_ref.py) ---------------------------------
constexpr int CAT_SMEM_ARITY = 2048;   // categorical features up to this arity are ordered inside select_var_kernel
constexpr int RANK_TILE = 2048;        // centroids per shared-memory tile of cat_rank_kernel

typedef unsigned __int128 u128;

// correctly rounded (to nearest, ties to even) conversions of 128-bit integers, as Python's float(int): the top 64
// bits with a sticky bit for the rest, then an exact power-of-two scale
__device__ __forceinline__ double u128_to_f64(u128 x) {
  const unsigned long long hi = (unsigned long long)(x >> 64);
  if (hi == 0) return __ull2double_rn((unsigned long long)x);
  const int lz = __clzll((long long)hi);
  const u128 y = x << lz;
  const unsigned long long top = (unsigned long long)(y >> 64) | ((unsigned long long)y != 0 ? 1ull : 0ull);
  return __dmul_rn(__ull2double_rn(top), __longlong_as_double((long long)(1023 + 64 - lz) << 52));
}
__device__ __forceinline__ double s128_to_f64(u128 x) {      // x: two's complement
  return (x >> 127) ? -u128_to_f64((u128)0 - x) : u128_to_f64(x);
}

// integer statistics of a set of rows; their fp64 form W = float(w), S = float(s) 2^-s, Q = float(q) 2^-2s
struct VarStat {
  unsigned long long w;
  u128 s, q;
};
__device__ __forceinline__ VarStat var_load(const unsigned long long* e) {
  VarStat v;
  v.w = e[0];
  v.s = ((u128)e[2] << 64) | e[1];
  v.q = ((u128)e[4] << 64) | e[3];
  return v;
}
__device__ __forceinline__ void var_store(unsigned long long* e, const VarStat& v) {
  e[0] = v.w, e[1] = (unsigned long long)v.s, e[2] = (unsigned long long)(v.s >> 64);
  e[3] = (unsigned long long)v.q, e[4] = (unsigned long long)(v.q >> 64);
}
__device__ __forceinline__ VarStat var_sum(const VarStat& a, const VarStat& b) { return {a.w + b.w, a.s + b.s, a.q + b.q}; }
__device__ __forceinline__ VarStat var_diff(const VarStat& a, const VarStat& b) { return {a.w - b.w, a.s - b.s, a.q - b.q}; }

// Variance.calculate: (Q - S * S / W) / W, 0 for an empty node; explicit roundings, no contraction
__device__ __forceinline__ double var_impurity(const VarStat& v, double scale1, double scale2) {
  if (v.w == 0) return 0.0;
  const double W = __ull2double_rn(v.w), S = __dmul_rn(s128_to_f64(v.s), scale1), Q = __dmul_rn(u128_to_f64(v.q), scale2);
  return __ddiv_rn(__dsub_rn(Q, __ddiv_rn(__dmul_rn(S, S), W)), W);
}
// a category's centroid: its mean label, Double.MaxValue without rows
__device__ __forceinline__ double var_centroid(const unsigned long long* e, double scale1) {
  const VarStat v = var_load(e);
  if (v.w == 0) return 1.7976931348623157e308;
  return __ddiv_rn(__dmul_rn(s128_to_f64(v.s), scale1), __ull2double_rn(v.w));
}

__device__ __forceinline__ VarStat var_shfl_up(const VarStat& v, int d) {
  VarStat o;
  o.w = __shfl_up_sync(0xffffffffu, v.w, d);
  const unsigned long long sl = __shfl_up_sync(0xffffffffu, (unsigned long long)v.s, d);
  const unsigned long long sh = __shfl_up_sync(0xffffffffu, (unsigned long long)(v.s >> 64), d);
  const unsigned long long ql = __shfl_up_sync(0xffffffffu, (unsigned long long)v.q, d);
  const unsigned long long qh = __shfl_up_sync(0xffffffffu, (unsigned long long)(v.q >> 64), d);
  o.s = ((u128)sh << 64) | sl;
  o.q = ((u128)qh << 64) | ql;
  return o;
}

struct VarSelArgs {
  const unsigned long long* hist;  // [slots of the chunk][K][NB][VAR_WORDS], slot hist_base first
  const int* sub;                  // [S][K]
  const int* n_thr;                // [F] thresholds per feature
  const int* arity;                // [F] categories per feature, 0: continuous
  uint32_t* order;                 // [slots of the chunk][K][NB] categories in split order (categorical features)
  double* gain;                    // [S][K] best gain of each subset feature (-inf: no valid split)
  int* best;                       // [S][K] its candidate index
  unsigned long long* left;        // [S][K][VAR_WORDS] statistics left of it
  unsigned long long* total;       // [S][VAR_WORDS] statistics of the node
  double scale1, scale2;           // 2^-s, 2^-2s
  int K, NB, hist_base, s0;
};

// One block per (node slot, subset feature): block slot * K + feature position.  The feature's M entries in split order (bins 0 .. n_thr for a continuous
// feature; for a categorical one its categories stably sorted by centroid, ranked here from shared memory when
// arity <= CAT_SMEM_ARITY, else read from `order` as cat_rank_kernel left it) are scanned 256 at a time with exact
// integer prefix sums; candidate j (< M - 1) splits after position j.  The block keeps the first maximum of the valid
// gains (nL >= 1, nR >= 1, gain >= 0); the host picks the first maximum over the features.
__global__ void __launch_bounds__(SEL_WARPS * 32) select_var_kernel(const VarSelArgs a) {
  __shared__ double s_cen[CAT_SMEM_ARITY];
  __shared__ unsigned long long s_red[SEL_WARPS][VAR_WORDS];
  __shared__ double s_g[SEL_WARPS];
  __shared__ int s_j[SEL_WARPS];
  const int s = a.s0 + (int)(blockIdx.x / a.K), kk = (int)(blockIdx.x % a.K);
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5, NT = SEL_WARPS * 32;
  const int f = a.sub[(int64_t)s * a.K + kk], ar = a.arity[f];
  const int M = ar > 0 ? ar : a.n_thr[f] + 1;
  const int64_t base = ((int64_t)(s - a.hist_base) * a.K + kk) * a.NB;
  const unsigned long long* H = a.hist + base * VAR_WORDS;
  uint32_t* ord = a.order ? a.order + base : nullptr;
  if (ar > 0 && ar <= CAT_SMEM_ARITY) {
    for (int c = threadIdx.x; c < ar; c += NT) s_cen[c] = var_centroid(H + (int64_t)c * VAR_WORDS, a.scale1);
    __syncthreads();
    for (int c = threadIdx.x; c < ar; c += NT) {
      const double me = s_cen[c];
      int rank = 0;
      for (int j = 0; j < ar; ++j) rank += (s_cen[j] < me || (s_cen[j] == me && j < c)) ? 1 : 0;
      ord[rank] = (uint32_t)c;
    }
    __syncthreads();
  }
  // the node's statistics
  VarStat tot{0ull, 0, 0};
  for (int p = threadIdx.x; p < M; p += NT) tot = var_sum(tot, var_load(H + (int64_t)p * VAR_WORDS));
  for (int d = 16; d >= 1; d >>= 1) {
    VarStat o;
    o.w = __shfl_xor_sync(0xffffffffu, tot.w, d);
    const unsigned long long sl = __shfl_xor_sync(0xffffffffu, (unsigned long long)tot.s, d);
    const unsigned long long sh = __shfl_xor_sync(0xffffffffu, (unsigned long long)(tot.s >> 64), d);
    const unsigned long long ql = __shfl_xor_sync(0xffffffffu, (unsigned long long)tot.q, d);
    const unsigned long long qh = __shfl_xor_sync(0xffffffffu, (unsigned long long)(tot.q >> 64), d);
    o.s = ((u128)sh << 64) | sl;
    o.q = ((u128)qh << 64) | ql;
    tot = var_sum(tot, o);
  }
  if (lane == 0) var_store(s_red[w], tot);
  __syncthreads();
  tot = VarStat{0ull, 0, 0};
  for (int q = 0; q < SEL_WARPS; ++q) tot = var_sum(tot, var_load(s_red[q]));
  __syncthreads();
  const double ip = var_impurity(tot, a.scale1, a.scale2);
  const double n = tot.w > 0 ? __ull2double_rn(tot.w) : 1.0;
  const bool cat = ar > 0;
  VarStat carry{0ull, 0, 0}, bl{0ull, 0, 0};
  double bg = -INFINITY;
  int bj = -1;
  for (int p0 = 0; p0 < M; p0 += NT) {
    const int p = p0 + threadIdx.x;
    VarStat v{0ull, 0, 0};
    if (p < M) v = var_load(H + (int64_t)(cat ? (int)ord[p] : p) * VAR_WORDS);
#pragma unroll
    for (int d = 1; d < 32; d <<= 1) {
      const VarStat t = var_shfl_up(v, d);
      if (lane >= d) v = var_sum(v, t);
    }
    if (lane == 31) var_store(s_red[w], v);
    __syncthreads();
    VarStat pre = carry;
    for (int q = 0; q < w; ++q) pre = var_sum(pre, var_load(s_red[q]));
    VarStat next = carry;
    for (int q = 0; q < SEL_WARPS; ++q) next = var_sum(next, var_load(s_red[q]));
    __syncthreads();
    const VarStat L = var_sum(pre, v), R = var_diff(tot, L);
    if (p < M - 1 && L.w >= 1 && R.w >= 1) {
      const double il = var_impurity(L, a.scale1, a.scale2), ir = var_impurity(R, a.scale1, a.scale2);
      const double g = __dsub_rn(__dsub_rn(ip, __dmul_rn(__ddiv_rn(__ull2double_rn(L.w), n), il)),
                                 __dmul_rn(__ddiv_rn(__ull2double_rn(R.w), n), ir));
      if (g >= 0.0 && g > bg) bg = g, bj = p, bl = L;        // a thread's positions rise: the first maximum
    }
    carry = next;
  }
  // the block's first maximum: the larger gain, ties to the smaller position
  double cg = bg;
  int cj = bj;
#pragma unroll
  for (int d = 16; d >= 1; d >>= 1) {
    const double og = __shfl_xor_sync(0xffffffffu, cg, d);
    const int oj = __shfl_xor_sync(0xffffffffu, cj, d);
    if (oj >= 0 && (cj < 0 || og > cg || (og == cg && oj < cj))) cg = og, cj = oj;
  }
  if (lane == 0) s_g[w] = cg, s_j[w] = cj;
  __syncthreads();
  if (threadIdx.x == 0) {
    double g = -INFINITY;
    int j = -1;
    for (int q = 0; q < SEL_WARPS; ++q)
      if (s_j[q] >= 0 && (j < 0 || s_g[q] > g || (s_g[q] == g && s_j[q] < j))) g = s_g[q], j = s_j[q];
    a.gain[(int64_t)s * a.K + kk] = g;
    a.best[(int64_t)s * a.K + kk] = j;
    s_j[0] = j;
    if (kk == 0) var_store(a.total + (int64_t)s * VAR_WORDS, tot);
  }
  __syncthreads();
  if (bj >= 0 && bj == s_j[0]) var_store(a.left + ((int64_t)s * a.K + kk) * VAR_WORDS, bl);
}

// Categorical features wider than CAT_SMEM_ARITY: seg[q] = (slot - hist_base, subset position) of each such (slot,
// feature) of the chunk.  cat_centroid_kernel writes every category's centroid, cat_rank_kernel its rank in the stable
// centroid order (smaller centroid first, equal centroids by category), tiled through shared memory, and puts the
// category at that rank of `order`: the same order select_var_kernel builds for narrower features.
__global__ void cat_centroid_kernel(const unsigned long long* __restrict__ hist, const int2* __restrict__ seg,
                                    const int* __restrict__ sub, const int* __restrict__ arity, int K, int NB,
                                    int hist_base, double scale1, double* __restrict__ cen) {
  const int2 q = seg[blockIdx.y];
  const int ar = arity[sub[(int64_t)(q.x + hist_base) * K + q.y]];
  const int64_t base = ((int64_t)q.x * K + q.y) * NB;
  for (int c = blockIdx.x * blockDim.x + threadIdx.x; c < ar; c += gridDim.x * blockDim.x)
    cen[base + c] = var_centroid(hist + (base + c) * VAR_WORDS, scale1);
}
__global__ void __launch_bounds__(256) cat_rank_kernel(const double* __restrict__ cen, const int2* __restrict__ seg,
                                                       const int* __restrict__ sub, const int* __restrict__ arity, int K,
                                                       int NB, int hist_base, uint32_t* __restrict__ order) {
  __shared__ double tile[RANK_TILE];
  const int2 q = seg[blockIdx.y];
  const int ar = arity[sub[(int64_t)(q.x + hist_base) * K + q.y]];
  if ((int)(blockIdx.x * blockDim.x) >= ar) return;
  const int64_t base = ((int64_t)q.x * K + q.y) * NB;
  const int c = blockIdx.x * blockDim.x + threadIdx.x;
  const double me = c < ar ? cen[base + c] : 0.0;
  int rank = 0;
  for (int t0 = 0; t0 < ar; t0 += RANK_TILE) {
    const int tn = min(RANK_TILE, ar - t0);
    __syncthreads();
    for (int i = threadIdx.x; i < tn; i += blockDim.x) tile[i] = cen[base + t0 + i];
    __syncthreads();
    if (c < ar)
      for (int i = 0; i < tn; ++i) rank += (tile[i] < me || (tile[i] == me && t0 + i < c)) ? 1 : 0;
  }
  if (c < ar) order[base + rank] = (uint32_t)c;
}

// one thread per row: every tree's walk (a continuous node sends x <= threshold left, a categorical node sends x left
// iff x equals one of its left categories cat_ids[cat_off[i] .. cat_off[i + 1]), ascending), the predictions summed in
// tree order from 0.0 and divided by the number of trees
__global__ void __launch_bounds__(128) predict_reg_kernel(const int* __restrict__ tree_off, int T,
                                                          const int* __restrict__ feat, const double* __restrict__ thr,
                                                          const int* __restrict__ left, const int* __restrict__ right,
                                                          const double* __restrict__ pred,
                                                          const long long* __restrict__ cat_off,
                                                          const int* __restrict__ cat_ids, const double* __restrict__ x,
                                                          int64_t n, int F, double* __restrict__ out) {
  const int64_t r = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (r >= n) return;
  const double* xr = x + r * F;
  double sum = 0.0;
  for (int t = 0; t < T; ++t) {
    int i = __ldg(tree_off + t);
    for (int f = __ldg(feat + i); f >= 0; f = __ldg(feat + i)) {
      const double v = xr[f];
      long long lo = __ldg(cat_off + i), hi = __ldg(cat_off + i + 1);
      bool go;
      if (hi > lo) {
        go = false;
        if (v >= 0.0 && v < 2147483648.0 && v == trunc(v)) {
          const int c = (int)v;
          while (lo < hi) {
            const long long mid = (lo + hi) >> 1;
            if (__ldg(cat_ids + mid) < c) lo = mid + 1;
            else hi = mid;
          }
          go = lo < __ldg(cat_off + i + 1) && __ldg(cat_ids + lo) == c;
        }
      } else {
        go = v <= __ldg(thr + i);
      }
      i = go ? __ldg(left + i) : __ldg(right + i);
    }
    sum = __dadd_rn(sum, __ldg(pred + i));
  }
  out[r] = __ddiv_rn(sum, (double)T);
}

}  // namespace rf
}  // namespace pio
