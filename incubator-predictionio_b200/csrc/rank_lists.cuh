// rank_lists.cuh -- the product ranking template's predict on batches (pio_als_rank_lists, DESIGN.md 4.17): every entry
// of a query's item list scored against the query's user, and the list stably ordered by java.lang.Double.compare
// descending (docs/manual/source/templates/productranking/dase.html.md.erb:471-530).
//   tile path   (lists of at most RL_TILE entries, packed into tiles by rank_plan.h): one CTA per tile scores two entries
//               per thread, sorts the tile by (query, order key, position) with a bitonic sort in shared memory and
//               writes positions and scores straight to the output;
//   radix path  (longer lists): rl_radix_score_kernel writes (order key, entry) pairs, one stable 64-bit radix sort by
//               the key and a second stable one by the query of each entry, then rl_radix_out_kernel writes the output.
// Entries start in (query, position) order, so both paths give equal keys in query order.  An entry without a score
// (unknown item, item without a factor, or the query's user unknown / without a factor) scores +0.0, so a query that is
// not ranked comes out as the identity order with zero scores; its flag says so.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include "rank_plan.h"

namespace pio {

constexpr int RL_THREADS = RL_TILE / 2;
constexpr uint64_t RL_CANON_NAN = 0x7ff8000000000000ull;   // Double.doubleToLongBits(Double.NaN)

// the factors a call reads: row r of a side is F[perm[r] * kp ..] when r is in [0, n) and deg[r] > 0
struct RlSide {
  const float* F;
  const int* perm;
  const uint32_t* deg;
  int n;
};

// one part of a call on the device; queries and entries are numbered from the part's first
struct RlPart {
  const int* users;        // [queries]
  const long long* lp;     // [queries + 1] entry offsets
  const int* items;        // [entries]
  int* out_pos;            // [entries]
  double* out_score;       // [entries]
  uint8_t* out_ranked;     // [queries]
};

__device__ __forceinline__ const float* rl_row(const RlSide& s, int r, int kp) {
  return (r >= 0 && r < s.n && __ldg(s.deg + r) > 0) ? s.F + (size_t)__ldg(s.perm + r) * kp : nullptr;
}

// dotProduct over the float factors widened to double: an fp64 sum in index order from 0.  The padded columns are zero
// on both sides and the sum never is -0.0, so adding their products changes nothing.
__device__ __forceinline__ double rl_dot(const float* __restrict__ x, const float* __restrict__ y, int kp) {
  const float4* x4 = reinterpret_cast<const float4*>(x);
  const float4* y4 = reinterpret_cast<const float4*>(y);
  double acc = 0.0;
  for (int c = 0; c < kp / 4; ++c) {
    const float4 a = __ldg(x4 + c), b = __ldg(y4 + c);
    acc = fma((double)a.x, (double)b.x, acc);   // the product of two widened floats is exact: fma == acc + x * y
    acc = fma((double)a.y, (double)b.y, acc);
    acc = fma((double)a.z, (double)b.z, acc);
    acc = fma((double)a.w, (double)b.w, acc);
  }
  return acc;
}

// the score of (user, item), +0.0 when either has no factor; *has: both have one.  A NaN comes back canonical.
__device__ __forceinline__ double rl_score(const RlSide& U, const RlSide& I, int kp, int user, int item, bool* has) {
  const float* u = rl_row(U, user, kp);
  const float* y = u ? rl_row(I, item, kp) : nullptr;
  *has = y != nullptr;
  if (!y) return 0.0;
  const double s = rl_dot(y, u, kp);
  return s != s ? __longlong_as_double((long long)RL_CANON_NAN) : s;
}

// ascending order key = Double.compare descending: NaN first, +inf ... +0.0, then -0.0, the negatives, -inf last
__device__ __forceinline__ uint64_t rl_order_key(double s) {
  const uint64_t b = (uint64_t)__double_as_longlong(s);
  return (b >> 63) ? b : ~(b | 0x8000000000000000ull);
}
__device__ __forceinline__ double rl_key_score(uint64_t k) {
  return __longlong_as_double((long long)((k >> 63) ? k : ~k & 0x7fffffffffffffffull));
}

// (query segment, order key, entry) order of a tile's sort; padding (segment 0xffff) sorts last
__device__ __forceinline__ bool rl_less(uint64_t ka, uint32_t aa, uint64_t kb, uint32_t ab) {
  if ((aa >> 16) != (ab >> 16)) return (aa >> 16) < (ab >> 16);
  if (ka != kb) return ka < kb;
  return aa < ab;
}

// One CTA per tile t: queries tile_q[tile_ptr[t] .. tile_ptr[t + 1]) with their entry offsets tile_off inside the tile
// and tile_n[t] entries in all.
__global__ void __launch_bounds__(RL_THREADS) rl_tile_kernel(RlSide U, RlSide I, int kp, RlPart p,
                                                              const int* __restrict__ tile_q,
                                                              const int* __restrict__ tile_ptr,
                                                              const int* __restrict__ tile_off,
                                                              const int* __restrict__ tile_n) {
  __shared__ uint64_t s_key[RL_TILE];
  __shared__ uint32_t s_aux[RL_TILE];   // segment << 16 | entry in the tile
  __shared__ int s_off[RL_TILE + 1];
  __shared__ int s_q[RL_TILE];
  __shared__ uint8_t s_has[RL_TILE];
  const int t = blockIdx.x;
  const int j0 = tile_ptr[t], nseg = tile_ptr[t + 1] - j0, n = tile_n[t];
  for (int s = threadIdx.x; s < nseg; s += RL_THREADS) {
    s_q[s] = tile_q[j0 + s];
    s_off[s] = tile_off[j0 + s];
    s_has[s] = 0;
  }
  if (threadIdx.x == 0) s_off[nseg] = n;
  __syncthreads();
  int n2 = 2;
  while (n2 < n) n2 <<= 1;
  for (int e = threadIdx.x; e < n2; e += RL_THREADS) {
    uint64_t key = ~0ull;
    uint32_t aux = 0xffffffffu;
    if (e < n) {
      int lo = 0, hi = nseg - 1;   // the segment of e: the last one starting at or before it
      while (lo < hi) {
        const int mid = (lo + hi + 1) >> 1;
        if (s_off[mid] <= e) lo = mid;
        else hi = mid - 1;
      }
      const int q = s_q[lo];
      bool has;
      const double sc = rl_score(U, I, kp, __ldg(p.users + q), __ldg(p.items + p.lp[q] + (e - s_off[lo])), &has);
      if (has) s_has[lo] = 1;   // the block-level OR of the segment's entries
      key = rl_order_key(sc);
      aux = (uint32_t)lo << 16 | (uint32_t)e;
    }
    s_key[e] = key;
    s_aux[e] = aux;
  }
  __syncthreads();
  for (int k = 2; k <= n2; k <<= 1) {
    for (int j = k >> 1; j > 0; j >>= 1) {
      for (int i = threadIdx.x; i < n2 / 2; i += RL_THREADS) {
        const int a = 2 * (i & ~(j - 1)) + (i & (j - 1)), b = a + j;
        const uint64_t ka = s_key[a], kb = s_key[b];
        const uint32_t aa = s_aux[a], ab = s_aux[b];
        if (rl_less(kb, ab, ka, aa) == ((a & k) == 0)) {
          s_key[a] = kb, s_key[b] = ka;
          s_aux[a] = ab, s_aux[b] = aa;
        }
      }
      __syncthreads();
    }
  }
  for (int s = threadIdx.x; s < n; s += RL_THREADS) {
    const uint32_t aux = s_aux[s];
    const int seg = (int)(aux >> 16), start = s_off[seg];
    const long long o = p.lp[s_q[seg]] + (s - start);
    p.out_pos[o] = (int)(aux & 0xffffu) - start;
    p.out_score[o] = rl_key_score(s_key[s]);
  }
  for (int s = threadIdx.x; s < nseg; s += RL_THREADS) p.out_ranked[s_q[s]] = s_has[s];
}

// the radix query of compacted entry x: the last k with c[k] <= x
__device__ __forceinline__ int rl_radix_query(const long long* __restrict__ c, int nr, long long x) {
  int lo = 0, hi = nr - 1;
  while (lo < hi) {
    const int mid = (lo + hi + 1) >> 1;
    if (__ldg(c + mid) <= x) lo = mid;
    else hi = mid - 1;
  }
  return lo;
}

// The part's radix queries rq[0 .. nr), their entries compacted: query k's at [c[k], c[k + 1]).  Writes (order key,
// entry) pairs, each entry's score, and has[k] = 1 when an entry of query k has a score (has is zeroed by the caller).
__global__ void rl_radix_score_kernel(RlSide U, RlSide I, int kp, RlPart p, const int* __restrict__ rq,
                                      const long long* __restrict__ c, int nr, long long n, uint64_t* __restrict__ key,
                                      uint32_t* __restrict__ val, double* __restrict__ score, uint8_t* __restrict__ has) {
  for (long long x = (long long)blockIdx.x * blockDim.x + threadIdx.x; x < n; x += (long long)gridDim.x * blockDim.x) {
    const int k = rl_radix_query(c, nr, x);
    const int q = __ldg(rq + k);
    bool h;
    const double sc = rl_score(U, I, kp, __ldg(p.users + q), __ldg(p.items + p.lp[q] + (x - c[k])), &h);
    if (h) has[k] = 1;
    key[x] = rl_order_key(sc);
    val[x] = (uint32_t)x;
    score[x] = sc;
  }
}

// after the sort by order key: (radix query of the entry, entry) pairs for the stable sort by query
__global__ void rl_radix_query_keys_kernel(const uint32_t* __restrict__ val, const long long* __restrict__ c, int nr,
                                           long long n, uint64_t* __restrict__ key, uint32_t* __restrict__ val_out) {
  for (long long s = (long long)blockIdx.x * blockDim.x + threadIdx.x; s < n; s += (long long)gridDim.x * blockDim.x) {
    const uint32_t x = val[s];
    key[s] = (uint64_t)rl_radix_query(c, nr, x);
    val_out[s] = x;
  }
}

// sorted position s holds query key[s]'s (s - c[key[s]])-th ranked entry
__global__ void rl_radix_out_kernel(RlPart p, const int* __restrict__ rq, const long long* __restrict__ c,
                                    const uint64_t* __restrict__ key, const uint32_t* __restrict__ val,
                                    const double* __restrict__ score, const uint8_t* __restrict__ has, long long n) {
  for (long long s = (long long)blockIdx.x * blockDim.x + threadIdx.x; s < n; s += (long long)gridDim.x * blockDim.x) {
    const int k = (int)key[s];
    const int q = __ldg(rq + k);
    const long long start = c[k], x = val[s];
    const long long o = p.lp[q] + (s - start);
    p.out_pos[o] = (int)(x - start);
    p.out_score[o] = score[x];
    if (s == start) p.out_ranked[q] = has[k];
  }
}

}  // namespace pio
