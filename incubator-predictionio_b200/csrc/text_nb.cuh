// text_nb.cuh -- the text classification template's featurizer and multinomial Naive Bayes on sparse TF-IDF vectors
// (DESIGN.md 4.18).  The rules are tests/textclassification_ref.py's; pio_als.cu runs the kernels part by part
// (text_plan.h).
//
// One part of documents, each a raw JSON string token:
//   tx_split_kernel    one thread per document: decode the token (decode_string_lenient), split on 0x20 with Java's
//                      String.split(" ") rules, drop stop words (a device hash set, bytes verified), and count the
//                      kept tokens and n-gram windows
//   tx_hash_kernel     one thread per window: Spark's murmur3 over the window's tokens as one byte string, hashed
//                      across token boundaries without a joined copy; key = (document, nonNegativeMod(h, D))
//   radix_sort_pairs   the keys (sort_scan.cuh); runs of equal keys are the document's term frequencies
//   tx_head_*          the runs: one entry (document, index, count) per run, in (document, index) order
// then, by caller:
//   tx_df_kernel       train: df_j += 1 per entry (integers), and the entry kept for the class sums
//   tx_sum_kernel      train: s_cj += tf * idf_j, exactly, in 192-bit fixed point (units of 2^-96)
//   tx_round_kernel    train: each s_cj rounded once to the nearest double, ties to even
//   tx_value_kernel    features / scores: x_j = tf, or tf * idf_j (one fp64 multiply)
//   tx_score_kernel    scores: per (query, class) a left fold over the query's entries, then + pi_c
// The k-fold evaluation (pio_text_folds_*, DESIGN.md 4.18.1) keeps every part's entries, documents made global
// (tx_doc_base_kernel), and cuts fold f's lists from them (document d tests in fold d % k):
//   tx_fold_flag_kernel / scan / tx_fold_gather_kernel   the training entries tagged with their document's class, or the
//                      test entries renumbered t = (d - f) / k; both keep (document, index) order
// and runs the kernels above on those lists unchanged.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include "event_line.h"
#include "sort_scan.cuh"

namespace pio {

// The stop-word set's 64-bit hash of p[0 .. n): FNV-1a with a splitmix64 finaliser (host and device).
__host__ __device__ __forceinline__ uint64_t tx_hash(const uint8_t* p, long long n) {
  uint64_t h = 0xcbf29ce484222325ull;
  for (long long b = 0; b < n; ++b) {
    h ^= (uint64_t)p[b];
    h *= 0x100000001b3ull;
  }
  h ^= h >> 30; h *= 0xBF58476D1CE4E5B9ull;
  h ^= h >> 27; h *= 0x94D049BB133111EBull;
  h ^= h >> 31;
  return h;
}

// An open-addressing set of the stop words (linear probing): slot -> word index or -1; bytes / off hold the words.
struct TxStop {
  const int* slot;
  const uint8_t* bytes;
  const long long* off;
  unsigned mask;      // slots - 1 (a power of two minus one)
  int n;              // words
};

__device__ __forceinline__ bool tx_is_stop(const TxStop& s, const uint8_t* p, int n) {
  if (s.n == 0) return false;
  unsigned i = (unsigned)tx_hash(p, n) & s.mask;
  for (;;) {
    const int w = s.slot[i];
    if (w < 0) return false;
    const long long a = s.off[w];
    if (s.off[w + 1] - a == n && ev::bytes_eq(s.bytes + a, p, n)) return true;
    i = (i + 1) & s.mask;
  }
}

// Per document d of a part (tokens raw[off[d] .. off[d + 1]), offsets local to the part): the decoded text in
// dec[off[d] ..], the kept tokens as (start in dec, length) in tok_b / tok_n from slot off[d] on (a token of L bytes
// holds at most L - 1 tokens), their count ntok[d] and the n-gram windows nwin[d].
__global__ void __launch_bounds__(256)
tx_split_kernel(const uint8_t* __restrict__ raw, const long long* __restrict__ off, int nd, TxStop stop, int n_gram,
                uint8_t* __restrict__ dec, uint32_t* __restrict__ tok_b, uint32_t* __restrict__ tok_n,
                uint32_t* __restrict__ ntok, uint32_t* __restrict__ nwin) {
  const int d = blockIdx.x * blockDim.x + threadIdx.x;
  if (d >= nd) return;
  const long long b = off[d], e = off[d + 1];
  uint8_t* out = dec + b;
  const int len = ev::decode_string_lenient(raw + b, 0, (int)(e - b), out);
  bool space = false;
  int end = len;
  for (int i = 0; i < len; ++i) space |= out[i] == ' ';
  if (space)
    while (end > 0 && out[end - 1] == ' ') --end;   // trailing empty pieces are dropped
  uint32_t k = 0;
  auto keep = [&](int s, int n) {
    if (!tx_is_stop(stop, out + s, n)) {
      tok_b[b + k] = (uint32_t)(b + s);
      tok_n[b + k] = (uint32_t)n;
      ++k;
    }
  };
  if (!space) {
    keep(0, len);                                    // no space at all: the whole text, "" included
  } else if (end > 0) {
    int s = 0;
    for (int i = 0; i <= end; ++i)
      if (i == end || out[i] == ' ') {
        keep(s, i - s);
        s = i + 1;
      }
  }
  ntok[d] = k;
  nwin[d] = k == 0 ? 0u : (k <= (uint32_t)n_gram ? 1u : k - (uint32_t)n_gram + 1u);
}

__device__ __forceinline__ uint32_t tx_rotl(uint32_t x, int r) { return (x << r) | (x >> (32 - r)); }

__device__ __forceinline__ uint32_t tx_mix(uint32_t h, uint32_t k) {
  k *= 0xCC9E2D51u;
  k = tx_rotl(k, 15);
  k *= 0x1B873593u;
  h ^= k;
  h = tx_rotl(h, 13);
  return h * 5u + 0xE6546B64u;
}

// One key per window w of the part: its document (by binary search of the window offsets) and the feature index of
// Spark's hashUnsafeBytes(seed 42) of the window's tokens joined with no separator.
__global__ void __launch_bounds__(256)
tx_hash_kernel(const uint8_t* __restrict__ dec, const long long* __restrict__ off, const uint32_t* __restrict__ tok_b,
               const uint32_t* __restrict__ tok_n, const uint32_t* __restrict__ ntok,
               const uint32_t* __restrict__ win_off, int nd, long long n_win, int n_gram, int num_features, int fbits,
               uint64_t* __restrict__ keys, uint32_t* __restrict__ vals) {
  const long long w = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (w >= n_win) return;
  int lo = 0, hi = nd - 1;   // the last document whose first window is <= w
  while (lo < hi) {
    const int mid = (lo + hi + 1) >> 1;
    if ((long long)win_off[mid] <= w) lo = mid;
    else hi = mid - 1;
  }
  const int d = lo;
  const long long t0 = off[d] + (w - (long long)win_off[d]);
  const long long t1 = t0 + min((long long)n_gram, (long long)ntok[d]);
  uint32_t h = 42u, k = 0u, total = 0u;
  int c = 0;
  for (long long t = t0; t < t1; ++t) {
    const uint8_t* p = dec + tok_b[t];
    const uint32_t n = tok_n[t];
    for (uint32_t i = 0; i < n; ++i) {
      k |= (uint32_t)p[i] << (8 * c);
      if (++c == 4) {
        h = tx_mix(h, k);
        k = 0u;
        c = 0;
      }
    }
    total += n;
  }
  for (int i = 0; i < c; ++i)   // Spark's tail: each byte sign-extended, mixed as a block of its own
    h = tx_mix(h, (uint32_t)(int32_t)(int8_t)(uint8_t)(k >> (8 * i)));
  h ^= total;
  h ^= h >> 16;
  h *= 0x85EBCA6Bu;
  h ^= h >> 13;
  h *= 0xC2B2AE35u;
  h ^= h >> 16;
  int r = (int)h % num_features;   // nonNegativeMod: Java's remainder, moved into [0, D)
  if (r < 0) r += num_features;
  keys[w] = ((uint64_t)d << fbits) | (uint64_t)r;
  vals[w] = (uint32_t)w;
}

// 1 where a run of equal keys starts
__global__ void __launch_bounds__(256)
tx_head_flag_kernel(const uint64_t* __restrict__ keys, long long n, uint32_t* __restrict__ flag) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) flag[i] = i == 0 || keys[i] != keys[i - 1];
}

// run u (rid = exclusive scan of the flags): its start
__global__ void __launch_bounds__(256)
tx_head_kernel(const uint64_t* __restrict__ keys, const uint32_t* __restrict__ flag, const uint32_t* __restrict__ rid,
               long long n, uint32_t* __restrict__ start) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n && flag[i]) start[rid[i]] = (uint32_t)i;
}

// entry u: document, feature index and term count
__global__ void __launch_bounds__(256)
tx_entry_kernel(const uint64_t* __restrict__ keys, const uint32_t* __restrict__ start, long long nu, long long n,
                int fbits, uint32_t* __restrict__ doc, uint32_t* __restrict__ idx, uint32_t* __restrict__ cnt) {
  const long long u = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (u >= nu) return;
  const uint32_t s = start[u];
  const uint64_t key = keys[s];
  doc[u] = (uint32_t)(key >> fbits);
  idx[u] = (uint32_t)(key & ((1ull << fbits) - 1ull));
  cnt[u] = (u + 1 < nu ? start[u + 1] : (uint32_t)n) - s;
}

// df_j: one per (document, j) entry
__global__ void __launch_bounds__(256)
tx_df_kernel(const uint32_t* __restrict__ idx, long long nu, unsigned long long* __restrict__ df) {
  const long long u = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (u < nu) atomicAdd(&df[idx[u]], 1ull);
}

// x = tf, or tf * idf_j rounded once
__global__ void __launch_bounds__(256)
tx_value_kernel(const uint32_t* __restrict__ idx, const uint32_t* __restrict__ cnt, const double* __restrict__ idf,
                long long nu, double* __restrict__ val) {
  const long long u = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (u >= nu) return;
  const double tf = (double)cnt[u];
  val[u] = idf ? __dmul_rn(tf, idf[idx[u]]) : tf;
}

// the class of each entry, from its document's label (cls may be the doc buffer itself)
__global__ void __launch_bounds__(256)
tx_label_kernel(const uint32_t* doc, const int* __restrict__ label, long long nu, int* cls) {
  const long long u = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (u < nu) cls[u] = label[doc[u]];
}

// Exact class sums.  Each term x = tf * idf_j (a double) is added into three 64-bit words w[0..2] of value
// sum_k w[k] 2^(64 k - 96).  A nonzero term must be at least 2^-44 (its last bit then lies at or above 2^-96) and below
// 2^63 (so fewer than 2^33 terms stay below 2^96); any other term sets *bad and adds nothing.  The atomic adds carry
// explicitly: each wrap of a word is seen by the thread that caused it, which adds the carry one word up.
__device__ __forceinline__ void tx_add192(unsigned long long* w, unsigned long long a0, unsigned long long a1,
                                          unsigned long long a2) {
  unsigned long long o, c1 = 0, c2 = 0;
  if (a0) {
    o = atomicAdd(&w[0], a0);
    c1 = o + a0 < o;
  }
  if (a1) {
    o = atomicAdd(&w[1], a1);
    c2 += o + a1 < o;
  }
  if (c1) {
    o = atomicAdd(&w[1], 1ull);
    c2 += o == ~0ull;
  }
  if (a2 + c2) atomicAdd(&w[2], a2 + c2);
}

__global__ void __launch_bounds__(256)
tx_sum_kernel(const uint32_t* __restrict__ idx, const uint32_t* __restrict__ cnt, const int* __restrict__ cls,
              const double* __restrict__ idf, long long nu, long long D, unsigned long long* __restrict__ acc,
              int* __restrict__ bad) {
  const long long u = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (u >= nu) return;
  const uint32_t j = idx[u];
  const double x = __dmul_rn((double)cnt[u], idf[j]);
  if (x == 0.0) return;
  if (!(x >= 0x1p-44 && x < 0x1p63)) {
    atomicExch(bad, 1);
    return;
  }
  const unsigned long long bits = (unsigned long long)__double_as_longlong(x);
  const int s = (int)((bits >> 52) & 0x7FF) - 979;   // x = mant 2^(exp - 1075) = mant 2^(s - 96), 0 <= s <= 106
  const unsigned long long mant = (bits & ((1ull << 52) - 1ull)) | (1ull << 52);
  const int off = s & 63;
  const unsigned long long lo = mant << off, hi = off ? mant >> (64 - off) : 0ull;
  unsigned long long* w = acc + 3 * ((long long)cls[u] * D + j);
  if (s < 64) tx_add192(w, lo, hi, 0ull);
  else tx_add192(w, 0ull, lo, hi);
}

__device__ __forceinline__ unsigned long long tx_word(unsigned long long w0, unsigned long long w1,
                                                      unsigned long long w2, int i) {
  return i == 0 ? w0 : i == 1 ? w1 : i == 2 ? w2 : 0ull;
}

// each 192-bit sum (units of 2^-96) rounded once to the nearest double, ties to even
__global__ void __launch_bounds__(256)
tx_round_kernel(const unsigned long long* __restrict__ acc, long long n, double* __restrict__ out) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const unsigned long long w0 = acc[3 * i], w1 = acc[3 * i + 1], w2 = acc[3 * i + 2];
  int p;   // the top set bit
  if (w2) p = 128 + 63 - __clzll((long long)w2);
  else if (w1) p = 64 + 63 - __clzll((long long)w1);
  else if (w0) p = 63 - __clzll((long long)w0);
  else {
    out[i] = 0.0;
    return;
  }
  if (p <= 52) {
    out[i] = ldexp((double)w0, -96);   // exact
    return;
  }
  const int sh = p - 52, wi = sh >> 6, bo = sh & 63;
  unsigned long long m = tx_word(w0, w1, w2, wi) >> bo;
  if (bo) m |= tx_word(w0, w1, w2, wi + 1) << (64 - bo);
  m &= (1ull << 53) - 1ull;
  const int rb = sh - 1, rw = rb >> 6, ro = rb & 63;   // the round bit, and every bit below it (sticky)
  const bool round = (tx_word(w0, w1, w2, rw) >> ro) & 1ull;
  bool sticky = (tx_word(w0, w1, w2, rw) & ((1ull << ro) - 1ull)) != 0ull;
  if (rw >= 1) sticky |= w0 != 0ull;
  if (rw >= 2) sticky |= w1 != 0ull;
  if (round && (sticky || (m & 1ull))) ++m;
  out[i] = ldexp((double)m, sh - 96);
}

// raw score of (query q, class c): a left fold from 0.0 over q's entries in index order, each product and add rounded on
// its own, NaN when theta_c has a non-finite entry at an index q lacks (the dense fold meets 0 * inf there), then + pi_c
__global__ void __launch_bounds__(256)
tx_score_kernel(const uint32_t* __restrict__ doc, const uint32_t* __restrict__ idx, const double* __restrict__ val,
                long long nu, int nq, int C, long long D, const double* __restrict__ theta, const double* __restrict__ pi,
                const int* __restrict__ nonfinite, double* __restrict__ out) {
  const long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= (long long)nq * C) return;
  const int q = (int)(t / C), c = (int)(t % C);
  long long lo = 0, hi = nu;   // the first entry of q
  while (lo < hi) {
    const long long mid = (lo + hi) >> 1;
    if (doc[mid] < (uint32_t)q) lo = mid + 1;
    else hi = mid;
  }
  const double* row = theta + (long long)c * D;
  double acc = 0.0;
  int present = 0;
  for (long long e = lo; e < nu && doc[e] == (uint32_t)q; ++e) {
    const double th = row[idx[e]];
    present += !isfinite(th);
    acc = __dadd_rn(acc, __dmul_rn(th, val[e]));
  }
  if (nonfinite[c] > present) acc = __longlong_as_double(0x7FF8000000000000ll);
  out[t] = __dadd_rn(acc, pi[c]);
}

// a part's entries with their documents made global: out[u] = doc[u] + d0
__global__ void __launch_bounds__(256)
tx_doc_base_kernel(const uint32_t* __restrict__ doc, long long nu, uint32_t d0, uint32_t* __restrict__ out) {
  const long long u = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (u < nu) out[u] = doc[u] + d0;
}

__device__ __forceinline__ bool tx_in_fold_list(uint32_t d, int k, int f, bool test) {
  return ((int)(d % (uint32_t)k) == f) == test;
}

// 1 where entry u belongs to fold f's list: its test list (test) or its training list
__global__ void __launch_bounds__(256)
tx_fold_flag_kernel(const uint32_t* __restrict__ doc, long long nu, int k, int f, bool test,
                    uint32_t* __restrict__ flag) {
  const long long u = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (u < nu) flag[u] = tx_in_fold_list(doc[u], k, f, test);
}

// entry u of the list goes to position pos[u] (the exclusive scan of the flags) with its index and count, and as its
// key either its document's class cls_doc[d] (the training list) or, cls_doc null, its test position (d - f) / k
__global__ void __launch_bounds__(256)
tx_fold_gather_kernel(const uint32_t* __restrict__ doc, const uint32_t* __restrict__ idx,
                      const uint32_t* __restrict__ cnt, const uint32_t* __restrict__ pos, long long nu, int k, int f,
                      bool test, const int* __restrict__ cls_doc, uint32_t* __restrict__ okey,
                      uint32_t* __restrict__ oidx, uint32_t* __restrict__ ocnt) {
  const long long u = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (u >= nu) return;
  const uint32_t d = doc[u];
  if (!tx_in_fold_list(d, k, f, test)) return;
  const uint32_t p = pos[u];
  okey[p] = cls_doc ? (uint32_t)cls_doc[d] : (d - (uint32_t)f) / (uint32_t)k;
  oidx[p] = idx[u];
  ocnt[p] = cnt[u];
}

}  // namespace pio
