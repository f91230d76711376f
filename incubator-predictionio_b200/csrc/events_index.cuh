// events_index.cuh -- the event index of pio_events_index_* (DESIGN.md section 3.3): the events of one `find` view
// (entityType, eventNames, targetEntityType) of an append-only event file, kept on the device, ordered so that the
// events of one entityId are one range in LEventStore.findByEntity's order (eventTime descending, file order).
//
// Entry: hash of the decoded entityId (ids_hash, the hash of ids_encode.cuh), eventTime (us), byte offset and length of
// the event's line in the file, and the id bytes in an arena (id_off / id_len).  Entries live in two sorted runs:
//   main    every entry up to the last merge
//   delta   entries appended since; every delta offset is larger than every main offset
// both in the order (hash, time descending, offset ascending).
//
//   build / append   the chunk loop of pio_events_scan (events_scan.cuh) with the view's filter; eix_take_kernel turns a
//                    chunk's matched events into entries on the device (line byte ranges from the chunk's `starts`), the
//                    id bytes are copied device to device; nothing goes back to the host but the fallback lines
//   sort             stable radix_sort_pairs by time (sign bit flipped, then inverted: descending) of the entries in
//                    file order, then stable by hash; eix_gather_kernel applies the permutation
//   merge            eix_merge_kernel (merge path): each CTA binary-searches its diagonal, each thread its own inside
//                    the CTA's span, and merges EIX_MERGE_ITEMS outputs.  The arenas are not moved: the second run's
//                    arena is appended to the first's and its id offsets are rebased.  A sorted append is merged into
//                    delta; delta is merged into main when it grows past 1 / PIO_EVENTS_INDEX_MERGE_DIVISOR of main.
//   lookup           one warp per queried id: hash, lower_bound in both runs, then the two equal-hash ranges walked as
//                    one merge (each lane finds the element at its merged position by merge path), id bytes compared
//                    exactly so that the entries of a colliding id are skipped.  eix_count_kernel counts (up to the
//                    limit), eix_write_kernel writes (offset, length) pairs at the scanned counts.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include "events_scan.cuh"
#include "ids_encode.cuh"

namespace pio {

// one run (or an unsorted batch) of entries, on the device
struct EixRun {
  long long n = 0;
  long long arena_bytes = 0;
  uint64_t* hash = nullptr;
  long long* time_us = nullptr;
  long long* off = nullptr;       // byte offset of the line in the file
  int32_t* len = nullptr;         // line length without its terminator
  long long* id_off = nullptr;    // entityId = arena[id_off .. id_off + id_len)
  int32_t* id_len = nullptr;
  uint8_t* arena = nullptr;
};

// (hash, time descending, offset ascending); offsets are unique, so no two entries tie
__device__ __forceinline__ bool eix_before(uint64_t h1, long long t1, long long o1, uint64_t h2, long long t2,
                                           long long o2) {
  if (h1 != h2) return h1 < h2;
  if (t1 != t2) return t1 > t2;
  return o1 < o2;
}

__device__ __forceinline__ bool eix_before(const EixRun& A, long long i, const EixRun& B, long long j) {
  return eix_before(A.hash[i], A.time_us[i], A.off[i], B.hash[j], B.time_us[j], B.off[j]);
}

// merge path: how many of A[a_lo ..) are among the first d outputs of merge(A[a_lo .. a_hi), B[b_lo .. b_hi))
__device__ __forceinline__ long long eix_split(const EixRun& A, long long a_lo, long long a_hi, const EixRun& B,
                                               long long b_lo, long long b_hi, long long d) {
  const long long na = a_hi - a_lo, nb = b_hi - b_lo;
  long long lo = d - nb > 0 ? d - nb : 0, hi = d < na ? d : na;
  while (lo < hi) {
    const long long m = (lo + hi) >> 1;
    if (eix_before(A, a_lo + m, B, b_lo + d - 1 - m)) lo = m + 1;
    else hi = m;
  }
  return lo;
}

// a chunk's matched events (events_scan.cuh EvOut, line order) -> entries at [n0, n0 + nm) of a batch whose arena
// holds the ids at the scan's id offsets
__global__ void eix_take_kernel(const EvOut o, const uint8_t* __restrict__ t, const uint32_t* __restrict__ starts,
                                long long nm, long long line_base, long long byte_base, long long eid_end,
                                uint64_t mask, EixRun b, long long n0) {
  const long long k = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (k >= nm) return;
  uint32_t lb, le;
  ev_line_range(t, starts, o.line[k] - line_base, &lb, &le);
  const long long io = o.eid_off[k], ie = k + 1 < nm ? o.eid_off[k + 1] : eid_end;
  b.hash[n0 + k] = ids_hash(b.arena + io, ie - io, mask);
  b.time_us[n0 + k] = o.time_us[k];
  b.off[n0 + k] = byte_base + lb;
  b.len[n0 + k] = (int32_t)(le - lb);
  b.id_off[n0 + k] = io;
  b.id_len[n0 + k] = (int32_t)(ie - io);
}

// hashes of host-provided entries (their ids are in the arena already)
__global__ void eix_hash_kernel(EixRun b, uint64_t mask) {
  const long long k = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (k < b.n) b.hash[k] = ids_hash(b.arena + b.id_off[k], b.id_len[k], mask);
}

// sort keys: eventTime descending (sign bit flipped as in events_fold.cuh, then inverted), then the hash
__global__ void eix_time_key_kernel(const long long* __restrict__ time_us, long long n, uint64_t* __restrict__ key,
                                    uint32_t* __restrict__ pay) {
  const long long e = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (e >= n) return;
  key[e] = ~((uint64_t)time_us[e] ^ (1ull << 63));
  pay[e] = (uint32_t)e;
}

__global__ void eix_hash_key_kernel(const uint32_t* __restrict__ pay, const uint64_t* __restrict__ hash, long long n,
                                    uint64_t* __restrict__ key) {
  const long long s = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (s < n) key[s] = hash[pay[s]];
}

__global__ void eix_gather_kernel(const EixRun src, const uint32_t* __restrict__ perm, EixRun dst) {
  const long long s = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (s >= dst.n) return;
  const uint32_t e = perm[s];
  dst.hash[s] = src.hash[e];
  dst.time_us[s] = src.time_us[e];
  dst.off[s] = src.off[e];
  dst.len[s] = src.len[e];
  dst.id_off[s] = src.id_off[e];
  dst.id_len[s] = src.id_len[e];
}

constexpr int EIX_MERGE_THREADS = 128;
constexpr int EIX_MERGE_ITEMS = 8;
constexpr int EIX_MERGE_SPAN = EIX_MERGE_THREADS * EIX_MERGE_ITEMS;

// out = merge(A, B); out.arena holds A's arena then B's, so B's id offsets move by A.arena_bytes
__global__ void __launch_bounds__(EIX_MERGE_THREADS) eix_merge_kernel(const EixRun A, const EixRun B, EixRun out) {
  __shared__ long long cta_a[2];
  const long long n = A.n + B.n;
  const long long d0 = (long long)blockIdx.x * EIX_MERGE_SPAN;
  const long long d1 = d0 + EIX_MERGE_SPAN < n ? d0 + EIX_MERGE_SPAN : n;
  if (threadIdx.x < 2) cta_a[threadIdx.x] = eix_split(A, 0, A.n, B, 0, B.n, threadIdx.x ? d1 : d0);
  __syncthreads();
  const long long a0 = cta_a[0], a1 = cta_a[1], b0 = d0 - a0, b1 = d1 - a1;
  const long long t0 = (long long)threadIdx.x * EIX_MERGE_ITEMS;
  if (d0 + t0 >= d1) return;
  const long long ta = eix_split(A, a0, a1, B, b0, b1, t0);
  long long i = a0 + ta, j = b0 + (t0 - ta);
  const long long tend = d0 + t0 + EIX_MERGE_ITEMS < d1 ? d0 + t0 + EIX_MERGE_ITEMS : d1;
  for (long long d = d0 + t0; d < tend; ++d) {
    const bool take_a = i < a1 && (j >= b1 || eix_before(A, i, B, j));
    if (take_a) {
      out.hash[d] = A.hash[i]; out.time_us[d] = A.time_us[i]; out.off[d] = A.off[i]; out.len[d] = A.len[i];
      out.id_off[d] = A.id_off[i]; out.id_len[d] = A.id_len[i];
      ++i;
    } else {
      out.hash[d] = B.hash[j]; out.time_us[d] = B.time_us[j]; out.off[d] = B.off[j]; out.len[d] = B.len[j];
      out.id_off[d] = B.id_off[j] + A.arena_bytes; out.id_len[d] = B.id_len[j];
      ++j;
    }
  }
}

// ---- lookup -------------------------------------------------------------------------------------------------------
constexpr int EIX_LOOKUP_WARPS = 4;

__device__ __forceinline__ long long eix_lower_bound(const uint64_t* hash, long long n, uint64_t h) {
  long long lo = 0, hi = n;
  while (lo < hi) {
    const long long m = (lo + hi) >> 1;
    if (hash[m] < h) lo = m + 1;
    else hi = m;
  }
  return lo;
}

__device__ __forceinline__ bool eix_same_id(const uint8_t* arena, const long long* id_off, const int32_t* id_len,
                                            long long k, const uint8_t* q, long long nq) {
  if (id_len[k] != nq) return false;
  const uint8_t* p = arena + id_off[k];
  for (long long c = 0; c < nq; ++c)
    if (p[c] != q[c]) return false;
  return true;
}

// the equal-hash ranges of query id q in both runs
struct EixRanges {
  long long ma, mb, da, db;
};

__device__ __forceinline__ EixRanges eix_ranges(const EixRun& M, const EixRun& D, uint64_t h) {
  EixRanges r;
  r.ma = eix_lower_bound(M.hash, M.n, h);
  r.mb = h == ~0ull ? M.n : eix_lower_bound(M.hash, M.n, h + 1);
  r.da = eix_lower_bound(D.hash, D.n, h);
  r.db = h == ~0ull ? D.n : eix_lower_bound(D.hash, D.n, h + 1);
  return r;
}

// count[q] = entries of id q in both runs, at most `limit` (limit < 0: no limit)
__global__ void __launch_bounds__(32 * EIX_LOOKUP_WARPS)
eix_count_kernel(const EixRun M, const EixRun D, const uint8_t* __restrict__ qb, const long long* __restrict__ qo,
                 int nq, uint64_t mask, long long limit, uint32_t* __restrict__ count) {
  const int q = blockIdx.x * EIX_LOOKUP_WARPS + (threadIdx.x >> 5), lane = threadIdx.x & 31;
  if (q >= nq) return;
  const uint8_t* id = qb + qo[q];
  const long long idn = qo[q + 1] - qo[q];
  const EixRanges r = eix_ranges(M, D, ids_hash(id, idn, mask));
  const long long na = r.mb - r.ma, nt = na + (r.db - r.da);
  const long long cap = limit < 0 ? nt : limit;
  long long c = 0;
  for (long long k = 0; k < nt && c < cap; k += 32) {
    const long long e = k + lane;
    bool m = false;
    if (e < nt)
      m = e < na ? eix_same_id(M.arena, M.id_off, M.id_len, r.ma + e, id, idn)
                 : eix_same_id(D.arena, D.id_off, D.id_len, r.da + e - na, id, idn);
    c += __popc(__ballot_sync(0xffffffffu, m));
  }
  if (lane == 0) count[q] = (uint32_t)(c < cap ? c : cap);
}

// the first count[q] entries of id q in merged (time descending, offset ascending) order, at pos[q]
__global__ void __launch_bounds__(32 * EIX_LOOKUP_WARPS)
eix_write_kernel(const EixRun M, const EixRun D, const uint8_t* __restrict__ qb, const long long* __restrict__ qo,
                 int nq, uint64_t mask, const uint32_t* __restrict__ count, const uint32_t* __restrict__ pos,
                 long long* __restrict__ out_off, int32_t* __restrict__ out_len) {
  const int q = blockIdx.x * EIX_LOOKUP_WARPS + (threadIdx.x >> 5), lane = threadIdx.x & 31;
  if (q >= nq || count[q] == 0) return;
  const uint8_t* id = qb + qo[q];
  const long long idn = qo[q + 1] - qo[q];
  const EixRanges r = eix_ranges(M, D, ids_hash(id, idn, mask));
  const long long nt = (r.mb - r.ma) + (r.db - r.da), want = count[q];
  long long done = 0;
  for (long long k = 0; k < nt && done < want; k += 32) {
    const long long d = k + lane;
    bool m = false;
    long long o = 0;
    int32_t l = 0;
    if (d < nt) {   // the element at merged position d
      const long long a = eix_split(M, r.ma, r.mb, D, r.da, r.db, d), i = r.ma + a, j = r.da + (d - a);
      const bool from_m = i < r.mb && (j >= r.db || eix_before(M, i, D, j));
      const long long e = from_m ? i : j;
      m = eix_same_id(from_m ? M.arena : D.arena, from_m ? M.id_off : D.id_off, from_m ? M.id_len : D.id_len, e, id,
                      idn);
      o = (from_m ? M.off : D.off)[e];
      l = (from_m ? M.len : D.len)[e];
    }
    const uint32_t bal = __ballot_sync(0xffffffffu, m);
    const long long rk = done + __popc(bal & ((1u << lane) - 1u));
    if (m && rk < want) {
      out_off[pos[q] + rk] = o;
      out_len[pos[q] + rk] = l;
    }
    done += __popc(bal);
  }
}

}  // namespace pio
