// ids_encode.cuh -- dictionary encoding of string ids on the GPU: what the templates do with
//     val userStringIntMap = BiMap.stringInt(data.ratings.map(_.user))      (keys.distinct.collect -> HashMap(key -> index))
// (data/src/main/scala/org/apache/predictionio/data/storage/BiMap.scala:116-128, called from
// examples/scala-parallel-recommendation/blacklist-items/src/main/scala/ALSAlgorithm.scala:59-65) before they can build
// MLlibRating(userIndex, itemIndex, rating).  SURVEY.md 8(f)-1: on 100 M events this (string hashing, distinct, lookup per
// event) dominates the CPU wall time of the reference's prep step.
//
// Input: n strings as one byte buffer + n + 1 offsets.  Output: a dense index per string, indices handed out in order of
// first occurrence (the reference's collect order is unspecified; results must be compared by string id), and the
// position of the first occurrence of every distinct string (= the inverse map).
//
// Pipeline (all HBM-bound integer work on the device): 64-bit hash per string -> stable radix sort of (hash, position) ->
// runs of equal hash -> every element finds its group head = the first element of its run with identical BYTES (one
// comparison unless two different strings share a 64-bit hash; then a short forward search inside the run) -> heads
// numbered by first occurrence (flag + scan over the original order) -> scatter.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdlib.h>

#include "sort_scan.cuh"

namespace pio {

// The 64-bit hash of the string p[0 .. n): FNV-1a, then a splitmix64 finaliser; & mask (all ones unless
// PIO_IDS_HASH_BITS shortens it, ids_hash_mask).  ids_encode and the event index (events_index.cuh) both hash with it.
__device__ __forceinline__ uint64_t ids_hash(const uint8_t* p, long long n, uint64_t mask) {
  uint64_t hsh = 0xcbf29ce484222325ull;
  for (long long b = 0; b < n; ++b) {
    hsh ^= (uint64_t)p[b];
    hsh *= 0x100000001b3ull;
  }
  hsh ^= hsh >> 30; hsh *= 0xBF58476D1CE4E5B9ull;
  hsh ^= hsh >> 27; hsh *= 0x94D049BB133111EBull;
  hsh ^= hsh >> 31;
  return hsh & mask;
}

// tests: PIO_IDS_HASH_BITS = b (1 <= b < 64) keeps the low b bits of the hash, so that different strings collide on
// purpose
inline uint64_t ids_hash_mask() {
  if (const char* hb = getenv("PIO_IDS_HASH_BITS")) {
    const int b = atoi(hb);
    if (b >= 1 && b < 64) return (1ull << b) - 1ull;
  }
  return ~0ull;
}

__global__ void ids_hash_kernel(const uint8_t* __restrict__ bytes, const long long* __restrict__ off, long long n,
                                uint64_t* __restrict__ keys, uint32_t* __restrict__ pay, uint64_t mask) {
  const long long e = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (e >= n) return;
  keys[e] = ids_hash(bytes + off[e], off[e + 1] - off[e], mask);
  pay[e] = (uint32_t)e;
}

__device__ __forceinline__ bool ids_same(const uint8_t* bytes, const long long* off, uint32_t a, uint32_t b) {
  const long long la = off[a + 1] - off[a], lb = off[b + 1] - off[b];
  if (la != lb) return false;
  const uint8_t* pa = bytes + off[a];
  const uint8_t* pb = bytes + off[b];
  for (long long t = 0; t < la; ++t)
    if (pa[t] != pb[t]) return false;
  return true;
}

__global__ void ids_runflag_kernel(const uint64_t* __restrict__ keys, long long n, uint32_t* __restrict__ flag) {
  const long long s = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (s < n) flag[s] = (s == 0 || keys[s] != keys[s - 1]) ? 1u : 0u;
}
// rid = exclusive scan of the run flags (+ flag - 1 = run id); run start of every run
__global__ void ids_runstart_kernel(const uint64_t* __restrict__ keys, const uint32_t* __restrict__ rid_ex, long long n,
                                    uint32_t* __restrict__ run_start) {
  const long long s = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (s < n && (s == 0 || keys[s] != keys[s - 1])) run_start[rid_ex[s]] = (uint32_t)s;
}
// head[s] = sorted position of the first element of s's run whose bytes equal those of s
__global__ void ids_head_kernel(const uint64_t* __restrict__ keys, const uint32_t* __restrict__ pay,
                                const uint32_t* __restrict__ rid_ex, const uint32_t* __restrict__ run_start,
                                const uint8_t* __restrict__ bytes, const long long* __restrict__ off, long long n,
                                uint32_t* __restrict__ head, uint32_t* __restrict__ ishead) {
  const long long s = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (s >= n) return;
  const bool starts = s == 0 || keys[s] != keys[s - 1];
  const uint32_t r = starts ? rid_ex[s] : rid_ex[s] - 1u;   // exclusive scan of the flags: past the start it is run id + 1
  uint32_t hd = run_start[r];
  const uint32_t me = pay[s];
  while (hd < (uint32_t)s && !ids_same(bytes, off, pay[hd], me)) ++hd;   // only two strings sharing a hash ever loop
  head[s] = hd;
  ishead[s] = hd == (uint32_t)s ? 1u : 0u;
}
// group g (in hash order) -> original position of its first occurrence; mark that position
__global__ void ids_firstpos_kernel(const uint32_t* __restrict__ pay, const uint32_t* __restrict__ ishead,
                                    const uint32_t* __restrict__ gid_ex, long long n, uint32_t* __restrict__ firstpos,
                                    uint32_t* __restrict__ isfirst) {
  const long long s = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (s < n && ishead[s]) {
    firstpos[gid_ex[s]] = pay[s];
    isfirst[pay[s]] = 1u;
  }
}
__global__ void ids_assign_kernel(const uint32_t* __restrict__ pay, const uint32_t* __restrict__ head,
                                  const uint32_t* __restrict__ oid_ex /* by original position */, long long n,
                                  int* __restrict__ out_index, long long* __restrict__ out_first) {
  const long long s = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (s >= n) return;
  const uint32_t first = pay[head[s]];          // original position of the group's first occurrence
  const uint32_t id = oid_ex[first];
  out_index[pay[s]] = (int)id;
  if (head[s] == (uint32_t)s && out_first) out_first[id] = (long long)first;
}

}  // namespace pio
