// events_fold.cuh -- LEventAggregator's $set / $unset / $delete fold (storage.py, LEventAggregator._fold) over event
// columns, restricted to the tracked keys of the keyed scan (DESIGN.md section 3.2).
//
// With the events of one entity in (eventTime, file order) -- Python's sorted() is stable -- the fold reduces to "last
// toucher" rules:
//   exists           the entity's last $set comes after its last $delete
//   winner of key k  the last event among {$delete, $set with k present, $unset with k present}; the key holds that
//                    $set's value if it is a $set, and is absent otherwise (an $unset without state is a no-op and
//                    leaves k absent as well)
//   first / last     min / max eventTime over all three kinds, also before a $delete
//
//   entity numbers   ids_encode.cuh, in order of first occurrence
//   fold_time_key_kernel, radix_sort_pairs     stable sort by time (sign bit flipped: times before 1970 are negative)
//   fold_entity_key_kernel, radix_sort_pairs   stable sort by entity: the order is now (entity, time, line)
//   fold_reduce_kernel     per sorted position: segment ends, and atomicMax of sorted positions for the last $set,
//                          the last $delete and each key's last toucher (a max does not depend on the order of atomics)
//   fold_finish_kernel     per entity: exists, first / last time, winning event per key
// The result is the same from run to run.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

namespace pio {

constexpr int FOLD_SET = 0, FOLD_UNSET = 1, FOLD_DELETE = 2;

__global__ void fold_time_key_kernel(const long long* __restrict__ time_us, long long n, uint64_t* __restrict__ key,
                                     uint32_t* __restrict__ pay) {
  const long long e = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (e >= n) return;
  key[e] = (uint64_t)time_us[e] ^ (1ull << 63);
  pay[e] = (uint32_t)e;
}

__global__ void fold_entity_key_kernel(const uint32_t* __restrict__ pay, const int* __restrict__ ent, long long n,
                                       uint64_t* __restrict__ key) {
  const long long s = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (s < n) key[s] = (uint64_t)(uint32_t)ent[pay[s]];
}

// ent_key: entity per sorted position; seg_first / seg_last: first / last sorted position per entity; last_set,
// last_del, win (n_ent x nk): -1, then the largest sorted position of the event kinds they stand for
__global__ void fold_reduce_kernel(const uint64_t* __restrict__ ent_key, const uint32_t* __restrict__ pay,
                                   const int32_t* __restrict__ code, const uint8_t* __restrict__ present, int nk,
                                   long long n, int* __restrict__ seg_first, int* __restrict__ seg_last,
                                   int* __restrict__ last_set, int* __restrict__ last_del, int* __restrict__ win) {
  const long long s = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (s >= n) return;
  const uint32_t g = (uint32_t)ent_key[s];
  if (s == 0 || (uint32_t)ent_key[s - 1] != g) seg_first[g] = (int)s;
  if (s == n - 1 || (uint32_t)ent_key[s + 1] != g) seg_last[g] = (int)s;
  const uint32_t e = pay[s];
  const int c = code[e];
  if (c == FOLD_SET) atomicMax(last_set + g, (int)s);
  if (c == FOLD_DELETE) atomicMax(last_del + g, (int)s);
  const uint32_t pm = nk ? present[e] : 0u;
  for (int q = 0; q < nk; ++q)
    if (c == FOLD_DELETE || ((pm >> q) & 1u)) atomicMax(win + (long long)g * nk + q, (int)s);
}

__global__ void fold_finish_kernel(const uint32_t* __restrict__ pay, const int32_t* __restrict__ code,
                                   const long long* __restrict__ time_us, const int* __restrict__ seg_first,
                                   const int* __restrict__ seg_last, const int* __restrict__ last_set,
                                   const int* __restrict__ last_del, const int* __restrict__ win, int nk, long long n_ent,
                                   uint8_t* __restrict__ exists, long long* __restrict__ first_us,
                                   long long* __restrict__ last_us, long long* __restrict__ winner) {
  const long long g = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (g >= n_ent) return;
  exists[g] = last_set[g] > last_del[g];
  first_us[g] = time_us[pay[seg_first[g]]];
  last_us[g] = time_us[pay[seg_last[g]]];
  for (int q = 0; q < nk; ++q) {
    const int w = win[g * nk + q];
    winner[g * nk + q] = w >= 0 && code[pay[w]] == FOLD_SET ? (long long)pay[w] : -1ll;
  }
}

}  // namespace pio
