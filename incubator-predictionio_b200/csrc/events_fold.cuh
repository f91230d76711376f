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

// ---- the fold of every key (pio_events_fold_props) ------------------------------------------------------------------
// The events are numbered and sorted as above; each event's records (one per key of its `properties`, in object order)
// are keyed by an interned key code (ids_encode.cuh) and sorted stably by the event's sorted position, then by (entity,
// key code): the order is (entity, key, time, line, index in the object).  Per (entity, key) segment, with positions in
// that order ("last toucher" rules, extended to dict order):
//   remover      max(the entity's last $delete, the segment's last $unset)     (sorted event positions)
//   value        the segment's last $set record; the key is present iff its event comes after the remover
//   place        the segment's first $set record after the remover: dict order is (its event, its index in the object)
// $delete records are ignored.  Among events at the latest instant, lastUpdated is the first in (time, line) order, as
// the strict ">" of LEventAggregator._fold keeps it; firstUpdated is the first event of the entity.
// Maxima and minima of positions only: the result does not depend on the order of atomics.

__global__ void fold_rank_kernel(const uint32_t* __restrict__ pay, long long n, uint32_t* __restrict__ rank) {
  const long long s = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (s < n) rank[pay[s]] = (uint32_t)s;
}

// last_time[g] = the first sorted position of the entity's last instant
__global__ void fold_last_time_kernel(const uint64_t* __restrict__ ent_key, const uint32_t* __restrict__ pay,
                                      const long long* __restrict__ time_us, const int* __restrict__ seg_last,
                                      long long n, int* __restrict__ last_time) {
  const long long s = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (s >= n) return;
  const uint32_t g = (uint32_t)ent_key[s];
  const long long ts = time_us[pay[s]];
  if (ts != time_us[pay[seg_last[g]]]) return;
  if (s == 0 || (uint32_t)ent_key[s - 1] != g || time_us[pay[s - 1]] != ts) last_time[g] = (int)s;
}

// per event: the event of each of its records
__global__ void fold_rec_event_kernel(const long long* __restrict__ prop_off, long long n, uint32_t* __restrict__ rec_ev) {
  const long long e = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (e >= n) return;
  for (long long r = prop_off[e]; r < prop_off[e + 1]; ++r) rec_ev[r] = (uint32_t)e;
}

__global__ void fold_rec_rank_key_kernel(const uint32_t* __restrict__ rec_ev, const uint32_t* __restrict__ rank,
                                         long long nr, uint64_t* __restrict__ key, uint32_t* __restrict__ pay) {
  const long long r = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (r >= nr) return;
  key[r] = rank[rec_ev[r]];
  pay[r] = (uint32_t)r;
}

__global__ void fold_rec_key_kernel(const uint32_t* __restrict__ rpay, const uint32_t* __restrict__ rec_ev,
                                    const int* __restrict__ ent, const int* __restrict__ kcode, int kbits, long long nr,
                                    uint64_t* __restrict__ key) {
  const long long p = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (p >= nr) return;
  const uint32_t r = rpay[p];
  key[p] = ((uint64_t)(uint32_t)ent[rec_ev[r]] << kbits) | (uint32_t)kcode[r];
}

__global__ void fold_seg_flag_kernel(const uint64_t* __restrict__ key, long long nr, uint32_t* __restrict__ flag) {
  const long long p = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (p < nr) flag[p] = p == 0 || key[p] != key[p - 1];
}

// seg_id: exclusive scan of the segment heads; the segment of p is seg_id[p] + head[p] - 1
__device__ __forceinline__ uint32_t fold_seg(const uint32_t* head, const uint32_t* seg_id, long long p) {
  return seg_id[p] + head[p] - 1u;
}

// seg_unset: -1, then the last $unset of the segment (sorted event position); seg_set: -1, then its last $set record
__global__ void fold_props_last_kernel(const uint32_t* __restrict__ rpay, const uint32_t* __restrict__ rec_ev,
                                       const uint32_t* __restrict__ rank, const int32_t* __restrict__ code,
                                       const uint32_t* __restrict__ head, const uint32_t* __restrict__ seg_id,
                                       long long nr, int* __restrict__ seg_unset, int* __restrict__ seg_set) {
  const long long p = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (p >= nr) return;
  const uint32_t e = rec_ev[rpay[p]], g = fold_seg(head, seg_id, p);
  const int c = code[e];
  if (c == FOLD_UNSET) atomicMax(seg_unset + g, (int)rank[e]);
  if (c == FOLD_SET) atomicMax(seg_set + g, (int)p);
}

// seg_place: INT_MAX, then the first $set record of the segment after its remover
__global__ void fold_props_place_kernel(const uint32_t* __restrict__ rpay, const uint32_t* __restrict__ rec_ev,
                                        const uint32_t* __restrict__ rank, const int32_t* __restrict__ code,
                                        const int* __restrict__ ent, const int* __restrict__ last_del,
                                        const uint32_t* __restrict__ head, const uint32_t* __restrict__ seg_id,
                                        const int* __restrict__ seg_unset, long long nr, int* __restrict__ seg_place) {
  const long long p = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (p >= nr) return;
  const uint32_t e = rec_ev[rpay[p]];
  if (code[e] != FOLD_SET) return;
  const uint32_t g = fold_seg(head, seg_id, p);
  const int rem = max(seg_unset[g], last_del[ent[e]]);
  if ((int)rank[e] > rem) atomicMin(seg_place + g, (int)p);
}

// per segment: present (then its exclusive scan in w_pos)
__global__ void fold_props_present_kernel(const uint32_t* __restrict__ rpay, const uint32_t* __restrict__ rec_ev,
                                          const uint32_t* __restrict__ rank, const int* __restrict__ ent,
                                          const int* __restrict__ last_del, const int* __restrict__ seg_unset,
                                          const int* __restrict__ seg_set, long long n_seg,
                                          uint32_t* __restrict__ present) {
  const long long g = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (g >= n_seg) return;
  const int p = seg_set[g];
  bool ok = false;
  if (p >= 0) {
    const uint32_t e = rec_ev[rpay[p]];
    ok = (int)rank[e] > max(seg_unset[g], last_del[ent[e]]);
  }
  present[g] = ok;
}

// the winners, keyed by their place in dict order: (sorted event position of the place, index in that event's object)
__global__ void fold_props_winner_kernel(const uint32_t* __restrict__ rpay, const uint32_t* __restrict__ rec_ev,
                                         const uint32_t* __restrict__ rank, const long long* __restrict__ prop_off,
                                         const uint32_t* __restrict__ present, const uint32_t* __restrict__ w_pos,
                                         const int* __restrict__ seg_set, const int* __restrict__ seg_place,
                                         int ibits, long long n_seg, uint64_t* __restrict__ w_key,
                                         uint32_t* __restrict__ w_rec) {
  const long long g = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (g >= n_seg || !present[g]) return;
  const uint32_t r = rpay[seg_place[g]], e = rec_ev[r];
  w_key[w_pos[g]] = ((uint64_t)rank[e] << ibits) | (uint64_t)(r - prop_off[e]);
  w_rec[w_pos[g]] = rpay[seg_set[g]];
}

// winners in dict order -> per-entity counts, caller's record index and key code of each
__global__ void fold_props_out_kernel(const uint32_t* __restrict__ w_rec, const uint32_t* __restrict__ rec_ev,
                                      const int* __restrict__ ent, const int* __restrict__ kcode, long long nw,
                                      uint32_t* __restrict__ count, long long* __restrict__ out_rec,
                                      int* __restrict__ out_key) {
  const long long w = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (w >= nw) return;
  const uint32_t r = w_rec[w];
  atomicAdd(count + ent[rec_ev[r]], 1u);
  out_rec[w] = r;
  out_key[w] = kcode[r];
}

__global__ void fold_props_finish_kernel(const uint32_t* __restrict__ pay, const int* __restrict__ seg_first,
                                         const int* __restrict__ last_time, const int* __restrict__ last_set,
                                         const int* __restrict__ last_del, const uint32_t* __restrict__ w_off,
                                         long long n_ent, uint8_t* __restrict__ exists, long long* __restrict__ first_ev,
                                         long long* __restrict__ last_ev, long long* __restrict__ win_off) {
  const long long g = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (g > n_ent) return;
  win_off[g] = w_off[g];
  if (g == n_ent) return;
  exists[g] = last_set[g] > last_del[g];
  first_ev[g] = pay[seg_first[g]];
  last_ev[g] = pay[last_time[g]];
}

}  // namespace pio
