// events_scan.cuh -- the device scanner of the JSON-lines event file (DESIGN.md section 3.1): one chunk of complete
// lines -> the matched events as columns, in line order, plus the lines the host must parse (event_line.h decides).
//
//   ev_start_flag_kernel   a line starts at byte 0 and after every terminator ("\n", "\r\n", or a lone "\r": Python's
//                          universal newlines)
//   scan_exclusive_u32     line ids (sort_scan.cuh), ev_start_scatter_kernel: line starts
//   ev_parse_smem_kernel   one line per thread through event_line.h, the block's lines staged in shared memory first
//                          (ev_parse_kernel reads global memory instead; PIO_EVENTS_SMEM=0); decoded ids land in a
//                          chunk-sized scratch at the line's own offset (decoded ids are never longer than the line)
//   scan_exclusive_u32 x4  output slots of the matched and fallback lines and of their id bytes
//   ev_compact_kernel      matched events and their id bytes, fallback lines, in line order
// The keyed scan (pio_events_scan_keys) runs the same kernels with KEYS = true: the parse also reports the tracked
// `properties` keys of each line (event_line.h parse_line_keys), one more scan places their token bytes, and the compaction
// copies present / number masks, numbers and token bytes next to the ids.  KEYS = false is the plain scan, unchanged.
// Output order comes from the scans alone: no atomics, the result is deterministic.  A chunk is < 2^31 bytes, so every
// per-chunk count fits the 32-bit scan.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include "event_line.h"
#include "sort_scan.cuh"

namespace pio {

constexpr int EV_THREADS = 256;

__global__ void ev_start_flag_kernel(const uint8_t* __restrict__ t, long long n, uint32_t* __restrict__ flag) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  uint32_t f = 1;
  if (i > 0) {
    const uint8_t p = t[i - 1];
    f = p == '\n' || (p == '\r' && t[i] != '\n');
  }
  flag[i] = f;
}

// starts[0 .. nl) = line starts, starts[nl] = n
__global__ void ev_start_scatter_kernel(const uint32_t* __restrict__ flag, const uint32_t* __restrict__ lid, long long n,
                                        long long nl, uint32_t* __restrict__ starts) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n && flag[i]) starts[lid[i]] = (uint32_t)i;
  if (i == 0) starts[nl] = (uint32_t)n;
}

// line j = [starts[j], starts[j + 1]) without its terminator
__device__ __forceinline__ void ev_line_range(const uint8_t* t, const uint32_t* starts, long long j, uint32_t* b,
                                              uint32_t* e) {
  *b = starts[j];
  uint32_t end = starts[j + 1];
  if (end > *b && t[end - 1] == '\n') {
    --end;
    if (end > *b && t[end - 1] == '\r') --end;
  } else if (end > *b && t[end - 1] == '\r') {
    --end;
  }
  *e = end;
}

struct EvLines {            // per line of the chunk
  uint32_t* is_match;       // then its exclusive scan in match_pos
  uint32_t* is_fb;
  uint32_t* eid_len;
  uint32_t* tid_len;
  uint32_t* match_pos;
  uint32_t* fb_pos;
  uint32_t* eid_pos;
  uint32_t* tid_pos;
  int32_t* code;
  double* value;
  long long* time_us;
  uint8_t* flags;           // bit 0: has value, bit 1: has target id
};

// the tracked keys of the keyed scan: per line of the chunk, then per matched event (unused when KEYS == false)
struct EvKeys {
  ev::KeyList list;         // device copy of the key names
  uint8_t* present;         // per line: KeyValues::present / number
  uint8_t* number;
  double* num;              // per line x list.n
  uint32_t* tok_b;          // per line x list.n, token range relative to the line start
  uint32_t* tok_e;
  uint32_t* tok_len;        // per line: token bytes of a matched line; then its exclusive scan in tok_pos
  uint32_t* tok_pos;
  long long tok_base;       // token bytes of the call before this chunk
  uint8_t* o_present;       // per matched event
  uint8_t* o_number;
  double* o_num;            // per matched event x list.n
  long long* o_tok_off;     // per matched event x list.n: start of the token in the caller's token column
  uint8_t* o_tok;
};

__device__ __forceinline__ void ev_store(const EvLines& L, long long j, const ev::Result& r) {
  const bool m = r.outcome == ev::MATCHED;
  L.is_match[j] = m;
  L.is_fb[j] = r.outcome == ev::FALLBACK;
  L.eid_len[j] = m ? (uint32_t)r.eid_len : 0u;
  L.tid_len[j] = m ? (uint32_t)r.tid_len : 0u;
  L.code[j] = r.code;
  L.value[j] = r.value;
  L.time_us[j] = r.time_us;
  L.flags[j] = (uint8_t)(r.has_value | (r.has_target << 1));
}

__device__ __forceinline__ void ev_store_keys(const EvKeys& K, long long j, const ev::Result& r, const ev::KeyValues& kv) {
  const int nk = K.list.n;
  uint32_t len = 0;
  K.present[j] = (uint8_t)kv.present;
  K.number[j] = (uint8_t)kv.number;
  for (int q = 0; q < nk; ++q) {
    K.num[j * nk + q] = kv.num[q];
    K.tok_b[j * nk + q] = (uint32_t)kv.tok_b[q];
    K.tok_e[j * nk + q] = (uint32_t)kv.tok_e[q];
    len += (uint32_t)(kv.tok_e[q] - kv.tok_b[q]);
  }
  K.tok_len[j] = r.outcome == ev::MATCHED ? len : 0u;
}

// the parse of one line, stored
template <bool KEYS>
__device__ __forceinline__ void ev_parse_store(const uint8_t* line, int n, const ev::Filter& f, uint8_t* scratch,
                                               const EvLines& L, const EvKeys& K, long long j) {
  if constexpr (KEYS) {
    ev::KeyValues kv;
    const ev::Result r = ev::parse_line_keys(line, n, f, K.list, scratch, &kv);
    ev_store(L, j, r);
    ev_store_keys(K, j, r, kv);
  } else {
    ev_store(L, j, ev::parse_line(line, n, f, scratch));
  }
}

// one line per thread, read from global memory
template <bool KEYS>
__global__ void __launch_bounds__(EV_THREADS)
ev_parse_kernel(const uint8_t* __restrict__ t, const uint32_t* __restrict__ starts, long long nl, const ev::Filter f,
                uint8_t* __restrict__ scratch, EvLines L, const EvKeys K) {
  const long long j = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (j >= nl) return;
  uint32_t b, e;
  ev_line_range(t, starts, j, &b, &e);
  ev_parse_store<KEYS>(t + b, (int)(e - b), f, scratch + b, L, K, j);
}

// The same parse with the block's lines first copied into shared memory by the whole block in coalesced 16-byte loads
// (one thread per line otherwise reads its own line byte by byte, 256 lines apart).  A block whose lines do not fit
// reads global memory like ev_parse_kernel.  `t` must be 16-byte aligned.
constexpr int EV_SMEM_BYTES = 64 * 1024;

template <bool KEYS>
__global__ void __launch_bounds__(EV_THREADS)
ev_parse_smem_kernel(const uint8_t* __restrict__ t, const uint32_t* __restrict__ starts, long long nl,
                     const ev::Filter f, uint8_t* __restrict__ scratch, EvLines L, const EvKeys K) {
  extern __shared__ __align__(16) uint8_t ev_sm[];
  const long long j0 = (long long)blockIdx.x * blockDim.x;
  const long long j1 = j0 + blockDim.x < nl ? j0 + blockDim.x : nl;
  const uint32_t a0 = starts[j0] & ~15u, b1 = starts[j1];
  const bool staged = b1 - a0 <= (uint32_t)EV_SMEM_BYTES;   // the same for every thread of the block
  if (staged) {
    const uint32_t n16 = (b1 - a0) / 16;
    const uint4* src = reinterpret_cast<const uint4*>(t + a0);
    uint4* dst = reinterpret_cast<uint4*>(ev_sm);
    for (uint32_t k = threadIdx.x; k < n16; k += blockDim.x) dst[k] = src[k];
    for (uint32_t k = a0 + n16 * 16 + threadIdx.x; k < b1; k += blockDim.x) ev_sm[k - a0] = t[k];
  }
  __syncthreads();
  const long long j = j0 + threadIdx.x;
  if (j >= nl) return;
  uint32_t b, e;
  ev_line_range(t, starts, j, &b, &e);
  ev_parse_store<KEYS>(staged ? ev_sm + (b - a0) : t + b, (int)(e - b), f, scratch + b, L, K, j);
}

struct EvOut {              // device output of one chunk, indexed by the chunk's match / fallback / byte slots
  long long* line;
  int32_t* code;
  double* value;
  uint8_t* flags;
  long long* time_us;
  long long* eid_off;       // start offset of each id in the caller's id column
  uint8_t* eid_bytes;
  long long* tid_off;
  uint8_t* tid_bytes;
  long long* fb_line;
  long long* fb_begin;      // byte range of the line without its terminator, in the caller's text
  long long* fb_end;
};

// bases: lines, text bytes and id bytes of the call before this chunk
struct EvBase {
  long long line, byte, eid, tid;
};

template <bool KEYS>
__global__ void __launch_bounds__(EV_THREADS)
ev_compact_kernel(const uint8_t* __restrict__ t, const uint32_t* __restrict__ starts, long long nl, const EvBase base,
                  const uint8_t* __restrict__ scratch, const EvLines L, EvOut o, const EvKeys K) {
  const long long j = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (j >= nl) return;
  if (L.is_match[j]) {
    const uint32_t k = L.match_pos[j];
    o.line[k] = base.line + j;
    o.code[k] = L.code[j];
    o.value[k] = L.value[j];
    o.flags[k] = L.flags[j];
    o.time_us[k] = L.time_us[j];
    const uint32_t b = starts[j], ne = L.eid_len[j], nt = L.tid_len[j], pe = L.eid_pos[j], pt = L.tid_pos[j];
    o.eid_off[k] = base.eid + pe;
    o.tid_off[k] = base.tid + pt;
    for (uint32_t q = 0; q < ne; ++q) o.eid_bytes[pe + q] = scratch[b + q];
    for (uint32_t q = 0; q < nt; ++q) o.tid_bytes[pt + q] = scratch[b + ne + q];
    if constexpr (KEYS) {   // token bytes straight from the text, in line order like the ids
      const int nk = K.list.n;
      K.o_present[k] = K.present[j];
      K.o_number[k] = K.number[j];
      uint32_t at = K.tok_pos[j];
      for (int q = 0; q < nk; ++q) {
        const uint32_t tb = K.tok_b[j * nk + q], te = K.tok_e[j * nk + q];
        K.o_num[(long long)k * nk + q] = K.num[j * nk + q];
        K.o_tok_off[(long long)k * nk + q] = K.tok_base + at;
        for (uint32_t c = tb; c < te; ++c) K.o_tok[at++] = t[b + c];
      }
    }
  } else if (L.is_fb[j]) {
    const uint32_t k = L.fb_pos[j];
    uint32_t b, e;
    ev_line_range(t, starts, j, &b, &e);
    o.fb_line[k] = base.line + j;
    o.fb_begin[k] = base.byte + b;
    o.fb_end[k] = base.byte + e;
  }
}

// totals of the chunk: matched events, fallback lines, entityId bytes, targetEntityId bytes
__global__ void ev_totals_kernel(const EvLines L, long long nl, uint32_t* __restrict__ out) {
  const long long j = nl - 1;
  out[0] = L.match_pos[j] + L.is_match[j];
  out[1] = L.fb_pos[j] + L.is_fb[j];
  out[2] = L.eid_pos[j] + L.eid_len[j];
  out[3] = L.tid_pos[j] + L.tid_len[j];
}

}  // namespace pio
