// als_pair_kernel.cuh -- rank 33..64 half-step, second generation: every warp is an independent worker that
// accumulates the Gramians of TWO destination rows one after the other on the warp-level tensor-core path (mma.sync
// m16n8k16 FP16 with fp32 accumulation, three passes hi*hi + lo*hi + hi*lo of a scaled hi/lo split = fp32-class
// products) and then solves both normal equations at once with the lockstep Cholesky of als_lockstep.cuh (16 lanes
// per matrix).
//
// Differences to the round-1 kernel (als_mma_kernel.cuh: four warps per CTA, one row each):
//   * no CTA-wide barrier: a warp stages its own eight gathered rows per chunk (cp.async, 4-deep ring, 64-float rows
//     with the features XOR-swizzled so that the fragment LDS.32 are conflict-free) and synchronises with __syncwarp
//     only; warps of unrelated rows no longer wait for each other;
//   * the right-hand side is accumulated from the fragment registers (16 FMA per 8 ratings, quad-reduced once per
//     row) instead of a second pass over the staged rows (24 LDS + 16 FMA per chunk);
//   * the solve costs ~1.8 k instead of ~6.4 k warp instructions per row and its 64-step pivot chain is shared by
//     the two matrices;
//   * work-list mode: an item may be a PART of a long row; its partial normal equation goes to global memory in the
//     slot layout and als_finish_pair_kernel adds the parts of a row in fixed order and solves.  Cutting rows above
//     1024 ratings into 512-rating parts is a two-level summation: the per-chunk round-to-nearest accumulation stays
//     short, which keeps the kernel inside the 1e-4 parity bound on rows of thousands of ratings (round 1: 1.1e-4).
// Per-row arithmetic depends on the row and on the half-step's scale exponent alone (sharded runs stay bit-identical:
// every rank derives the exponent from the same replicated source matrix and the same global rating maximum).
//
// Replaces, per destination row: NormalEquation.add + CholeskySolver.solve of Spark 2.4 ml.recommendation.ALS
// (SURVEY.md section 8(c) items 5-6), reached from examples/scala-parallel-recommendation/.../ALSAlgorithm.scala:76-86.
#pragma once
#include <cuda_fp16.h>
#include <cuda_runtime.h>
#include <stdint.h>

#include "als_kernels.cuh"
#include "als_lockstep.cuh"

namespace pio {
namespace pr {

constexpr int KP = 64;
constexpr int CH = 8;                     // ratings per staged chunk (one cp.async stage); a loop step takes two = K 16
constexpr int RSTR = KP;                  // floats per staged source row (features XOR-swizzled by 8 * row)
constexpr int NSTAGE = 4;                 // two stages consumed per step, two in flight
constexpr int STAGE = CH * RSTR;          // floats per stage
constexpr int NTILE = 20;                 // 16x8 accumulator tiles covering the lower triangle of 64x64
using LL = LsLayout<KP>;
constexpr int SLOT_STRIDE = LL::STRIDE;   // 2096 floats: the second matrix starts 16 banks further
constexpr int VSTR = 80;                  // per-matrix stride of the small vectors (== 16 mod 32)
constexpr int PART_FLOATS = LL::SIZE + KP;   // one partial normal equation in global memory: slot + right-hand side
static_assert(NSTAGE * STAGE <= SLOT_STRIDE, "the staging ring lives in the second slot");
static_assert(NSTAGE % 2 == 0, "a loop step consumes two stages");
// per-warp shared memory (floats): two slots (the ring aliases slot 1), b vectors, pivot lines, rating ring
constexpr int W_BVEC = 2 * SLOT_STRIDE;
constexpr int W_COL = W_BVEC + 2 * VSTR;
constexpr int W_MVAL = W_COL + 2 * VSTR;
constexpr int W_FLOATS = W_MVAL + NSTAGE * CH + 8;
constexpr size_t smem_bytes(int warps) { return sizeof(float) * (size_t)W_FLOATS * warps; }

// The FP16 split needs every value below the f16 range: the values X sqrt(c1) (implicit) or X (explicit) of a
// half-step are multiplied by s = 2^e, with e chosen so that max |X sqrt(c1)| s < 2^15.  hi = f16(v) is then finite
// and lo = f16(v - hi) stays a normal f16 down to max / 2^18 (below that its absolute error is under 2^-25 of the
// largest value).  e is clamped so that 2^-2e, which takes the scale out of the accumulators, is a normal float; an
// all-zero source gives e = 0.
__device__ __forceinline__ int split_exponent(float vmax) {
  if (!(vmax > 0.f)) return 0;
  if (isinf(vmax)) return -63;
  int x;
  frexpf(vmax, &x);                       // vmax < 2^x
  const int e = 15 - x;
  return e < -63 ? -63 : e > 63 ? 63 : e;
}
__device__ __forceinline__ float pow2f(int e) { return __int_as_float((127 + e) << 23); }   // -126 <= e <= 127

// max |x[0 .. n)| as float bits, atomicMax-ed into *out (which the caller zeroes): the bound of the FP16 split scale
// (source factors, every half-step) and the rating maximum (once per ingest).  NaNs are ignored.
__global__ void __launch_bounds__(256) abs_max_kernel(const float* __restrict__ x, long long n, unsigned* out) {
  float m = 0.f;
  const long long stride = (long long)gridDim.x * blockDim.x;
  const long long i0 = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  long long tail = 0;
  if ((reinterpret_cast<uintptr_t>(x) & 15) == 0) {
    const long long n4 = n >> 2;
    for (long long i = i0; i < n4; i += stride) {
      const float4 v = __ldg(reinterpret_cast<const float4*>(x) + i);
      m = fmaxf(m, fmaxf(fmaxf(fabsf(v.x), fabsf(v.y)), fmaxf(fabsf(v.z), fabsf(v.w))));
    }
    tail = 4 * n4;
  }
  for (long long i = tail + i0; i < n; i += stride) m = fmaxf(m, fabsf(__ldg(x + i)));
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, o));
  if ((threadIdx.x & 31) == 0) atomicMax(out, __float_as_uint(m));   // non-negative floats order like their bits
}

// D (+)= A B, m16n8k16, f16 inputs, f32 accumulation.  The B fragment is one 64-bit register pair.
__device__ __forceinline__ uint64_t pack2(uint32_t x, uint32_t y) {
  uint64_t r;
  asm("mov.b64 %0, {%1, %2};" : "=l"(r) : "r"(x), "r"(y));
  return r;
}
__device__ __forceinline__ void mma_f16_p(float (&d)[4], const uint32_t (&a)[4], uint64_t b) {
  asm volatile(
      "{\n .reg .b32 b0, b1;\n mov.b64 {b0, b1}, %8;\n"
      "mma.sync.aligned.m16n8k16.row.col.f32.f16.f16.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {b0,b1}, {%0,%1,%2,%3};\n}\n"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3])
      : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(b));
}
// First mma of a chain: C = 0 as an immediate (no registers to clear)
__device__ __forceinline__ void mma_f16_zp(float (&d)[4], const uint32_t (&a)[4], uint64_t b) {
  asm volatile(
      "{\n .reg .b32 b0, b1;\n mov.b64 {b0, b1}, %4;\n"
      "mma.sync.aligned.m16n8k16.row.col.f32.f16.f16.f32 {%0,%1,%2,%3}, {%5,%6,%7,%8}, {b0,b1}, {%9,%9,%9,%9};\n}\n"
      : "=f"(d[0]), "=f"(d[1]), "=f"(d[2]), "=f"(d[3])
      : "l"(b), "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "f"(0.f));
}

// hi/lo split of the pair (a, b) (k, k + 1 of one fragment register): hi = f16(a), f16(b); lo = f16 of the exact
// fp32 remainders.  The intrinsics keep the compiler from contracting the scale multiply into the subtraction.
__device__ __forceinline__ void split2(float a, float b, uint32_t& hi, uint32_t& lo) {
  const __half2 h = __floats2half2_rn(a, b);          // .x (low 16 bits) = a
  const float2 hf = __half22float2(h);
  const __half2 l = __floats2half2_rn(__fsub_rn(a, hf.x), __fsub_rn(b, hf.y));
  hi = *reinterpret_cast<const uint32_t*>(&h);
  lo = *reinterpret_cast<const uint32_t*>(&l);
}

// Accumulates sum c1 y y^T (lower triangle, slot layout) and b of ratings [beg, end) into `slot` / `bv`; a non-null
// `yty` (N x N row-major, global) is added to the lower triangle as the accumulators are written out.
template <bool IMPLICIT>
__device__ __forceinline__ void accumulate_row(const SolveParams& p, long long beg, long long end, float s, float unscale,
                                               const float* __restrict__ yty, float* ring, float* mval, float* slot,
                                               float* bv) {
  const int lane = threadIdx.x & 31;
  const int g = lane >> 2, t = lane & 3;
  const int nchunks = 2 * (int)((end - beg + 2 * CH - 1) / (2 * CH));   // whole steps; the last chunk may be all zero
  const int prow = lane >> 4, psl = lane & 15;     // staging: piece j of this lane = (staged row 2 j + prow, 16-byte slot psl)

  // metadata of the two chunks of a step: lane l holds the index of rating l & 15 and (l < 16) its value
  int nidx;
  float nval;
  auto prefetch_meta = [&](int c) {   // c even
    const long long e = beg + (long long)c * CH + (lane & 15);
    nidx = (c < nchunks && e < end) ? __ldg(p.idx + e) : -1;
    nval = (lane < 2 * CH && c < nchunks && e < end) ? __ldg(p.val + e) : 0.f;
  };
  // staged row r holds feature f at r * RSTR + (f ^ 8 r): 16-byte pieces stay whole, and the fragment loads of rows
  // t and t + 4 at features 16 i + g (+ 8) hit 32 different banks
  auto issue = [&](int c) {   // chunks c, c + 1 from the metadata prefetched for them; rows past the end are zero-filled
    if (c < nchunks) {
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        float* sbuf = ring + ((c + h) % NSTAGE) * STAGE;
#pragma unroll
        for (int j = 0; j < 4; ++j) {
          const int r = 2 * j + prow;
          const int src = __shfl_sync(0xffffffffu, nidx, CH * h + r);
          float4* d4 = reinterpret_cast<float4*>(sbuf + r * RSTR + ((psl * 4) ^ (8 * r)));
          if (src >= 0) cp_async16(d4, p.src + (size_t)src * KP + psl * 4);
          else *d4 = make_float4(0.f, 0.f, 0.f, 0.f);
        }
      }
      if (lane < 2 * CH) mval[(c % NSTAGE) * CH + lane] = nval;
    }
    cp_async_commit();
  };

  float acc[NTILE][4];
#pragma unroll
  for (int i = 0; i < NTILE; ++i)
#pragma unroll
    for (int e = 0; e < 4; ++e) acc[i][e] = 0.f;
  float pb[4][2];             // right-hand side partials: columns 16 i + 8 e + g over the ratings t, t + 4 of the chunks
#pragma unroll
  for (int i = 0; i < 4; ++i) pb[i][0] = pb[i][1] = 0.f;

  // the fragment columns of this lane: feature 16 i + 8 e + g of staged row t sits at column g + xo[(2 i + e) & 3] +
  // 32 ((2 i + e) >> 2), of staged row t + 4 at column g + xo[(2 i + e) & 3] + 32 (1 - ((2 i + e) >> 2))
  int xo[4];
#pragma unroll
  for (int q = 0; q < 4; ++q) xo[q] = g + 8 * (q ^ t);

  prefetch_meta(0);
  issue(0);
  prefetch_meta(2);

#pragma unroll 1
  for (int c = 0; c < nchunks; c += 2) {
    cp_async_wait<0>();
    __syncwarp();
    issue(c + 2);
    prefetch_meta(c + 4);
    const float* XA = ring + (c % NSTAGE) * STAGE + t * RSTR;   // stage A = chunk c (k 0..7), row t
    const float* XB = XA + STAGE;                                // stage B = chunk c + 1 (k 8..15)
    const float* mv = mval + (c % NSTAGE) * CH;
    float wb[4], sc[4];       // ratings t, t + 4 of stage A, then of stage B
    {
      const float r[4] = {mv[t], mv[t + 4], mv[CH + t], mv[CH + t + 4]};
#pragma unroll
      for (int q = 0; q < 4; ++q) {
        wb[q] = r[q];
        sc[q] = s;
        if (IMPLICIT) {
          const float c1 = p.alpha * fabsf(r[q]);
          sc[q] = __fmul_rn(sqrtf(c1), s);
          wb[q] = r[q] > 0.f ? 1.f + c1 : 0.f;
        }
      }
    }
    // f16x2 fragments of m-tile i: register 0 = feature 16i+g, 1 = 16i+8+g of stage A, 2 and 3 the same of stage B;
    // each holds ratings (t, t + 4).  The same registers are the A fragment of m-tile i and, as pairs (0, 2) and
    // (1, 3), the B fragments of n-tiles 2i and 2i+1.
    uint32_t hi[4][4], lo[4][4];
#pragma unroll
    for (int i = 0; i < 4; ++i) {
#pragma unroll
      for (int e = 0; e < 2; ++e) {
        const int q = 2 * i + e;
        const int c0 = xo[q & 3] + 32 * (q >> 2), c4 = 4 * RSTR + xo[q & 3] + 32 * (1 - (q >> 2));
        const float a0 = XA[c0], a4 = XA[c4], b0 = XB[c0], b4 = XB[c4];
        pb[i][e] = fmaf(wb[0], a0, pb[i][e]);
        pb[i][e] = fmaf(wb[1], a4, pb[i][e]);
        pb[i][e] = fmaf(wb[2], b0, pb[i][e]);
        pb[i][e] = fmaf(wb[3], b4, pb[i][e]);
        split2(__fmul_rn(a0, sc[0]), __fmul_rn(a4, sc[1]), hi[i][e], lo[i][e]);
        split2(__fmul_rn(b0, sc[2]), __fmul_rn(b4, sc[3]), hi[i][e + 2], lo[i][e + 2]);
      }
    }
    // D(16i.., 8j..) += A_i B_j for the tiles on or below the diagonal: j <= 2i+1.  The tensor core adds with
    // truncation: only the 16 products of one step are summed inside it (small terms first), the running sum over
    // the steps is a round-to-nearest FADD in registers.
    // n-tile j outermost: its B fragments (two registers each, hi and lo) are formed once and serve every m-tile
    // i >= j/2 below it -- SASS wants the pair in adjacent registers, so each use of a fresh pair costs two MOVs.
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      const int bi = j >> 1, be = j & 1;
      // packed as 64-bit values: the pair is materialised once (two MOVs) and stays adjacent for all its uses
      const uint64_t bh = pack2(hi[bi][be], hi[bi][be + 2]), bl = pack2(lo[bi][be], lo[bi][be + 2]);
#pragma unroll
      for (int i = bi; i < 4; ++i) {
        const int tile = i * (i + 1) + j;               // tiles of m-tile i start at sum_{i' < i} (2 i' + 2) = i (i + 1)
        float d[4];
        mma_f16_zp(d, lo[i], bh);
        mma_f16_p(d, hi[i], bl);
        mma_f16_p(d, hi[i], bh);
        acc[tile][0] += d[0];
        acc[tile][1] += d[1];
        acc[tile][2] += d[2];
        acc[tile][3] += d[3];
      }
    }
  }
  cp_async_wait<0>();
  __syncwarp();   // the ring is dead from here on

  // ---- right-hand side: reduce over the four lanes of a quad (fixed order), lane t == 0 stores -------------------------
#pragma unroll
  for (int i = 0; i < 4; ++i)
#pragma unroll
    for (int e = 0; e < 2; ++e) {
      float v = pb[i][e];
      v += __shfl_xor_sync(0xffffffffu, v, 1);
      v += __shfl_xor_sync(0xffffffffu, v, 2);
      if (t == 0) bv[16 * i + 8 * e + g] = v;
    }
  // ---- accumulators -> slot layout, the scale s^2 taken out (exact: a power of two), YtY added ------------------------
  {
    const float* yl = yty ? yty + g * KP + 2 * t : nullptr;   // YtY(16 i + g (+ 8), 8 j + 2 t (+ 1))
    int tile = 0;
#pragma unroll
    for (int i = 0; i < 4; ++i) {
#pragma unroll
      for (int j = 0; j <= 2 * i + 1; ++j, ++tile) {
        const int cb = j >> 1;
        const int cc = 8 * (j & 1) + 2 * t;           // column inside the 16-wide block (even)
        float d0 = acc[tile][0] * unscale, d1 = acc[tile][1] * unscale;
        float d2 = acc[tile][2] * unscale, d3 = acc[tile][3] * unscale;
        if (yl) {
          const float2 y0 = __ldg(reinterpret_cast<const float2*>(yl + 16 * i * KP + 8 * j));
          const float2 y1 = __ldg(reinterpret_cast<const float2*>(yl + (16 * i + 8) * KP + 8 * j));
          d0 += y0.x; d1 += y0.y;
          d2 += y1.x; d3 += y1.y;
        }
        if (cb < i) {
          // off-diagonal block: two 8-byte stores (rows g and g + 8 of the block)
          *reinterpret_cast<float2*>(slot + LL::offd(i, cb, g, cc)) = make_float2(d0, d1);
          *reinterpret_cast<float2*>(slot + LL::offd(i, cb, g + 8, cc)) = make_float2(d2, d3);
        } else {
          // diagonal block: packed triangle, keep c <= r
          if (cc <= g) slot[LL::diag(i, g, cc)] = d0;
          if (cc + 1 <= g) slot[LL::diag(i, g, cc + 1)] = d1;
          if (cc <= g + 8) slot[LL::diag(i, g + 8, cc)] = d2;
          if (cc + 1 <= g + 8) slot[LL::diag(i, g + 8, cc + 1)] = d3;
        }
      }
    }
  }
  __syncwarp();
}

// identity system for the unused half of the last warp
__device__ __forceinline__ void fill_identity(float* slot, float* bv) {
  const int lane = threadIdx.x & 31;
  for (int o = lane; o < LL::SIZE; o += 32) slot[o] = 0.f;
  __syncwarp();
  for (int r = lane; r < KP; r += 32) {
    slot[LL::at(r, r)] = 1.f;
    bv[r] = 0.f;
  }
  __syncwarp();
}

// WARPS independent workers per CTA.  The only CTA-wide synchronisation is one barrier before the solve: the warps of
// a CTA then walk the (fully unrolled, ~80 KB) lockstep solver together, so that an SM's instruction cache holds a few
// positions of that code instead of twelve (ncu, one-warp CTAs: "no instruction" was the first stall reason of the
// user half-step, 1.7 per issued instruction).
template <bool IMPLICIT, int WARPS>
__global__ void __launch_bounds__(32 * WARPS, 12 / WARPS) als_solve_pair_kernel(const SolveParams p, int n_items) {
  extern __shared__ __align__(16) float smem_all[];
  const int warp = threadIdx.x >> 5;
  float* smem = smem_all + warp * W_FLOATS;
  float* slot0 = smem;
  float* slot1 = smem + SLOT_STRIDE;
  float* ring = slot1;                  // dead whenever slot 1 is written
  float* bvec = smem + W_BVEC;          // [2][VSTR]
  float* colbuf = smem + W_COL;         // [2][VSTR]
  float* mval = smem + W_MVAL;          // [NSTAGE][CH]
  const int lane = threadIdx.x & 31;
  const int grp = lane >> 4;
  const int npairs = (n_items + 1) >> 1;
  const float c1_root_max = IMPLICIT ? sqrtf(p.alpha * __uint_as_float(__ldg(p.absmax + 1))) : 1.f;
  const int e = split_exponent(__uint_as_float(__ldg(p.absmax)) * c1_root_max);
  const float s = pow2f(e), unscale = pow2f(-2 * e);

#pragma unroll 1
  for (int base = blockIdx.x * WARPS; base < npairs; base += gridDim.x * WARPS) {
    const int pair = base + warp;
    int row0 = -1, row1 = -1;
    if (pair < npairs) {
#pragma unroll 1
      for (int h = 0; h < 2; ++h) {
        const int item = 2 * pair + h;
        float* slot = h ? slot1 : slot0;
        float* bv = bvec + h * VSTR;
        if (item >= n_items) {
          fill_identity(slot, bv);
          continue;
        }
        long long beg, end;
        if (p.partial) {
          beg = p.wl_beg[item];
          end = p.wl_end[item];
        } else {
          const int r = p.row_begin + item;
          beg = p.ptr[r];
          end = p.ptr[r + 1];
          if (h) row1 = r;
          else row0 = r;
        }
        // a part carries no YtY: the finish kernel adds it once to the sum of the parts
        accumulate_row<IMPLICIT>(p, beg, end, s, unscale, IMPLICIT && !p.partial ? p.yty : nullptr, ring, mval, slot, bv);
        if (p.partial) {
          // part of a long row: emit the partial normal equation (slot layout + b); als_finish_pair_kernel sums and solves
          float* out = p.partial + (size_t)item * PART_FLOATS;
          for (int o = lane; o < LL::SIZE / 4; o += 32)
            reinterpret_cast<float4*>(out)[o] = reinterpret_cast<const float4*>(slot)[o];
          for (int o = lane; o < KP; o += 32) out[LL::SIZE + o] = bv[o];
          __syncwarp();
        }
      }
    }
    if (p.partial) continue;
    if (WARPS > 1) __syncthreads();
    if (pair < npairs) {
      const int myrow = grp ? row1 : row0;
      const int rr = myrow < 0 ? p.row_begin : myrow;
      chol_lockstep<KP>(grp ? slot1 : slot0, bvec + grp * VSTR, p.lambda * p.nreg[rr], p.k, colbuf + grp * VSTR,
                        p.dst + (size_t)(p.dst_row_offset + rr) * KP, myrow >= 0, p.fail);
      __syncwarp();
    }
  }
}

// Finish kernel for rows that were cut into parts: one warp per two rows; fixed-order sum of the partial normal
// equations (float4 lanes over the slot), then the lockstep solve.
template <bool IMPLICIT>
__global__ void __launch_bounds__(32, 12) als_finish_pair_kernel(const SolveParams p, const int* __restrict__ row_part_ptr,
                                                                  int n_rows) {
  extern __shared__ __align__(16) float smem[];
  float* bvec = smem + W_BVEC;
  float* colbuf = smem + W_COL;
  const int lane = threadIdx.x & 31;
  const int grp = lane >> 4;
  const int npairs = (n_rows + 1) >> 1;
#pragma unroll 1
  for (int pair = blockIdx.x; pair < npairs; pair += gridDim.x) {
#pragma unroll 1
    for (int h = 0; h < 2; ++h) {
      const int r = 2 * pair + h;
      float* slot = smem + h * SLOT_STRIDE;
      float* bv = bvec + h * VSTR;
      if (r >= n_rows) {
        fill_identity(slot, bv);
        continue;
      }
      const int p0 = row_part_ptr[r], p1 = row_part_ptr[r + 1];
      for (int o = lane; o < PART_FLOATS / 4; o += 32) {
        float4 s = make_float4(0.f, 0.f, 0.f, 0.f);
        for (int q = p0; q < p1; ++q) {
          const float4 v = __ldg(reinterpret_cast<const float4*>(p.partial + (size_t)q * PART_FLOATS) + o);
          s.x += v.x; s.y += v.y; s.z += v.z; s.w += v.w;
        }
        if (o < LL::SIZE / 4) reinterpret_cast<float4*>(slot)[o] = s;
        else reinterpret_cast<float4*>(bv)[o - LL::SIZE / 4] = s;
      }
      __syncwarp();
      if (IMPLICIT) {
        ls_add_yty<KP>(slot, p.yty);
        __syncwarp();
      }
    }
    const int myrow = 2 * pair + grp;
    const bool valid = myrow < n_rows;
    const int rr = valid ? myrow : 0;
    chol_lockstep<KP>(smem + grp * SLOT_STRIDE, bvec + grp * VSTR, p.lambda * p.nreg[rr], p.k, colbuf + grp * VSTR,
                      p.dst + (size_t)(p.dst_row_offset + rr) * KP, valid, p.fail);
    __syncwarp();
  }
}

}  // namespace pr
}  // namespace pio
