// als_pair_kernel.cuh -- rank 33..64 half-step, second generation: every warp is an independent worker that
// accumulates the Gramians of TWO destination rows one after the other on the warp-level tensor-core path (mma.sync
// m16n8k8 TF32, three passes hi*hi + lo*hi + hi*lo = fp32-class products) and then solves both normal equations at once
// with the lockstep Cholesky of als_lockstep.cuh (16 lanes per matrix).
//
// Differences to the round-1 kernel (als_mma_kernel.cuh: four warps per CTA, one row each):
//   * no CTA-wide barrier: a warp stages its own eight gathered rows per chunk (cp.async, 3-deep ring, 72-float row
//     stride so that the fragment LDS.32 are conflict-free) and synchronises with __syncwarp only; warps of unrelated
//     rows no longer wait for each other;
//   * the right-hand side is accumulated from the fragment registers (16 FMA per chunk, quad-reduced once per row)
//     instead of a second pass over the staged rows (24 LDS + 16 FMA per chunk);
//   * the solve costs ~1.8 k instead of ~6.4 k warp instructions per row and its 64-step pivot chain is shared by
//     the two matrices;
//   * work-list mode: an item may be a PART of a long row; its partial normal equation goes to global memory in the
//     slot layout and als_finish_pair_kernel adds the parts of a row in fixed order and solves.  Cutting rows above
//     1024 ratings into 512-rating parts is a two-level summation: the per-chunk round-to-nearest accumulation stays
//     short, which keeps the kernel inside the 1e-4 parity bound on rows of thousands of ratings (round 1: 1.1e-4).
// Per-row arithmetic depends on the row alone (sharded runs stay bit-identical).
//
// Replaces, per destination row: NormalEquation.add + CholeskySolver.solve of Spark 2.4 ml.recommendation.ALS
// (SURVEY.md section 8(c) items 5-6), reached from examples/scala-parallel-recommendation/.../ALSAlgorithm.scala:76-86.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include "als_kernels.cuh"
#include "als_lockstep.cuh"

namespace pio {
namespace pr {

constexpr int KP = 64;
constexpr int CH = 8;                     // ratings per chunk = K of one mma
constexpr int RSTR = 72;                  // floats per staged source row (64 + 8 pad)
constexpr int NSTAGE = 3;
constexpr int STAGE = CH * RSTR;          // floats per stage
constexpr int NTILE = 20;                 // 16x8 accumulator tiles covering the lower triangle of 64x64
using LL = LsLayout<KP>;
constexpr int SLOT_STRIDE = LL::STRIDE;   // 2096 floats: the second matrix starts 16 banks further
constexpr int VSTR = 80;                  // per-matrix stride of the small vectors (== 16 mod 32)
constexpr int PART_FLOATS = LL::SIZE + KP;   // one partial normal equation in global memory: slot + right-hand side
static_assert(NSTAGE * STAGE <= SLOT_STRIDE, "the staging ring lives in the second slot");
// per-warp shared memory (floats): two slots (the ring aliases slot 1), b vectors, pivot lines, rating ring
constexpr int W_BVEC = 2 * SLOT_STRIDE;
constexpr int W_COL = W_BVEC + 2 * VSTR;
constexpr int W_MVAL = W_COL + 2 * VSTR;
constexpr int W_FLOATS = W_MVAL + NSTAGE * CH + 8;
constexpr size_t smem_bytes(int warps) { return sizeof(float) * (size_t)W_FLOATS * warps; }

__device__ __forceinline__ void mma_tf32(float (&d)[4], const uint32_t (&a)[4], uint32_t b0, uint32_t b1) {
  asm volatile(
      "mma.sync.aligned.m16n8k8.row.col.f32.tf32.tf32.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};\n"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3])
      : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
}

// First mma of a chain: C = 0 as an immediate (no registers to clear)
__device__ __forceinline__ void mma_tf32_z(float (&d)[4], const uint32_t (&a)[4], uint32_t b0, uint32_t b1) {
  asm volatile(
      "mma.sync.aligned.m16n8k8.row.col.f32.tf32.tf32.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%10,%10,%10,%10};\n"
      : "=f"(d[0]), "=f"(d[1]), "=f"(d[2]), "=f"(d[3])
      : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1), "f"(0.f));
}

// B fragment as one 64-bit register pair
__device__ __forceinline__ uint64_t pack2(uint32_t x, uint32_t y) {
  uint64_t r;
  asm("mov.b64 %0, {%1, %2};" : "=l"(r) : "r"(x), "r"(y));
  return r;
}
__device__ __forceinline__ void mma_tf32_p(float (&d)[4], const uint32_t (&a)[4], uint64_t b) {
  asm volatile(
      "{\n .reg .b32 b0, b1;\n mov.b64 {b0, b1}, %8;\n"
      "mma.sync.aligned.m16n8k8.row.col.f32.tf32.tf32.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {b0,b1}, {%0,%1,%2,%3};\n}\n"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3])
      : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(b));
}
__device__ __forceinline__ void mma_tf32_zp(float (&d)[4], const uint32_t (&a)[4], uint64_t b) {
  asm volatile(
      "{\n .reg .b32 b0, b1;\n mov.b64 {b0, b1}, %4;\n"
      "mma.sync.aligned.m16n8k8.row.col.f32.tf32.tf32.f32 {%0,%1,%2,%3}, {%5,%6,%7,%8}, {b0,b1}, {%9,%9,%9,%9};\n}\n"
      : "=f"(d[0]), "=f"(d[1]), "=f"(d[2]), "=f"(d[3])
      : "l"(b), "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "f"(0.f));
}

// Accumulates sum c1 y y^T (lower triangle, slot layout) and b of ratings [beg, end) into `slot` / `bv`.
template <bool IMPLICIT>
__device__ __forceinline__ void accumulate_row(const SolveParams& p, long long beg, long long end, float* ring,
                                               float* mval, float* slot, float* bv) {
  const int lane = threadIdx.x & 31;
  const int g = lane >> 2, t = lane & 3;
  const int nchunks = (int)((end - beg + CH - 1) / CH);
  const int prow = lane >> 4, psl = lane & 15;     // staging: piece j of this lane = (staged row 2 j + prow, 16-byte slot psl)

  int nidx[4];
  float nval;
  auto prefetch_meta = [&](int c) {
    const long long e0 = beg + (long long)c * CH;
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const long long e = e0 + 2 * j + prow;
      nidx[j] = (c < nchunks && e < end) ? __ldg(p.idx + e) : -1;
    }
    nval = 0.f;
    if (lane < CH && c < nchunks && e0 + lane < end) nval = __ldg(p.val + e0 + lane);
  };
  auto issue = [&](int c) {   // uses the metadata prefetched for chunk c; rows past the end are zero-filled
    if (c < nchunks) {
      float* sbuf = ring + (c % NSTAGE) * STAGE;
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        float4* d4 = reinterpret_cast<float4*>(sbuf + (2 * j + prow) * RSTR + psl * 4);
        if (nidx[j] >= 0) cp_async16(d4, p.src + (size_t)nidx[j] * KP + psl * 4);
        else *d4 = make_float4(0.f, 0.f, 0.f, 0.f);
      }
      if (lane < CH) mval[(c % NSTAGE) * CH + lane] = nval;
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

  prefetch_meta(0);
  issue(0);
  prefetch_meta(1);
  issue(1);
  prefetch_meta(2);

#pragma unroll 1
  for (int c = 0; c < nchunks; ++c) {
    cp_async_wait<1>();
    __syncwarp();
    issue(c + 2);
    prefetch_meta(c + 3);
    const float* X = ring + (c % NSTAGE) * STAGE;
    const float* mv = mval + (c % NSTAGE) * CH;
    const float r0 = mv[t], r1 = mv[t + 4];
    float sc0 = 1.f, sc1 = 1.f, wb0 = r0, wb1 = r1;
    if (IMPLICIT) {
      const float c0 = p.alpha * fabsf(r0), c1 = p.alpha * fabsf(r1);
      sc0 = sqrtf(c0);
      sc1 = sqrtf(c1);
      wb0 = r0 > 0.f ? 1.f + c0 : 0.f;
      wb1 = r1 > 0.f ? 1.f + c1 : 0.f;
    }
    // fragments: v[i][0..3] = X[t][16i+g], X[t][16i+8+g], X[t+4][16i+g], X[t+4][16i+8+g]: the same registers are the A
    // fragment of m-tile i and the B fragments of n-tiles 2i, 2i+1
    uint32_t hi[4][4], lo[4][4];
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      float v[4];
      v[0] = X[t * RSTR + 16 * i + g];
      v[1] = X[t * RSTR + 16 * i + 8 + g];
      v[2] = X[(t + 4) * RSTR + 16 * i + g];
      v[3] = X[(t + 4) * RSTR + 16 * i + 8 + g];
      pb[i][0] = fmaf(wb0, v[0], pb[i][0]);
      pb[i][1] = fmaf(wb0, v[1], pb[i][1]);
      pb[i][0] = fmaf(wb1, v[2], pb[i][0]);
      pb[i][1] = fmaf(wb1, v[3], pb[i][1]);
      if (IMPLICIT) {
        v[0] *= sc0; v[1] *= sc0; v[2] *= sc1; v[3] *= sc1;
      }
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        // Veltkamp split: h = the 11 leading bits of v rounded to nearest (exactly a TF32 value), v - h exact; three
        // FMA-pipe instructions instead of the ALU sequence cvt.rna.tf32 expands to.  |v - h| <= 2^-11 |v|;
        // the dropped lo*lo term is 2^-22.
        // (intrinsics: the compiler must not contract c - (c - v) into FMAs, which would return v itself)
        const float c = __fmul_rn(v[e], 8193.f);       // 2^13 + 1
        const float h = __fsub_rn(c, __fsub_rn(c, v[e]));
        hi[i][e] = __float_as_uint(h);
        lo[i][e] = __float_as_uint(__fsub_rn(v[e], h));
      }
    }
    // D(16i.., 8j..) += A_i B_j for the tiles on or below the diagonal: j <= 2i+1.  The tensor core adds with
    // truncation: only the 8 products of one chunk are summed inside it (small terms first), the running sum over
    // the chunks is a round-to-nearest FADD in registers.
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
        mma_tf32_zp(d, lo[i], bh);
        mma_tf32_p(d, hi[i], bl);
        mma_tf32_p(d, hi[i], bh);
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
  // ---- accumulators -> slot layout ----------------------------------------------------------------------------------------
  {
    int tile = 0;
#pragma unroll
    for (int i = 0; i < 4; ++i) {
#pragma unroll
      for (int j = 0; j <= 2 * i + 1; ++j, ++tile) {
        const int cb = j >> 1;
        const int cc = 8 * (j & 1) + 2 * t;           // column inside the 16-wide block (even)
        if (cb < i) {
          // off-diagonal block: two 8-byte stores (rows g and g + 8 of the block)
          *reinterpret_cast<float2*>(slot + LL::offd(i, cb, g, cc)) = make_float2(acc[tile][0], acc[tile][1]);
          *reinterpret_cast<float2*>(slot + LL::offd(i, cb, g + 8, cc)) = make_float2(acc[tile][2], acc[tile][3]);
        } else {
          // diagonal block: packed triangle, keep c <= r
          if (cc <= g) slot[LL::diag(i, g, cc)] = acc[tile][0];
          if (cc + 1 <= g) slot[LL::diag(i, g, cc + 1)] = acc[tile][1];
          if (cc <= g + 8) slot[LL::diag(i, g + 8, cc)] = acc[tile][2];
          if (cc + 1 <= g + 8) slot[LL::diag(i, g + 8, cc + 1)] = acc[tile][3];
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
        accumulate_row<IMPLICIT>(p, beg, end, ring, mval, slot, bv);
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
      chol_lockstep<KP, IMPLICIT>(grp ? slot1 : slot0, bvec + grp * VSTR, p.yty, p.lambda * p.nreg[rr], p.k,
                                  colbuf + grp * VSTR, p.dst + (size_t)(p.dst_row_offset + rr) * KP, myrow >= 0, p.fail);
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
    }
    const int myrow = 2 * pair + grp;
    const bool valid = myrow < n_rows;
    const int rr = valid ? myrow : 0;
    chol_lockstep<KP, IMPLICIT>(smem + grp * SLOT_STRIDE, bvec + grp * VSTR, p.yty, p.lambda * p.nreg[rr], p.k,
                                colbuf + grp * VSTR, p.dst + (size_t)(p.dst_row_offset + rr) * KP, valid, p.fail);
    __syncwarp();
  }
}

}  // namespace pr
}  // namespace pio
