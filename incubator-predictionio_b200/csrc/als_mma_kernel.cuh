// als_mma_kernel.cuh -- rank 33..64 half-step for SHORT rows: one warp per destination row, Gramian on the warp-level
// tensor-core path (mma.sync m16n8k8 TF32, three passes hi*hi + lo*hi + hi*lo = fp32-class products), then the same
// warp Cholesky as the other kernels.
//
// Why a third kernel: the FP32 kernel (als_kernels.cuh) is bound by shared-memory bandwidth by construction (an 8x8
// register block reads 1 byte of operands per FMA = the SM's 128 B/clk) and spends 137 warp instructions per rating;
// the wgmma kernel (als_tc_kernel.cuh) is built for long rows but needs half of its sixteen warps for the producer
// pipeline, so on short rows (the user side of the headline workload: ~100 ratings per row) it is bound by its eight
// solver warps.  Here every warp gathers, accumulates AND solves its own row: a chunk of 8 ratings costs 16 LDS.32
// (each loaded value serves as A and as B fragment), a cvt/subtract split, 60 mma.sync and 80 FADD -- ~30 warp
// instructions per rating -- and all resident warps take part in the latency-bound Cholesky phase.
//
// Replaces, per destination row: NormalEquation.add + CholeskySolver.solve of Spark 2.4 ml.recommendation.ALS
// (SURVEY.md section 8(c) items 5-6), reached from examples/scala-parallel-recommendation/.../ALSAlgorithm.scala:76-86.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include "als_kernels.cuh"

namespace pio {
namespace mm {

constexpr int KP = 64;
constexpr int WARPS = 4;                 // rows per CTA
constexpr int NT = WARPS * 32;
constexpr int CH = 8;                    // ratings per chunk and row = K of one mma
constexpr int RSTR = 72;                 // floats per staged source row: 64 + 8 pad -> fragment LDS.32 are conflict-free
constexpr int NSTAGE = 3;
constexpr int ROWS = WARPS * CH;         // staged source rows per stage
constexpr int STAGE = ROWS * RSTR;       // floats
constexpr int NF = ROWS * (KP / 4) / NT; // 16-byte copies per thread and stage (4)
constexpr int H = 32, L21S = H + 4;
constexpr int OFF21 = H * (H + 1) / 2, OFF22 = OFF21 + H * L21S, ASLOT = OFF22 + H * (H + 1) / 2;   // packed L layout
constexpr int NTILE = 20;                // 16x8 accumulator tiles covering the lower triangle of 64x64
// ring (dead after the last chunk) and the Cholesky slots share the first region
constexpr int REGION0 = NSTAGE * STAGE > WARPS * ASLOT ? NSTAGE * STAGE : WARPS * ASLOT;
constexpr size_t SMEM_BYTES = sizeof(float) * (size_t)(REGION0 + NSTAGE * ROWS + WARPS * KP + WARPS * 2 * KP + WARPS * KP) +
                              sizeof(long long) * 2 * WARPS + sizeof(int) * WARPS + 16;

__device__ __forceinline__ void mma_tf32(float (&d)[4], const uint32_t (&a)[4], uint32_t b0, uint32_t b1) {
  asm volatile(
      "mma.sync.aligned.m16n8k8.row.col.f32.tf32.tf32.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};\n"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3])
      : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
}

template <bool IMPLICIT>
__global__ void __launch_bounds__(NT, 3) als_solve_mma_kernel(const SolveParams p) {
  extern __shared__ __align__(16) float smem[];
  float* stage = smem;                               // [NSTAGE][ROWS][RSTR]
  float* slots = smem;                               // [WARPS][ASLOT], aliases the ring once it is dead
  float* mval = smem + REGION0;                      // [NSTAGE][ROWS] ratings of the staged rows
  float* bvec = mval + NSTAGE * ROWS;                // [WARPS][KP]
  float* colbuf = bvec + WARPS * KP;                 // [WARPS][2 KP]
  float* dinvb = colbuf + WARPS * 2 * KP;            // [WARPS][KP]
  long long* segb = reinterpret_cast<long long*>((reinterpret_cast<uintptr_t>(dinvb + WARPS * KP) + 15) & ~uintptr_t(15));
  long long* sege = segb + WARPS;
  int* srow = reinterpret_cast<int*>(sege + WARPS);

  const int tid = threadIdx.x, lane = tid & 31, w = tid >> 5;
  const int g = lane >> 2, t = lane & 3;             // mma fragment coordinates
  if (tid < WARPS) {
    const int r = p.row_begin + blockIdx.x * WARPS + tid;
    if (r < p.row_end) {
      segb[tid] = p.ptr[r];
      sege[tid] = p.ptr[r + 1];
      srow[tid] = r;
    } else {
      segb[tid] = 0;
      sege[tid] = 0;
      srow[tid] = -1;
    }
  }
  __syncthreads();
  long long maxlen = 0;
#pragma unroll
  for (int q = 0; q < WARPS; ++q) {
    const long long len = sege[q] - segb[q];
    maxlen = len > maxlen ? len : maxlen;
  }
  const int nchunks = (int)((maxlen + CH - 1) / CH);
  const long long mylen = sege[w] - segb[w];

  // ---- cooperative staging: thread f -> (staged row q = f / 16, 16-byte chunk f % 16); metadata one chunk ahead ----
  int nidx[NF];
  float nval[NF];
  auto prefetch_meta = [&](int c) {
#pragma unroll
    for (int j = 0; j < NF; ++j) {
      const int f = tid + j * NT;
      nidx[j] = -1;
      nval[j] = 0.f;
      if (c < nchunks) {
        const int q = f >> 4;
        const int gg = q / CH, i = q % CH;
        const long long e = segb[gg] + (long long)c * CH + i;
        if (e < sege[gg]) {
          nidx[j] = __ldg(p.idx + e);
          nval[j] = __ldg(p.val + e);
        }
      }
    }
  };
  auto issue = [&](int c) {  // uses nidx/nval prefetched for chunk c; rows past the end of a segment are zero-filled
    float* sbuf = stage + (c % NSTAGE) * STAGE;
    float* mv = mval + (c % NSTAGE) * ROWS;
    if (c < nchunks) {
#pragma unroll
      for (int j = 0; j < NF; ++j) {
        const int f = tid + j * NT;
        const int q = f >> 4, sl = f & 15;
        float4* d4 = reinterpret_cast<float4*>(sbuf + q * RSTR + sl * 4);
        if (nidx[j] >= 0) cp_async16(d4, p.src + (size_t)nidx[j] * KP + sl * 4);
        else *d4 = make_float4(0.f, 0.f, 0.f, 0.f);
        if (sl == 0) mv[q] = nval[j];
      }
    }
    cp_async_commit();
  };

  float acc[NTILE][4];
#pragma unroll
  for (int i = 0; i < NTILE; ++i)
#pragma unroll
    for (int e = 0; e < 4; ++e) acc[i][e] = 0.f;
  float b0 = 0.f, b1 = 0.f;   // right-hand side, columns lane and lane + 32

  prefetch_meta(0);
  issue(0);
  prefetch_meta(1);
  issue(1);
  prefetch_meta(2);

#pragma unroll 1
  for (int c = 0; c < nchunks; ++c) {
    cp_async_wait<1>();
    __syncthreads();
    issue(c + 2);
    prefetch_meta(c + 3);
    if (mylen - (long long)c * CH > 0) {
      const float* X = stage + (c % NSTAGE) * STAGE + (w * CH) * RSTR;   // this warp's 8 gathered rows
      const float* mv = mval + (c % NSTAGE) * ROWS + w * CH;
      // b += wb * y over the 8 ratings (zero-filled rows contribute nothing)
#pragma unroll
      for (int rr = 0; rr < CH; ++rr) {
        const float r = mv[rr];
        float wb;
        if (IMPLICIT) wb = r > 0.f ? 1.f + p.alpha * fabsf(r) : 0.f;
        else wb = r;
        b0 = fmaf(wb, X[rr * RSTR + lane], b0);
        b1 = fmaf(wb, X[rr * RSTR + 32 + lane], b1);
      }
      // fragments: v[i][0..3] = X[t][16i+g], X[t][16i+8+g], X[t+4][16i+g], X[t+4][16i+8+g]  (scaled by sqrt(c1))
      float sc0 = 1.f, sc1 = 1.f;
      if (IMPLICIT) {
        sc0 = sqrtf(p.alpha * fabsf(mv[t]));
        sc1 = sqrtf(p.alpha * fabsf(mv[t + 4]));
      }
      uint32_t hi[4][4], lo[4][4];
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        float v[4];
        v[0] = X[t * RSTR + 16 * i + g] * sc0;
        v[1] = X[t * RSTR + 16 * i + 8 + g] * sc0;
        v[2] = X[(t + 4) * RSTR + 16 * i + g] * sc1;
        v[3] = X[(t + 4) * RSTR + 16 * i + 8 + g] * sc1;
#pragma unroll
        for (int e = 0; e < 4; ++e) {
          uint32_t h;   // round-to-nearest TF32 part: |v - h| <= 2^-11 |v|, v - h exact (the dropped lo*lo term is 2^-22)
          asm("cvt.rna.tf32.f32 %0, %1;" : "=r"(h) : "f"(v[e]));
          hi[i][e] = h;
          lo[i][e] = __float_as_uint(v[e] - __uint_as_float(h));
        }
      }
      // D(16i.., 8j..) += A_i B_j for the tiles on or below the diagonal: j <= 2i+1
      int tile = 0;
#pragma unroll
      for (int i = 0; i < 4; ++i) {
#pragma unroll
        for (int j = 0; j <= 2 * i + 1; ++j, ++tile) {
          const int bi = j >> 1, be = j & 1;   // B fragment of n-tile j = elements (be, be+2) of the values of m-tile j/2
          // the tensor core adds with truncation: only the 8 products of one chunk are summed inside it (small
          // terms first), the running sum over the chunks is a round-to-nearest FADD in registers
          float d[4] = {0.f, 0.f, 0.f, 0.f};
          mma_tf32(d, lo[i], hi[bi][be], hi[bi][be + 2]);
          mma_tf32(d, hi[i], lo[bi][be], lo[bi][be + 2]);
          mma_tf32(d, hi[i], hi[bi][be], hi[bi][be + 2]);
          acc[tile][0] += d[0];
          acc[tile][1] += d[1];
          acc[tile][2] += d[2];
          acc[tile][3] += d[3];
        }
      }
    }
  }
  cp_async_wait<0>();
  __syncthreads();   // the ring is dead: the slots may overwrite it

  // ---- accumulators -> packed lower triangle (layout of chol_solve_warp<..., PACKED_IN>) -------------------------
  float* slot = slots + w * ASLOT;
  auto put = [&](int r, int c, float v) {
    if (c > r) return;
    if (r < H) slot[r * (r + 1) / 2 + c] = v;
    else if (c < H) slot[OFF21 + (r - H) * L21S + c] = v;
    else slot[OFF22 + (r - H) * (r - H + 1) / 2 + (c - H)] = v;
  };
  {
    int tile = 0;
#pragma unroll
    for (int i = 0; i < 4; ++i) {
#pragma unroll
      for (int j = 0; j <= 2 * i + 1; ++j, ++tile) {
        const int r0 = 16 * i + g, c0 = 8 * j + 2 * t;
        put(r0, c0, acc[tile][0]);
        put(r0, c0 + 1, acc[tile][1]);
        put(r0 + 8, c0, acc[tile][2]);
        put(r0 + 8, c0 + 1, acc[tile][3]);
      }
    }
  }
  bvec[w * KP + lane] = b0;
  bvec[w * KP + 32 + lane] = b1;
  __syncwarp();
  const int r = srow[w];
  if (r >= 0 && mylen > 0) {   // rows without ratings own no factor (MLlib emits none)
    chol_solve_warp<KP, 8, 72, IMPLICIT, true>(slot, bvec + w * KP, p.yty, p.lambda * p.nreg[r], p.k, colbuf + w * 2 * KP,
                                               dinvb + w * KP, p.dst + (size_t)(p.dst_row_offset + r) * KP, p.fail);
  }
}

}  // namespace mm
}  // namespace pio
