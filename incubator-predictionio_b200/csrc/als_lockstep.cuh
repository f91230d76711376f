// als_lockstep.cuh -- the per-row solve of the ALS half-step (MLlib's CholeskySolver.solve: dppsv on the packed normal
// equation, SURVEY.md 8(c)-6; reached from examples/scala-parallel-recommendation/.../ALSAlgorithm.scala:76-86), as a
// LOCKSTEP warp routine: N/4 lanes own one N x N matrix (four rows each, dealt cyclically), so a warp factorises
// 32/(N/4) matrices at once -- two for rank 64, one for rank 128 -- through one instruction stream.
//
// Why: the round-1 routine (chol_solve_warp: one warp per 64 x 64 matrix, right-looking by single columns, half of the
// matrix in registers) needed ~6.4 k warp instructions and ~50-60 k cycles per matrix -- 64 column steps whose
// shuffle -> rsqrt -> store -> sync -> load -> FMA chain cannot overlap -- and was ~45 % of the dominant launch at
// 0.1 IPC.  Here the 64 pivot steps are shared by two matrices (the chain costs half per matrix), the work between
// pivots is panel-blocked (left-looking by 16-column panels: the update of a panel from the finished columns is a
// stream of independent FMAs fed by broadcast LDS.128), the triangular waste shrinks (16 instead of 32 lanes per
// matrix), no shuffle is on the pivot chain (the pivot column goes through a 128-byte shared line that every lane
// reads back), and forward substitution rides along as one more column.  ~3.6 k warp instructions per matrix.
//
// Matrix layout in shared memory ("slot", LsLayout): 16 x 16 blocks of the lower triangle.  Off-diagonal blocks are
// row-major with the four 16-byte chunks of a row XOR-swizzled by the row bits, so that (a) a lane group reading one
// row each (LDS.128), (b) the mma.sync accumulator dump (STS.64) and (c) a row read across lanes (LDS.32, back
// substitution) are all bank-conflict-free; diagonal blocks are packed triangles (136 floats).  2080 floats for N = 64.
// The second matrix of a warp sits 16 words (mod 32) further, so both halves of the warp hit disjoint banks.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

namespace pio {

template <int N>
struct LsLayout {
  static constexpr int NBK = N / 16;
  static constexpr int NOFF = NBK * (NBK - 1) / 2;
  static constexpr int DIAG0 = NOFF * 256;
  static constexpr int SIZE = DIAG0 + NBK * 136;          // floats per matrix
  static constexpr int STRIDE = SIZE + ((SIZE % 32) == 16 ? 0 : (48 - SIZE % 32) % 32);  // == 16 (mod 32)
  __host__ __device__ static constexpr int swz(int rr) { return ((rr >> 1) & 1) * 2 + ((rr >> 2) & 1); }
  // block (rb, cb), rb > cb
  __host__ __device__ static constexpr int offd_base(int rb, int cb) { return (rb * (rb - 1) / 2 + cb) * 256; }
  __host__ __device__ static constexpr int offd(int rb, int cb, int rr, int cc) {
    return offd_base(rb, cb) + rr * 16 + 4 * ((cc >> 2) ^ swz(rr)) + (cc & 3);
  }
  __host__ __device__ static constexpr int diag(int rb, int rr, int cc) { return DIAG0 + rb * 136 + rr * (rr + 1) / 2 + cc; }
  // element (r, c), c <= r
  __host__ __device__ static constexpr int at(int r, int c) {
    return (r >> 4) == (c >> 4) ? diag(r >> 4, r & 15, c & 15) : offd(r >> 4, c >> 4, r & 15, c & 15);
  }
};

__device__ __forceinline__ float ls_rsqrt(float x) {
  float r;
  asm("rsqrt.approx.ftz.f32 %0, %1;" : "=f"(r) : "f"(x));
  return r;
}

// slot += YtY on the lower triangle (yty: N x N row-major, global), by all 32 lanes.  Implicit feedback adds YtY once
// per matrix where the slot is filled from parts, so that the solver's panel loads stay in shared memory.
template <int N>
__device__ __forceinline__ void ls_add_yty(float* __restrict__ slot, const float* __restrict__ yty) {
  using LL = LsLayout<N>;
  const int lane = threadIdx.x & 31;
  for (int o = lane; o < LL::NOFF * 64; o += 32) {     // off-diagonal blocks, one 16-byte piece of a row per step
    const int b = o >> 6, rr = (o >> 2) & 15, cg = o & 3;
    int rb = 1;
    while (rb * (rb + 1) / 2 <= b) ++rb;               // block b = rb (rb - 1) / 2 + cb
    const int cb = b - rb * (rb - 1) / 2;
    float4* d = reinterpret_cast<float4*>(slot + LL::offd_base(rb, cb) + rr * 16 + 4 * (cg ^ LL::swz(rr)));
    const float4 y = __ldg(reinterpret_cast<const float4*>(yty + (size_t)(16 * rb + rr) * N + 16 * cb + 4 * cg));
    float4 v = *d;
    v.x += y.x; v.y += y.y; v.z += y.z; v.w += y.w;
    *d = v;
  }
  for (int o = lane; o < LL::NBK * 256; o += 32) {     // diagonal blocks, c <= r
    const int rb = o >> 8, rr = (o >> 4) & 15, cc = o & 15;
    if (cc <= rr) slot[LL::diag(rb, rr, cc)] += __ldg(yty + (size_t)(16 * rb + rr) * N + 16 * rb + cc);
  }
}

// Solves (A + ridge I) x = b for the matrix of this lane's group.
//   slot   : this group's matrix in LsLayout<N> (lower triangle; implicit feedback: sum c y y^T + YtY); destroyed (L is
//            written over it)
//   bvec   : this group's right-hand side (N floats, shared memory)
//   ridge  : lambda * n; dimensions >= k get a unit diagonal
//   colbuf : this group's pivot line, 2 x 32 floats of shared memory
//   dst_row: N floats (global); written only if `valid` (a warp whose second matrix is a dummy still runs the code)
// All 32 lanes must call it together.
template <int N>
__device__ __forceinline__ void chol_lockstep(float* __restrict__ slot, const float* __restrict__ bvec, float ridge, int k,
                                              float* __restrict__ colbuf, float* __restrict__ dst_row, bool valid,
                                              int* __restrict__ fail) {
  using LL = LsLayout<N>;
  constexpr int LANES = N / 4;        // lanes per matrix
  constexpr int Q = LANES / 16;       // 16-row blocks per row slot (1: N = 64, 2: N = 128)
  constexpr int NBK = N / 16;
  static_assert(N == 64 || N == 128, "lockstep solver: N = 64 (two matrices per warp) or 128 (one)");
  const int lane = threadIdx.x & 31;
  const int l = lane % LANES, lq = l >> 4, lr = l & 15;
  const int sw = LL::swz(lr);
  float bb[4], yv[4], dv[4];
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    bb[i] = bvec[i * LANES + l];
    yv[i] = 0.f;
    dv[i] = 0.f;
  }
  bool bad = false;
  __syncwarp();

#pragma unroll
  for (int p = 0; p < NBK; ++p) {
    constexpr int dummy = 0;
    (void)dummy;
    const int sp = p / Q;                               // row slot that holds the panel's diagonal block
    const bool isdiag = (Q == 1) || (lq == (p % Q));    // this lane's slot-sp row lies in the diagonal block
    float a[4][16];
    // ---- load the panel: rows at or below the diagonal block, 16 columns --------------------------------------
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      if (i < sp) continue;
      const int bi = i * Q + lq;                        // block row of this lane's row in slot i
      const int r = i * LANES + l;
      if (i == sp) {
        // diagonal block (packed) for the lanes in it, the block below for the others (N = 128, even p)
#pragma unroll
        for (int c = 0; c < 16; ++c) {
          float v = 0.f;
          if (bi == p) {
            if (c <= lr) v = slot[LL::diag(p, lr, c)];
          } else if (bi > p) {
            v = slot[LL::offd(bi, p, lr, c)];
          }
          a[i][c] = v;
        }
      } else {
        const float* rowp = slot + LL::offd_base(bi, p) + lr * 16;
#pragma unroll
        for (int cg = 0; cg < 4; ++cg) {
          const float4 v = *reinterpret_cast<const float4*>(rowp + 4 * (cg ^ sw));
          a[i][4 * cg + 0] = v.x; a[i][4 * cg + 1] = v.y; a[i][4 * cg + 2] = v.z; a[i][4 * cg + 3] = v.w;
        }
      }
      if (i == sp) {
#pragma unroll
        for (int c = 0; c < 16; ++c)
          if (bi == p && c == lr) a[i][c] += ridge + (r >= k ? 1.f : 0.f);
      }
    }
    // ---- left-looking update from the finished block columns: a[i][c] -= sum_t L[row_i][t] * L[16p+c][t] ---------
    if (p > 0) {
#pragma unroll 1
      for (int q = 0; q < p; ++q) {
        const float* dblk = slot + LL::offd_base(p, q);
        const float* own[4];
#pragma unroll
        for (int i = 0; i < 4; ++i) {
          int bi = i * Q + lq;
          if (bi < p) bi = p;                           // rows above the panel compute (unused) garbage in bounds
          own[i] = slot + LL::offd_base(bi, q) + lr * 16;
        }
#pragma unroll 1
        for (int tg = 0; tg < 4; ++tg) {
          float4 o[4];
#pragma unroll
          for (int i = 0; i < 4; ++i)
            if (i >= sp) o[i] = *reinterpret_cast<const float4*>(own[i] + 4 * (tg ^ sw));
#pragma unroll
          for (int c = 0; c < 16; ++c) {
            const float4 d = *reinterpret_cast<const float4*>(dblk + c * 16 + 4 * (tg ^ LL::swz(c)));   // broadcast
#pragma unroll
            for (int i = 0; i < 4; ++i) {
              if (i < sp) continue;
              float v = a[i][c];
              v = fmaf(-o[i].x, d.x, v);
              v = fmaf(-o[i].y, d.y, v);
              v = fmaf(-o[i].z, d.z, v);
              v = fmaf(-o[i].w, d.w, v);
              a[i][c] = v;
            }
          }
        }
      }
    }
    // ---- factorise the panel column by column; b rides along (forward substitution) ------------------------------
#pragma unroll
    for (int j = 0; j < 16; ++j) {
      float* cb = colbuf + (j & 1) * 32;
      if (isdiag) {
        cb[lr] = a[sp][j];
        cb[16 + lr] = bb[sp];
      }
      __syncwarp();
      float col[16];
#pragma unroll
      for (int cg = j / 4; cg < 4; ++cg) {
        const float4 v = *reinterpret_cast<const float4*>(cb + 4 * cg);
        col[4 * cg + 0] = v.x; col[4 * cg + 1] = v.y; col[4 * cg + 2] = v.z; col[4 * cg + 3] = v.w;
      }
      const float bg = cb[16 + j];
      float d = col[j];
      if (!(d > 0.f)) { bad = true; d = 1.f; }
      float inv = ls_rsqrt(d);
      inv = inv * (1.5f - 0.5f * d * inv * inv);
      const float inv2 = inv * inv;
      const float z = inv2 * bg;
      if (isdiag && lr == j) {
        yv[sp] = bg * inv;
        dv[sp] = inv;
      }
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        if (i < sp) continue;
        const float aj = a[i][j];
        const float w = aj * inv2;
        if (i == sp) {
          const int bi = i * Q + lq;
          if (bi > p || (bi == p && lr > j)) bb[i] = fmaf(-aj, z, bb[i]);
        } else {
          bb[i] = fmaf(-aj, z, bb[i]);
        }
        a[i][j] = aj * inv;
#pragma unroll
        for (int c = j + 1; c < 16; ++c) a[i][c] = fmaf(-w, col[c], a[i][c]);
      }
    }
    // ---- store L of the panel ----------------------------------------------------------------------------------------
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      if (i < sp) continue;
      const int bi = i * Q + lq;
      if (i == sp) {
#pragma unroll
        for (int c = 0; c < 16; ++c) {
          if (bi == p) {
            if (c <= lr) slot[LL::diag(p, lr, c)] = a[i][c];
          } else if (bi > p) {
            slot[LL::offd(bi, p, lr, c)] = a[i][c];
          }
        }
      } else {
        float* rowp = slot + LL::offd_base(bi, p) + lr * 16;
#pragma unroll
        for (int cg = 0; cg < 4; ++cg)
          *reinterpret_cast<float4*>(rowp + 4 * (cg ^ sw)) =
              make_float4(a[i][4 * cg + 0], a[i][4 * cg + 1], a[i][4 * cg + 2], a[i][4 * cg + 3]);
      }
    }
    __syncwarp();
  }

  // ---- back substitution L^T x = y: column-oriented, x_g broadcast inside the lane group -----------------------------
  float xs[4] = {0.f, 0.f, 0.f, 0.f};
#pragma unroll
  for (int g = N - 1; g >= 0; --g) {
    const int sg = g / LANES, lg = g % LANES, gb = g >> 4, gr = g & 15;
    const float t = yv[sg] * dv[sg];
    const float xg = __shfl_sync(0xffffffffu, t, lg, LANES);
    if (l == lg) xs[sg] = xg;
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      if (i * Q > gb) continue;                         // every row of this slot lies below row g
      const int bi = i * Q + lq;
      if (bi < gb) yv[i] = fmaf(-slot[LL::offd(gb, bi, gr, lr)], xg, yv[i]);
      else if (bi == gb && lr < gr) yv[i] = fmaf(-slot[LL::diag(gb, gr, lr)], xg, yv[i]);
    }
  }
  if (valid) {
#pragma unroll
    for (int i = 0; i < 4; ++i) dst_row[i * LANES + l] = xs[i];
    if (bad && l == 0) atomicAdd(fail, 1);
  }
}

}  // namespace pio
