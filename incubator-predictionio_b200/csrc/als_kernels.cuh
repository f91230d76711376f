// als_kernels.cuh -- the ALS half-iteration on sm_90a (H100).
//
// Replaces MLlib's `computeFactors` (SURVEY.md 8(c)-5/6; called through als.run at
// examples/scala-parallel-recommendation/blacklist-items/src/main/scala/ALSAlgorithm.scala:86):
// for every destination row j with rated set Omega_j
//     explicit:  A = sum y y^T + lambda n I,                 b = sum r y
//     implicit:  A = YtY + sum c1 y y^T + lambda n+ I,       b = sum_{r>0} (1+c1) y,  c1 = alpha |r|
// solve A x = b by Cholesky, store x (fp32).
//
// Design (one kernel does gather -> Gramian -> Cholesky -> factor row, nothing round-trips HBM):
//  * rows are processed in degree-descending order (the ingest renumbers rows that way), so the
//    NG rows of one CTA batch have near-equal length;
//  * the upper triangle of the KPxKP Gramian is tiled in TBxTB register blocks, one block per
//    thread, G = NB(NB+1)/2 threads ("group") per row; a CTA runs NG groups = NG rows at once
//    or NG parts of very long rows (work-list mode: the partial normal equations go to global memory);
//  * gathered source rows are staged by cp.async (16 B per thread) into a 3-deep shared-memory
//    ring; a short in-place pass scales them by sqrt(c1) (implicit) and accumulates b;
//  * each warp then factorises one row's matrix with the rows held in registers
//    (lane l owns rows l and N/2+l), pivots broadcast by shuffle, columns through shared memory;
//    forward substitution is fused into the factorisation, back substitution reads L from smem.
// FP32 FFMA throughout the Gramian: this kernel serves the ranks outside 33..64 and the parts of very long rows of
// every rank; for rank 33..64 the tensor-core kernels (als_mma_kernel.cuh, als_tc_kernel.cuh) take the rows up to 8192
// ratings because an 8x8 register block is shared-memory-bound by construction (DESIGN.md 4.1).  The warp Cholesky
// below (chol_solve_warp) is shared by all three kernels.  YtY is accumulated in fp64 by gram_partial_kernel.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include "als_lockstep.cuh"

namespace pio {

struct SolveParams {
  const long long* ptr;  // local CSR row pointers, offsets into idx/val
  const int* idx;        // internal ids of source rows
  const float* val;      // ratings
  const float* src;      // source factor matrix, row stride KP (zero padded)
  float* dst;            // destination factor matrix (full replica), row stride KP
  const float* yty;      // KP x KP (implicit only)
  const float* nreg;     // per local row: n of the ridge term lambda * n
  int* fail;             // incremented once per row whose matrix was not positive definite
  float lambda;
  float alpha;
  int k;                 // true rank (<= KP)
  int row_begin;         // local rows [row_begin, row_end) are covered by this launch
  int row_end;
  int dst_row_offset;    // internal id of local row 0
  // optional work list (parts of very long rows): item i covers ratings [wl_beg[i], wl_end[i]); its Gramian
  // blocks and right-hand side go to partial[i * (SLOT + KP)] instead of being solved in this kernel
  const long long* wl_beg;
  const long long* wl_end;
  float* partial;
  int n_items;
};

template <int KP_, int TB_, int NG_, int CH_>
struct SolveCfg {
  static constexpr int KP = KP_, TB = TB_, NB = KP_ / TB_, G = NB * (NB + 1) / 2;
  static constexpr int NG = NG_, CH = CH_;
  static constexpr int NT = ((NG * G + 31) / 32) * 32;
  static constexpr int NW = NT / 32;
  static constexpr int ROWS = NG * CH;          // gathered rows per stage
  static constexpr int F4ROW = KP / 4;
  static constexpr int STAGE = ROWS * KP;       // floats
  static constexpr int STAGE_F4 = ROWS * F4ROW;
  static constexpr int NF = (STAGE_F4 + NT - 1) / NT;
  static constexpr int NSTAGE = 3;
  static constexpr int BLK = TB * TB + 8;       // padded block stride inside a slot (floats)
  static constexpr int SLOT = G * BLK;
  static constexpr bool WARP_CHOL = KP <= 64;
  // rank 65..128: every row goes through the work-list path -- the kernel emits (partial) normal equations in the
  // LsLayout<128> slot layout and als_finish_ls128_kernel sums the parts and runs the lockstep Cholesky
  static constexpr bool LS_PARTIAL = KP == 128;
  static constexpr int PART_FLOATS = LS_PARTIAL ? LsLayout<LS_PARTIAL ? KP : 64>::SIZE + KP : SLOT + KP;
  static constexpr int LM = 0;

  // the Cholesky slots alias the (dead) staging ring and b partials
  __host__ __device__ static constexpr int region0() {
    return (NSTAGE + 1) * STAGE > NG * SLOT ? (NSTAGE + 1) * STAGE : NG * SLOT;
  }
  __host__ __device__ static constexpr size_t smem_bytes() {
    return sizeof(float) * (size_t)(region0() + NG * KP + NW * 2 * KP + NW * KP +
                                    NSTAGE * ROWS + LM) +
           sizeof(long long) * 2 * NG + sizeof(int) * NG + 16;
  }
};

__device__ __forceinline__ void cp_async16(void* smem_dst, const void* gsrc) {
  const unsigned s = (unsigned)__cvta_generic_to_shared(smem_dst);
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16;\n" ::"r"(s), "l"(gsrc));
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;\n" ::); }
template <int N>
__device__ __forceinline__ void cp_async_wait() {
  asm volatile("cp.async.wait_group %0;\n" ::"n"(N));
}

// position (in float4 units) of original float4 column-group cg inside a staged row.
// TB == 8: the two halves of every 8-wide block are split so that the NB first halves are
// contiguous (bank-conflict-free LDS.128 for lanes that differ in the block index).
template <int TB, int NB>
__device__ __forceinline__ int f4slot(int cg) {
  if (TB == 8) return (cg & 1) * NB + (cg >> 1);
  return cg;
}

// pivots of a positive definite fp32 matrix are far from the denormal range: the flush-to-zero approximation plus one
// Newton step (in the callers) gives 1/sqrt to ~1 ulp without rsqrtf()'s denormal fix-up code
__device__ __forceinline__ float rsqrt_fast(float x) {
  float r;
  asm("rsqrt.approx.ftz.f32 %0, %1;" : "=f"(r) : "f"(x));
  return r;
}

// inverse of f4slot: which source column group lands in staged slot sl
template <int TB, int NB>
__device__ __forceinline__ int f4cg(int sl) {
  if (TB == 8) return ((sl % NB) << 1) | (sl / NB);
  return sl;
}

// ------------------------------------------------------------------------------------------
// Warp Cholesky + solve for N <= 64 (N = KP). Matrix comes from `slot` (upper-triangular TBxTB
// blocks, block (bi,bj) at ((bi*NB - bi*(bi-1)/2) + bj - bi) * BLK, element [a][b] at a*TB+b).
//
// 2x2 blocked, H = N/2, lane l < H owns row l (top) and row H+l (bottom):
//   A: right-looking Cholesky of [A11; A21] (rows in registers, pivots by shuffle, the scaled
//      column through a double-buffered shared line), forward substitution of b fused in;
//   B: A22 -= L21 L21^T as H dot products per lane (own L21 row in registers, the other rows
//      broadcast from shared memory);
//   C: Cholesky of A22 as in A;
//   then back substitution reading L (packed) from shared memory.
// Deferring the A22 update keeps at most 2*H row registers live (no local-memory spills).
// L is written over the slot: L11 packed at 0, L21 dense (row stride H+4) after it, L22 packed
// behind; the layout never overwrites a block that is still to be read (static_asserts below).
// ------------------------------------------------------------------------------------------
// PACKED_IN = true: the matrix arrives already in the L layout (A11 packed lower at 0, A21 dense with
// row stride H+4 at OFF21, A22 packed lower at OFF22) and is factorised in place (tensor-core path).
template <int N, int TB, int BLK, bool IMPLICIT, bool PACKED_IN = false>
__device__ __forceinline__ void chol_solve_warp(float* slot, const float* bvec, const float* yty,
                                                float ridge, int k, float* colbuf, float* dinv,
                                                float* dst_row, int* fail) {
  constexpr int H = N / 2;
  constexpr int NB = N / TB;
  constexpr int L21S = H + 4;
  constexpr int OFF21 = H * (H + 1) / 2;
  constexpr int OFF22 = OFF21 + H * L21S;
  constexpr int A22_FIRST = ((NB / 2) * NB - (NB / 2) * (NB / 2 - 1) / 2) * BLK;
  static_assert(PACKED_IN || OFF22 <= A22_FIRST, "L11/L21 would overwrite unread A22 blocks");
  static_assert(PACKED_IN || OFF22 + H * (H + 1) / 2 <= (NB * (NB + 1) / 2) * BLK, "L does not fit in the slot");
  static_assert(H % 4 == 0, "H must be a multiple of 4");
  const int lane = threadIdx.x & 31;
  const bool act = lane < H;
  const int l = act ? lane : 0;
  const int rA = l, rB = H + l;
  const int ibA = rA / TB, bA_ = rA % TB, ibB = rB / TB, bB_ = rB % TB;
  auto cbase = [](int c) { return ((c / TB) * NB - (c / TB) * ((c / TB) - 1) / 2 - (c / TB)) * BLK + (c % TB) * TB; };

  float ra[H], rm[H];
#pragma unroll
  for (int c = 0; c < H; ++c) {
    float v = 0.f;
    if (c <= rA) {
      v = PACKED_IN ? slot[rA * (rA + 1) / 2 + c] : slot[cbase(c) + ibA * BLK + bA_];
      if (IMPLICIT) v += yty[rA * N + c];
      if (c == rA) v += ridge + (rA >= k ? 1.f : 0.f);
    }
    ra[c] = v;
    float w = PACKED_IN ? slot[OFF21 + l * L21S + c] : slot[cbase(c) + ibB * BLK + bB_];
    if (IMPLICIT) w += yty[rB * N + c];
    rm[c] = w;
  }
  float bAv = bvec[rA], bBv = bvec[rB];
  float yA = 0.f, yB = 0.f;
  bool bad = false;
  __syncwarp();
  // ---- phase A ----
#pragma unroll
  for (int j = 0; j < H; ++j) {
    float* cb_ = colbuf + (j & 1) * N;
    const float d = __shfl_sync(0xffffffffu, ra[j], j);
    const float bj = __shfl_sync(0xffffffffu, bAv, j);
    float dd = d;
    if (!(dd > 0.f)) { bad = true; dd = 1.f; }
    float inv = rsqrt_fast(dd);
    inv = inv * (1.5f - 0.5f * dd * inv * inv);
    const float yj = bj * inv;
    const float la = ra[j] * inv;
    const float lm = rm[j] * inv;
    ra[j] = la;
    rm[j] = lm;
    if (act) cb_[rA] = la;
    if (lane == 0) dinv[j] = inv;
    if (rA == j) yA = yj;
    bAv -= la * yj;
    bBv -= lm * yj;
    __syncwarp();
    // the scaled column is read back as broadcast LDS.128 (one wavefront per four columns)
#pragma unroll
    for (int g = (j + 1) / 4; g < H / 4; ++g) {
      const float4 x = reinterpret_cast<const float4*>(cb_)[g];
      if (4 * g + 0 > j) { ra[4 * g + 0] -= la * x.x; rm[4 * g + 0] -= lm * x.x; }
      if (4 * g + 1 > j) { ra[4 * g + 1] -= la * x.y; rm[4 * g + 1] -= lm * x.y; }
      if (4 * g + 2 > j) { ra[4 * g + 2] -= la * x.z; rm[4 * g + 2] -= lm * x.z; }
      if (4 * g + 3 > j) { ra[4 * g + 3] -= la * x.w; rm[4 * g + 3] -= lm * x.w; }
    }
  }
  __syncwarp();
  float* L21 = slot + OFF21;
  if (act) {
#pragma unroll
    for (int c = 0; c < H; ++c)
      if (c <= rA) slot[rA * (rA + 1) / 2 + c] = ra[c];
#pragma unroll
    for (int c = 0; c < H; c += 4)
      *reinterpret_cast<float4*>(L21 + l * L21S + c) = make_float4(rm[c], rm[c + 1], rm[c + 2], rm[c + 3]);
  }
  // ---- phase B ----
  float r2[H];
#pragma unroll
  for (int c = 0; c < H; ++c) {
    float v = 0.f;
    if (c <= l) {
      v = PACKED_IN ? slot[OFF22 + l * (l + 1) / 2 + c] : slot[cbase(H + c) + ibB * BLK + bB_];
      if (IMPLICIT) v += yty[rB * N + H + c];
      if (c == l) v += ridge + (rB >= k ? 1.f : 0.f);
    }
    r2[c] = v;
  }
  __syncwarp();
#pragma unroll
  for (int c = 0; c < H; ++c) {
    float s0 = 0.f, s1 = 0.f, s2 = 0.f, s3 = 0.f;
    const float4* row = reinterpret_cast<const float4*>(L21 + c * L21S);
#pragma unroll
    for (int t = 0; t < H; t += 4) {
      const float4 x = row[t / 4];
      s0 = fmaf(rm[t], x.x, s0);
      s1 = fmaf(rm[t + 1], x.y, s1);
      s2 = fmaf(rm[t + 2], x.z, s2);
      s3 = fmaf(rm[t + 3], x.w, s3);
    }
    r2[c] -= (s0 + s1) + (s2 + s3);
  }
  // ---- phase C ----
#pragma unroll
  for (int j = 0; j < H; ++j) {
    float* cb_ = colbuf + (j & 1) * N;
    const float d = __shfl_sync(0xffffffffu, r2[j], j);
    const float bj = __shfl_sync(0xffffffffu, bBv, j);
    float dd = d;
    if (!(dd > 0.f)) { bad = true; dd = 1.f; }
    float inv = rsqrt_fast(dd);
    inv = inv * (1.5f - 0.5f * dd * inv * inv);
    const float yj = bj * inv;
    const float l2 = r2[j] * inv;
    r2[j] = l2;
    if (act) cb_[l] = l2;
    if (lane == 0) dinv[H + j] = inv;
    if (l == j) yB = yj;
    bBv -= l2 * yj;
    __syncwarp();
#pragma unroll
    for (int g = (j + 1) / 4; g < H / 4; ++g) {
      const float4 x = reinterpret_cast<const float4*>(cb_)[g];
      if (4 * g + 0 > j) r2[4 * g + 0] -= l2 * x.x;
      if (4 * g + 1 > j) r2[4 * g + 1] -= l2 * x.y;
      if (4 * g + 2 > j) r2[4 * g + 2] -= l2 * x.z;
      if (4 * g + 3 > j) r2[4 * g + 3] -= l2 * x.w;
    }
  }
  __syncwarp();
  float* L22 = slot + OFF22;
  if (act) {
#pragma unroll
    for (int c = 0; c < H; ++c)
      if (c <= l) L22[l * (l + 1) / 2 + c] = r2[c];
  }
  __syncwarp();
  // ---- back substitution: L^T x = y ----
  float xA = 0.f, xB = 0.f;
#pragma unroll
  for (int i = H - 1; i >= 0; --i) {  // bottom rows H+i
    const float xi = __shfl_sync(0xffffffffu, yB, i) * dinv[H + i];
    if (l == i) xB = xi;
    if (act) {
      if (l < i) yB -= L22[i * (i + 1) / 2 + l] * xi;
      yA -= L21[i * L21S + l] * xi;
    }
  }
#pragma unroll
  for (int i = H - 1; i >= 0; --i) {  // top rows i
    const float xi = __shfl_sync(0xffffffffu, yA, i) * dinv[i];
    if (l == i) xA = xi;
    if (act && l < i) yA -= slot[i * (i + 1) / 2 + l] * xi;
  }
  if (act) {
    dst_row[rA] = xA;
    dst_row[rB] = xB;
  }
  if (bad && lane == 0) atomicAdd(fail, 1);
}

// ------------------------------------------------------------------------------------------
// The half-step kernel.
// ------------------------------------------------------------------------------------------
template <class Cfg, bool IMPLICIT>
__global__ void __launch_bounds__(Cfg::NT, Cfg::WARP_CHOL ? 2 : 1)
als_solve_kernel(const SolveParams p) {
  constexpr int KP = Cfg::KP, TB = Cfg::TB, NB = Cfg::NB, G = Cfg::G, NG = Cfg::NG, CH = Cfg::CH;
  constexpr int NT = Cfg::NT, NW = Cfg::NW, ROWS = Cfg::ROWS, F4ROW = Cfg::F4ROW;
  constexpr int STAGE = Cfg::STAGE, STAGE_F4 = Cfg::STAGE_F4, NF = Cfg::NF, NSTAGE = Cfg::NSTAGE;
  constexpr int BLK = Cfg::BLK, SLOT = Cfg::SLOT;

  extern __shared__ __align__(16) float smem[];
  float* stage = smem;
  float* bpart = stage + NSTAGE * STAGE;
  float* slots = smem;   // aliases the ring: written only after the last chunk has been consumed
  float* bvec = smem + Cfg::region0();
  float* colbuf = bvec + NG * KP;
  float* dinvb = colbuf + NW * 2 * KP;
  float* mval = dinvb + NW * KP;
  float* lm = mval + NSTAGE * ROWS;
  long long* segb = reinterpret_cast<long long*>(
      (reinterpret_cast<uintptr_t>(lm + Cfg::LM) + 15) & ~uintptr_t(15));
  long long* sege = segb + NG;
  int* srow = reinterpret_cast<int*>(sege + NG);

  const int tid = threadIdx.x;
  const int g = tid / G;                 // group of this thread (>= NG: staging helper only)
  const int bid = tid - g * G;           // block id inside the triangle
  const bool worker = g < NG;
  int bi = 0, bj = 0;
  {
    int t = bid;
    while (t >= NB - bi) { t -= NB - bi; ++bi; }
    bj = bi + t;
  }

  if (tid < NG) {
    if (p.partial) {
      const int item = blockIdx.x * NG + tid;
      if (item < p.n_items) {
        segb[tid] = p.wl_beg[item];
        sege[tid] = p.wl_end[item];
        srow[tid] = item;
      } else {
        segb[tid] = 0;
        sege[tid] = 0;
        srow[tid] = -1;
      }
    } else {
      const int r = p.row_begin + blockIdx.x * NG + tid;
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
  }
  // zero the b partials
  for (int o = tid; o < STAGE; o += NT) bpart[o] = 0.f;
  __syncthreads();

  long long maxlen = 0;
#pragma unroll 1
  for (int q = 0; q < NG; ++q) {
    const long long len = sege[q] - segb[q];
    maxlen = len > maxlen ? len : maxlen;
  }
  const int nchunks = (int)((maxlen + CH - 1) / CH);
  const long long mylen = worker ? sege[g] - segb[g] : 0;

  // ---- staging helpers -----------------------------------------------------------------
  int nidx[NF];
  float nval[NF];
  auto prefetch_meta = [&](int c) {
#pragma unroll
    for (int j = 0; j < NF; ++j) {
      const int f = tid + j * NT;
      nidx[j] = -1;
      nval[j] = 0.f;
      if (f < STAGE_F4 && c < nchunks) {
        const int q = f / F4ROW;
        const int gg = q / CH, i = q % CH;
        const long long e = segb[gg] + (long long)c * CH + i;
        if (e < sege[gg]) {
          nidx[j] = __ldg(p.idx + e);
          nval[j] = __ldg(p.val + e);
        }
      }
    }
  };
  auto issue = [&](int c) {  // uses nidx/nval prefetched for chunk c
    float* sbuf = stage + (c % NSTAGE) * STAGE;
    float* mv = mval + (c % NSTAGE) * ROWS;
#pragma unroll
    for (int j = 0; j < NF; ++j) {
      const int f = tid + j * NT;
      if (f < STAGE_F4 && c < nchunks) {
        // consecutive threads fill consecutive 16 B slots of the staged row (conflict-free);
        // the slot -> source column-group map is the inverse of f4slot
        const int q = f / F4ROW, sl = f % F4ROW;
        const int cg = f4cg<TB, NB>(sl);
        float4* d4 = reinterpret_cast<float4*>(sbuf) + f;
        if (nidx[j] >= 0) {
          cp_async16(d4, p.src + (size_t)nidx[j] * KP + cg * 4);
        } else {
          *d4 = make_float4(0.f, 0.f, 0.f, 0.f);
        }
        if (sl == 0) mv[q] = nval[j];
      }
    }
    cp_async_commit();
  };

  float acc[TB][TB];
#pragma unroll
  for (int a = 0; a < TB; ++a)
#pragma unroll
    for (int b = 0; b < TB; ++b) acc[a][b] = 0.f;

  float* myslot = slots + (worker ? g : 0) * SLOT + bid * BLK;

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
    float* sbuf = stage + (c % NSTAGE) * STAGE;
    const float* mv = mval + (c % NSTAGE) * ROWS;
    // b accumulation (+ sqrt(c1) scaling in place for implicit feedback)
#pragma unroll
    for (int j = 0; j < NF; ++j) {
      const int f = tid + j * NT;
      if (f < STAGE_F4) {
        const int q = f / F4ROW;
        const int o4 = f;
        const float r = mv[q];
        float4 y = reinterpret_cast<float4*>(sbuf)[o4];
        float wb, sc;
        if (IMPLICIT) {
          const float c1 = p.alpha * fabsf(r);
          wb = r > 0.f ? 1.f + c1 : 0.f;
          sc = sqrtf(c1);
        } else {
          wb = r;
          sc = 1.f;
        }
        float4 bp = reinterpret_cast<float4*>(bpart)[o4];
        bp.x = fmaf(wb, y.x, bp.x);
        bp.y = fmaf(wb, y.y, bp.y);
        bp.z = fmaf(wb, y.z, bp.z);
        bp.w = fmaf(wb, y.w, bp.w);
        reinterpret_cast<float4*>(bpart)[o4] = bp;
        if (IMPLICIT) {
          y.x *= sc; y.y *= sc; y.z *= sc; y.w *= sc;
          reinterpret_cast<float4*>(sbuf)[o4] = y;
        }
      }
    }
    if (IMPLICIT) __syncthreads();
    if (worker) {
      // every staged row of the chunk is consumed unconditionally: rows past the end of a segment were zero-filled by
      // issue(), and without a per-rating branch the operand loads of rating i+1 overlap the FMAs of rating i
      const float4* rowp = reinterpret_cast<const float4*>(sbuf + (g * CH) * KP);
      if (mylen - (long long)c * CH > 0) {
#pragma unroll
        for (int i = 0; i < CH; ++i) {
          const float4* rp = rowp + i * F4ROW;
          float P[TB], Q[TB];
          if (TB == 8) {
            const float4 p0 = rp[bi], p1 = rp[NB + bi], q0 = rp[bj], q1 = rp[NB + bj];
            P[0] = p0.x; P[1] = p0.y; P[2] = p0.z; P[3] = p0.w;
            P[4 % TB] = p1.x; P[5 % TB] = p1.y; P[6 % TB] = p1.z; P[7 % TB] = p1.w;
            Q[0] = q0.x; Q[1] = q0.y; Q[2] = q0.z; Q[3] = q0.w;
            Q[4 % TB] = q1.x; Q[5 % TB] = q1.y; Q[6 % TB] = q1.z; Q[7 % TB] = q1.w;
          } else {
            const float4 p0 = rp[bi], q0 = rp[bj];
            P[0] = p0.x; P[1] = p0.y; P[2] = p0.z; P[3] = p0.w;
            Q[0] = q0.x; Q[1] = q0.y; Q[2] = q0.z; Q[3] = q0.w;
          }
#pragma unroll
          for (int a = 0; a < TB; ++a)
#pragma unroll
            for (int b = 0; b < TB; ++b) acc[a][b] = fmaf(P[a], Q[b], acc[a][b]);
        }
      }
    }
  }
  cp_async_wait<0>();
  __syncthreads();

  // ---- b: fixed-order reduction of the per-staged-row partials ----------------------------
  for (int o = tid; o < NG * KP; o += NT) {
    const int gg = o / KP, col = o % KP;
    const int pos = f4slot<TB, NB>(col >> 2) * 4 + (col & 3);
    float s = 0.f;
#pragma unroll
    for (int i = 0; i < CH; ++i) s += bpart[(gg * CH + i) * KP + pos];
    bvec[o] = s;
  }
  __syncthreads();  // ring + bpart are dead from here on (the slots alias them)
  if (p.partial) {
    // part of a long row: emit the partial normal equations; als_finish_kernel sums the parts and solves
    if (Cfg::LS_PARTIAL) {
      // lower triangle in the LsLayout<KP> slot layout: this thread's block holds G[8 bi + a][8 bj + b] (bi <= bj), i.e. the
      // lower-triangle elements (r = 8 bj + b, c = 8 bi + a); the 8 columns of one r are two aligned chunks of four
      using LL = LsLayout<Cfg::LS_PARTIAL ? KP : 64>;
      if (worker && srow[g] >= 0) {
        float* out = p.partial + (size_t)srow[g] * Cfg::PART_FLOATS;
#pragma unroll
        for (int b = 0; b < TB; ++b) {
          const int r = TB * bj + b, rb = r >> 4, rr = r & 15;
#pragma unroll
          for (int hh = 0; hh < TB / 4; ++hh) {
            const int c0 = TB * bi + 4 * hh, cb = c0 >> 4, cc = c0 & 15;
            if (cb < rb) {
              *reinterpret_cast<float4*>(out + LL::offd(rb, cb, rr, cc)) =
                  make_float4(acc[4 * hh + 0][b], acc[4 * hh + 1][b], acc[4 * hh + 2][b], acc[4 * hh + 3][b]);
            } else {
#pragma unroll
              for (int e = 0; e < 4; ++e)
                if (cc + e <= rr) out[LL::diag(rb, rr, cc + e)] = acc[4 * hh + e][b];
            }
          }
        }
      }
      for (int o = tid; o < NG * KP; o += NT) {
        const int gg = o / KP;
        if (srow[gg] >= 0) p.partial[(size_t)srow[gg] * Cfg::PART_FLOATS + LL::SIZE + (o % KP)] = bvec[o];
      }
      return;
    }
    if (worker && srow[g] >= 0) {
      float* out = p.partial + (size_t)srow[g] * (SLOT + KP) + bid * BLK;
#pragma unroll
      for (int a = 0; a < TB; ++a)
#pragma unroll
        for (int b = 0; b < TB; b += 4)
          *reinterpret_cast<float4*>(out + a * TB + b) = make_float4(acc[a][b], acc[a][b + 1], acc[a][b + 2], acc[a][b + 3]);
    }
    for (int o = tid; o < NG * KP; o += NT) {
      const int gg = o / KP;
      if (srow[gg] >= 0) p.partial[(size_t)srow[gg] * (SLOT + KP) + SLOT + (o % KP)] = bvec[o];
    }
    return;
  }
  if (worker) {
#pragma unroll
    for (int a = 0; a < TB; ++a)
#pragma unroll
      for (int b = 0; b < TB; ++b) myslot[a * TB + b] = acc[a][b];
  }
  __syncthreads();

  // ---- Cholesky + triangular solves ---------------------------------------------------------
  constexpr int NMAT = NG;
  if (Cfg::WARP_CHOL) {
    const int w = tid >> 5;
    for (int m = w; m < NMAT; m += NW) {
      const int r = srow[m];
      if (r < 0) continue;
      if (p.ptr[r + 1] == p.ptr[r]) continue;  // no ratings: MLlib emits no factor
      const float ridge = p.lambda * p.nreg[r];
      chol_solve_warp<Cfg::WARP_CHOL ? KP : 16, TB, BLK, IMPLICIT>(
          slots + m * SLOT, bvec + m * KP, p.yty, ridge, p.k, colbuf + w * 2 * KP, dinvb + w * KP,
          p.dst + (size_t)(p.dst_row_offset + r) * KP, p.fail);
    }
  }
  // rank 65..128 never reaches this point: all of its rows are work-list items (LS_PARTIAL)
}

// ------------------------------------------------------------------------------------------
// Finish kernel for rows that were split into parts: fixed-order sum of the partial normal equations,
// then the same Cholesky + solves. One warp per row (rank <= 64) or one CTA per row (rank > 64).
// ------------------------------------------------------------------------------------------
template <class Cfg, bool IMPLICIT>
__global__ void __launch_bounds__(Cfg::WARP_CHOL ? 128 : Cfg::NT)
als_finish_kernel(const SolveParams p, const int* __restrict__ row_part_ptr, int n_rows) {
  constexpr int KP = Cfg::KP, SLOT = Cfg::SLOT;
  extern __shared__ __align__(16) float fsm[];
  if (Cfg::WARP_CHOL) {
    const int w = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int r = blockIdx.x * 4 + w;
    if (r >= n_rows) return;
    float* slot = fsm + w * (SLOT + 4 * KP);
    float* bv = slot + SLOT;
    float* colbuf = bv + KP;
    float* dinv = colbuf + 2 * KP;
    const int p0 = row_part_ptr[r], p1 = row_part_ptr[r + 1];
    for (int o = lane; o < SLOT + KP; o += 32) {
      float s = 0.f;
      for (int q = p0; q < p1; ++q) s += p.partial[(size_t)q * (SLOT + KP) + o];
      slot[o] = s;   // o >= SLOT lands in bv (contiguous)
    }
    __syncwarp();
    chol_solve_warp<Cfg::WARP_CHOL ? KP : 16, Cfg::TB, Cfg::BLK, IMPLICIT>(
        slot, bv, p.yty, p.lambda * p.nreg[r], p.k, colbuf, dinv, p.dst + (size_t)(p.dst_row_offset + r) * KP, p.fail);
  }
}

// Rank 65..128: one warp per row; fixed-order sum of the row's partial normal equations (LsLayout<128> + b) into shared
// memory, then the lockstep Cholesky with all 32 lanes on the one 128 x 128 matrix.  FIN128_WARPS warps per CTA (one CTA per
// SM: 33 KB of shared memory per matrix) share one barrier before the solve, so that they walk the large unrolled solver
// together (instruction-cache locality, as in the pair kernel).
constexpr int FIN128_WARPS = 6;
constexpr int FIN128_FLOATS = LsLayout<128>::STRIDE + 128 + 80;   // slot, b, pivot line -- per warp

template <bool IMPLICIT>
__global__ void __launch_bounds__(32 * FIN128_WARPS, 1)
als_finish_ls128_kernel(const SolveParams p, const int* __restrict__ row_part_ptr, int row0, int n_rows, int part0) {
  using LL = LsLayout<128>;
  constexpr int PF = LL::SIZE + 128;
  extern __shared__ __align__(16) float fsm128[];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  float* slot = fsm128 + warp * FIN128_FLOATS;
  float* bv = slot + LL::STRIDE;
  float* colbuf = bv + 128;
#pragma unroll 1
  for (int base = blockIdx.x * FIN128_WARPS; base < n_rows; base += gridDim.x * FIN128_WARPS) {
    const int rr = base + warp;
    const bool have = rr < n_rows;
    const int r = row0 + (have ? rr : 0);
    if (have) {
      const int p0 = row_part_ptr[r] - part0, p1 = row_part_ptr[r + 1] - part0;
      for (int o = lane; o < PF / 4; o += 32) {
        float4 s = make_float4(0.f, 0.f, 0.f, 0.f);
        for (int q = p0; q < p1; ++q) {
          const float4 v = __ldg(reinterpret_cast<const float4*>(p.partial + (size_t)q * PF) + o);
          s.x += v.x; s.y += v.y; s.z += v.z; s.w += v.w;
        }
        if (o < LL::SIZE / 4) reinterpret_cast<float4*>(slot)[o] = s;
        else reinterpret_cast<float4*>(bv)[o - LL::SIZE / 4] = s;
      }
    }
    __syncthreads();
    if (have)
      chol_lockstep<128, IMPLICIT>(slot, bv, p.yty, p.lambda * p.nreg[r], p.k, colbuf,
                                   p.dst + (size_t)(p.dst_row_offset + r) * 128, true, p.fail);
    __syncthreads();
  }
}

// ------------------------------------------------------------------------------------------
// YtY (implicit feedback): fp64 accumulation of X^T X over all rows of a zero-padded factor
// matrix; per-CTA partials reduced in fixed order (deterministic).
// ------------------------------------------------------------------------------------------
constexpr int GRAM_THREADS = 256;
constexpr int GRAM_ROWS = 32;
// YtY = sum over GRAM_GROUPS = 8 CLASSES of rows, each class summed block by block in a fixed order, then the class sums
// in class order.  Class g = the rows whose degree-rank position p has p mod 16 in {g, 15 - g}: exactly the rows the
// serpentine dealing of assign_internal_kernel gives to rank g of an 8-GPU job, and for 4 / 2 / 1 GPUs every rank owns
// whole classes.  So on any of these world sizes a rank can sum its classes from its OWN rows right after solving them
// (while the factor all-gather is still in flight), the ranks all-gather 8 x KP^2 doubles, and the result is
// bit-identical to the single-GPU sum.
constexpr int GRAM_GROUPS = 8;
struct GramMap {
  int cls[GRAM_GROUPS];      // class of the lg-th group this launch computes
  int slot_of[GRAM_GROUPS];  // storage slot of class g (a rank's slots are contiguous: the all-gather concatenates by rank)
};

template <int KP>
__global__ void __launch_bounds__(GRAM_THREADS)
gram_partial_kernel(const float* __restrict__ X, const int* __restrict__ p2i, int n_rows, double* __restrict__ partial,
                    int slot0, int bpg, const GramMap map) {
  // grid: (groups of this launch) x bpg blocks; block b of a class covers a fixed range of the class's positions
  constexpr int TM = KP / 16;
  __shared__ __align__(16) float tile[GRAM_ROWS * KP];
  const int tid = threadIdx.x, ty = tid / 16, tx = tid % 16;
  double acc[TM][TM];
#pragma unroll
  for (int i = 0; i < TM; ++i)
#pragma unroll
    for (int j = 0; j < TM; ++j) acc[i][j] = 0.0;
  const int lg = blockIdx.x / bpg, b = blockIdx.x % bpg, g = map.cls[lg];
  const int rem = n_rows % 16;
  const int T = 2 * (n_rows / 16) + (g < rem ? 1 : 0) + (15 - g < rem ? 1 : 0);   // positions in class g
  const int per = (T + bpg - 1) / bpg;
  const int t0 = min(T, b * per);
  const int t1 = min(T, t0 + per);
  for (int base = t0; base < t1; base += GRAM_ROWS) {
    const int nr = min(GRAM_ROWS, t1 - base);
    for (int o = tid; o < GRAM_ROWS * KP / 4; o += GRAM_THREADS) {
      const int rr = o / (KP / 4);
      float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
      if (rr < nr) {
        const int t = base + rr;
        const int pos = 16 * (t >> 1) + ((t & 1) ? 15 - g : g);     // increasing in t
        v = reinterpret_cast<const float4*>(X + (size_t)__ldg(p2i + pos) * KP)[o % (KP / 4)];
      }
      reinterpret_cast<float4*>(tile)[o] = v;
    }
    __syncthreads();
#pragma unroll 4
    for (int rr = 0; rr < GRAM_ROWS; ++rr) {
      double a[TM], bb[TM];
#pragma unroll
      for (int i = 0; i < TM; ++i) {
        a[i] = (double)tile[rr * KP + ty * TM + i];
        bb[i] = (double)tile[rr * KP + tx * TM + i];
      }
#pragma unroll
      for (int i = 0; i < TM; ++i)
#pragma unroll
        for (int j = 0; j < TM; ++j) acc[i][j] = fma(a[i], bb[j], acc[i][j]);
    }
    __syncthreads();
  }
  double* out = partial + ((size_t)(slot0 + lg) * bpg + b) * KP * KP;
#pragma unroll
  for (int i = 0; i < TM; ++i)
#pragma unroll
    for (int j = 0; j < TM; ++j) out[(ty * TM + i) * KP + tx * TM + j] = acc[i][j];
}

// slot sums: the bpg block partials of a slot in block order
__global__ void gram_group_kernel(const double* __restrict__ partial, int blocks_per_group, int n, int g0,
                                  double* __restrict__ gsum) {
  const int o = blockIdx.x * blockDim.x + threadIdx.x;
  const int g = g0 + blockIdx.y;
  if (o >= n) return;
  const double* p = partial + (size_t)g * blocks_per_group * n;
  double s = 0.0;
  for (int q = 0; q < blocks_per_group; ++q) s += p[(size_t)q * n + o];
  gsum[(size_t)g * n + o] = s;
}

// the class sums in class order
__global__ void gram_reduce_kernel(const double* __restrict__ gsum, int n, float* __restrict__ out, const GramMap map) {
  const int o = blockIdx.x * blockDim.x + threadIdx.x;
  if (o >= n) return;
  double s = 0.0;
#pragma unroll
  for (int g = 0; g < GRAM_GROUPS; ++g) s += gsum[(size_t)map.slot_of[g] * n + o];
  out[o] = (float)s;
}

}  // namespace pio
