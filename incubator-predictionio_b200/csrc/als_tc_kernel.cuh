// als_tc_kernel.cuh -- rank 33..64 ALS half-step with the Gramian on the Hopper tensor cores (wgmma).
//
// Same mathematics as als_solve_kernel (als_kernels.cuh) for KP = 64, but  A = sum (s y)(s y)^T  is a
// split-precision SYRK on wgmma:
//   every gathered, sqrt(c1)-scaled source row x is split into hi (top 10 mantissa bits) and lo = x - hi (exact);
//   8 ratings form one K-block of two 64 x 8 tiles (hi, lo) in the K-major, un-swizzled wgmma layout (tf32 wgmma
//   reads both operands K-major only: features are M / N, ratings are K).  Per K-block three m64n64k8 wgmmas add
//   lo hi^T + hi lo^T + hi hi^T to the team's register accumulator (lo lo^T, ~2^-20 relative, is dropped).  The
//   tensor core's fp32 accumulation truncates, so a chain covers one 24-rating stage; stage sums are added into A in
//   shared memory with round-to-nearest fp32 adds.
//
// Warp roles (512 threads, 1 CTA per SM, persistent; degree-sorted rows are dealt statically: groups of
// NTEAM*NSLOT consecutive rows go to the CTAs in snake order):
//   warp 0              scheduler, warp-parallel: lane t*4+s keeps row lane (team t, slot s) in registers, builds
//                       the flat stage list of a batch with shuffles and publishes it
//   warps 1..NGATHER    gather warps: gw owns every NGATHER-th stage; source indices two stages ahead in
//                       registers, 12 LDGSTS per 24-rating stage into the raw ring (rows padded to 288 bytes),
//                       completion by cp.async.mbarrier.arrive.noinc
//   next NCONV warps    converters: cw owns the stages whose number inside their segment is cw mod NCONV: LDS.128
//                       of the raw rows, scale, hi/lo split, 96 conflict-free STS.32 into the wgmma stage ring,
//                       fence.proxy.async, arrive on full[stage]; right-hand side b reduced at segment ends
//   last 4*NTEAM warps  teams of four warps = one warpgroup each: issue the wgmmas of their batch stage by stage
//                       (the stage is released when they complete), add the accumulator of every finished
//                       segment into its A slot in shared memory, then each warp Cholesky-solves one of the four
//                       rows (chol_solve_warp<PACKED_IN>), or - split mode - stores the normal equations for
//                       als_solve_packed_kernel.  While one team solves, the other one consumes the stages.
// A batch = up to four (row, rating-segment) pairs, accumulated one after the other; rows longer than SEG ratings
// take several batches.  Every sum has a fixed order that depends on the row alone, so results do not depend on the
// grid or on how rows are sharded over GPUs.
// Every blocking mbarrier wait has a watchdog (mbar_wait): a protocol error traps with a diagnostic.
// This header is included once per role partition (pio_als.cu): TC_NS names the namespace, TC_NTEAM / TC_NCONV /
// TC_NGATHER / TC_NSTAGE / TC_NRAW fix how the sixteen warps and the shared memory of the CTA are divided.
#ifndef TC_NS
#error "define TC_NS, TC_NTEAM, TC_NCONV, TC_NGATHER, TC_NSTAGE, TC_NRAW before including als_tc_kernel.cuh"
#endif
#include <cuda_runtime.h>
#include <stddef.h>
#include <stdint.h>

#include "als_kernels.cuh"

#ifndef PIO_TC_TIMING
#define PIO_TC_TIMING 0
#endif

namespace pio {
namespace TC_NS {

constexpr int KP = 64;
constexpr int KB_RATINGS = 8;                    // K of one tf32 wgmma
constexpr int CORE_K_BYTES = 144;                // leading byte offset: the second 4-rating core matrix of a feature group
constexpr int CORE_M_BYTES = 288;                // stride byte offset: the next group of 8 features
constexpr int TILE_BYTES = (KP / 8) * CORE_M_BYTES;   // one 64 x 8 operand tile (hi or lo): 2304
constexpr int KB_BYTES = 2 * TILE_BYTES;         // hi tile, lo tile: 4608
constexpr int STAGE_KB = 3;                      // one K-block per producer warp
constexpr int STAGE_RATINGS = STAGE_KB * KB_RATINGS;  // 24
constexpr int STAGE_BYTES = STAGE_KB * KB_BYTES;      // 13824
constexpr int NSTAGE = TC_NSTAGE;                 // wgmma stage ring
constexpr int NRAW = TC_NRAW;                          // raw ring: stages of gathered rows in flight
constexpr int RAW_ROW = 288;                     // bytes per gathered row in the raw ring (256 + 32 pad: conflict-free LDS.128)
constexpr int NGATHER = TC_NGATHER;                       // gather warps (each owns every NGATHER-th stage)
constexpr int NCONV = TC_NCONV;                         // converter warps (each owns every NCONV-th stage)
constexpr int CONV0 = 1 + NGATHER;               // first converter warp
constexpr int TEAM0 = CONV0 + NCONV;             // first team warp (a multiple of 4: every team is one warpgroup)
static_assert(TEAM0 % 4 == 0, "team warps must start at a multiple of four");
constexpr int SEG = 21 * STAGE_RATINGS;          // 504 ratings per accumulation segment
constexpr int NTEAM = TC_NTEAM;                   // drain + solve teams of four warps
constexpr int NSLOT = 4;
constexpr int NTHREADS = 512;
static_assert((TEAM0 + 4 * NTEAM) * 32 == NTHREADS, "the role partition must fill the sixteen warps of the CTA");
constexpr int H = 32;
constexpr int L21S = H + 4;
constexpr int OFF21 = H * (H + 1) / 2;           // 528
constexpr int OFF22 = OFF21 + H * L21S;          // 1680
constexpr int ASLOT = OFF22 + H * (H + 1) / 2;   // 2208 floats

// one wgmma stage (<= 24 ratings of one segment), pre-expanded by the scheduler so producers need no bookkeeping
struct StageEnt {
  long long beg;   // offset of the stage's first rating in idx/val
  int valid;       // ratings in this stage (1..24)
  int info;        // bits 0-1 slot, bit 2 last stage of its segment, bit 3 last stage of the batch, bit 4 first stage of its segment
};
constexpr int MAX_STAGES = NSLOT * (SEG / STAGE_RATINGS);   // 84

struct BatchDesc {
  int row[NSLOT];    // local row, -1 = empty slot
  int first[NSLOT];  // segment starts its row (overwrite the A slot instead of accumulating)
  int last[NSLOT];   // segment ends its row (solve after draining)
  int exit;
  unsigned stage0;   // global number of the batch's first stage (ring slot stage0 % NSTAGE)
  int nstages;
  int pad;
  StageEnt st[MAX_STAGES];
};

struct Smem {
  alignas(128) unsigned char stage[NSTAGE][STAGE_BYTES];
  alignas(16) float aslot[NTEAM][NSLOT][ASLOT];
  alignas(16) float bslot[NTEAM][NSLOT][KP];
  alignas(16) float bstage[NTEAM][2][NSLOT][KP];
  alignas(16) float bpart[NCONV][KP];
  alignas(16) unsigned char raw[NRAW][STAGE_RATINGS * RAW_ROW];   // gathered source rows (cp.async.bulk destinations)
  float rawval[NRAW][32];                                          // their ratings
  alignas(16) float colbuf[NTEAM * NSLOT][2 * KP];
  alignas(16) float dinv[NTEAM * NSLOT][KP];
  BatchDesc desc[NTEAM][2];   // double-buffered per team: batch n+1 is produced while the team still solves batch n
  alignas(8) unsigned long long full[NSTAGE];
  unsigned long long descfull[NTEAM][2];
  unsigned long long teamdone[NTEAM][2];
  unsigned long long bfull[NTEAM][2];
  unsigned long long rawfull[NRAW];    // gather warp -> converters (transaction-count barrier)
  unsigned long long rawempty[NRAW];   // converters -> gather warp
  unsigned consumed;   // stages whose wgmmas have completed; the teams consume the ring strictly in stage order
};

// ---- PTX wrappers -------------------------------------------------------------------------
__device__ __forceinline__ uint32_t s32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void mbar_init(unsigned long long* bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(s32(bar)), "r"(count) : "memory");
}
__device__ __forceinline__ void mbar_arrive(unsigned long long* bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(s32(bar)) : "memory");
}
__device__ __forceinline__ bool mbar_try(unsigned long long* bar, uint32_t parity) {
  uint32_t ok;
  asm volatile(
      "{\n"
      ".reg .pred P1;\n"
      "mbarrier.try_wait.parity.shared::cta.b64 P1, [%1], %2, %3;\n"
      "selp.u32 %0, 1, 0, P1;\n"
      "}"
      : "=r"(ok)
      : "r"(s32(bar)), "r"(parity), "r"(200000u)   // suspend-time hint (ns): the waiting warp sleeps instead of polling
      : "memory");
  return ok != 0;
}
// Blocking wait with a watchdog: a protocol error must end the kernel with a diagnostic, never hang the GPU.
__device__ __noinline__ void mbar_timeout(unsigned long long* bar, uint32_t parity) {
  extern __shared__ __align__(1024) unsigned char tc_smem_base_[];
  if ((threadIdx.x & 31) == 0) printf("pio tc kernel: mbarrier wait timed out: cta %d warp %d lane %d barrier word %d (full%d descfull%d teamdone%d bfull%d rawfull%d rawempty%d) parity %u\n", (int)blockIdx.x,
         (int)(threadIdx.x >> 5), (int)(threadIdx.x & 31), (int)(s32(bar) - s32(tc_smem_base_) - (uint32_t)offsetof(Smem, full)) / 8,
         NSTAGE, 2 * NTEAM, 2 * NTEAM, 2 * NTEAM, NRAW, NRAW, parity);
  __trap();
}
__device__ __forceinline__ void mbar_wait(unsigned long long* bar, uint32_t parity) {
  if (mbar_try(bar, parity)) return;
  const long long t0 = clock64();
  while (!mbar_try(bar, parity)) {
    if (clock64() - t0 > 16000000000ll) mbar_timeout(bar, parity);   // ~8 s (a half-step takes tens of ms; tools like compute-sanitizer slow the kernel ~100x)
  }
}
// the consumed-stage counter: written by one thread of the consuming team (release), polled by converters and teams
// (acquire).  Counting instead of a parity barrier per slot: a waiter may be several laps of the ring ahead of the
// stage it needs, which a phase parity cannot tell apart.
__device__ __forceinline__ uint32_t ld_acquire(const unsigned* p) {
  uint32_t v;
  asm volatile("ld.acquire.cta.shared::cta.u32 %0, [%1];" : "=r"(v) : "r"(s32(p)) : "memory");
  return v;
}
__device__ __forceinline__ void st_release(unsigned* p, uint32_t v) {
  asm volatile("st.release.cta.shared::cta.u32 [%0], %1;" ::"r"(s32(p)), "r"(v) : "memory");
}
// until *cnt >= target (wrap-safe), with the same watchdog as mbar_wait
__device__ __forceinline__ void wait_count(const unsigned* cnt, uint32_t target) {
  if ((int)(ld_acquire(cnt) - target) >= 0) return;
  const long long t0 = clock64();
  while ((int)(ld_acquire(cnt) - target) < 0) {
    __nanosleep(100);
    if (clock64() - t0 > 16000000000ll) {
      if ((threadIdx.x & 31) == 0)
        printf("pio tc kernel: stage count wait timed out: cta %d warp %d count %u target %u\n", (int)blockIdx.x,
               (int)(threadIdx.x >> 5), ld_acquire(cnt), target);
      __trap();
    }
  }
}
__device__ __forceinline__ bool mbar_test(unsigned long long* bar, uint32_t parity) {
  uint32_t ok;
  asm volatile(
      "{\n"
      ".reg .pred P1;\n"
      "mbarrier.test_wait.parity.shared::cta.b64 P1, [%1], %2;\n"   // test_wait never suspends (try_wait may)
      "selp.u32 %0, 1, 0, P1;\n"
      "}"
      : "=r"(ok)
      : "r"(s32(bar)), "r"(parity)
      : "memory");
  return ok != 0;
}
__device__ __forceinline__ void fence_barrier_init() { asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory"); }
__device__ __forceinline__ void fence_proxy_async() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }
// warpgroup-wide wgmma plumbing: fence before the first wgmma that touches registers written by other instructions,
// commit the issued wgmmas as one group, wait until none is pending
__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_wait_all() { asm volatile("wgmma.wait_group.sync.aligned 0;" ::: "memory"); }
// keeps the compiler from moving accesses of an accumulator register across the asynchronous wgmma
__device__ __forceinline__ void acc_fence(float& r) { asm volatile("" : "+f"(r)::"memory"); }
// D[m][n] (+)= sum_k A[m][k] B[n][k] over one K-block of 8 ratings: m64n64k8, tf32 operands from shared memory,
// fp32 accumulator in the registers of the warpgroup (warp w holds rows 16w..16w+15; see drain below)
__device__ __forceinline__ void wgmma_tf32(float (&d)[32], uint64_t adesc, uint64_t bdesc, uint32_t accum) {
  asm volatile(
      "{\n"
      ".reg .pred p;\n"
      "setp.ne.b32 p, %34, 0;\n"
      "wgmma.mma_async.sync.aligned.m64n64k8.f32.tf32.tf32 "
      "{%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,%16,%17,%18,%19,%20,%21,%22,%23,%24,%25,%26,%27,%28,%29,%30,%31}, "
      "%32, %33, p, 1, 1;\n"
      "}"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]),
        "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]),
        "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]),
        "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
      : "l"(adesc), "l"(bdesc), "r"(accum)
      : "memory");
}
// the mbarrier receives one arrival from this thread once all of its earlier cp.async copies have landed
__device__ __forceinline__ void cp_async_mbar_arrive_noinc(unsigned long long* bar) {
  asm volatile("cp.async.mbarrier.arrive.noinc.shared::cta.b64 [%0];" ::"r"(s32(bar)) : "memory");
}
__device__ __forceinline__ void mbar_arrive_expect_tx(unsigned long long* bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(s32(bar)), "r"(bytes) : "memory");
}
// one contiguous global -> shared copy (UBLKCP); completion is signalled on the mbarrier's transaction count
__device__ __forceinline__ void bulk_copy_g2s(void* smem_dst, const void* gsrc, uint32_t bytes, unsigned long long* bar) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(s32(smem_dst)),
               "l"(gsrc), "r"(bytes), "r"(s32(bar))
               : "memory");
}
__device__ __forceinline__ void cp_async4(void* smem_dst, const void* gsrc) {
  asm volatile("cp.async.ca.shared.global [%0], [%1], 4;\n" ::"r"(s32(smem_dst)), "l"(gsrc));
}
// allow at most `pend` of the most recent commit groups to stay in flight (exact up to 8, else conservative)
__device__ __forceinline__ void cp_async_wait_dyn(uint32_t pend) {
  switch (pend) {
    case 0: cp_async_wait<0>(); break;
    case 1: cp_async_wait<1>(); break;
    case 2: cp_async_wait<2>(); break;
    case 3: cp_async_wait<3>(); break;
    case 4: cp_async_wait<4>(); break;
    case 5: cp_async_wait<5>(); break;
    case 6: cp_async_wait<6>(); break;
    case 7: cp_async_wait<7>(); break;
    default: cp_async_wait<8>(); break;
  }
}
__device__ __forceinline__ void named_bar_sync(int id, int nthreads) {
  asm volatile("bar.sync %0, %1;" ::"r"(id), "r"(nthreads) : "memory");
}
// hi part of the split: the top 10 mantissa bits by truncation (one LOP3 on the full-rate integer pipe; cvt.rna.tf32
// goes through the quarter-rate conversion pipe, 48 per lane and stage).  x - hi is exact and has at most 13 significant
// bits, so the split loses nothing; the tensor core's own truncation of lo costs 2^-21 relative, the dropped lo*lo
// term 2^-20.
__device__ __forceinline__ float tf32_round(float x) {
  return __uint_as_float(__float_as_uint(x) & 0xFFFFE000u);
}

// wgmma shared-memory matrix descriptor, K-major without swizzle: start address >> 4 at [0,14); leading byte offset
// (between the two 4-rating core matrices of a K-block) >> 4 at [16,30); stride byte offset (between groups of 8
// features) >> 4 at [32,46); layout type 0 (no swizzle) at [62,64).  Element (feature f, rating k) of a 64 x 8 tile
// sits at  (f/8)*CORE_M_BYTES + (k/4)*CORE_K_BYTES + (f%8)*16 + (k%4)*4.
__device__ __forceinline__ uint64_t make_desc(uint32_t smem_addr) {
  uint64_t d = 0;
  d |= (uint64_t)((smem_addr >> 4) & 0x3FFF);
  d |= (uint64_t)((CORE_K_BYTES >> 4) & 0x3FFF) << 16;
  d |= (uint64_t)((CORE_M_BYTES >> 4) & 0x3FFF) << 32;
  return d;
}
__device__ __forceinline__ int tile_off(int f, int k) {
  return (f >> 3) * CORE_M_BYTES + (k >> 2) * CORE_K_BYTES + (f & 7) * 16 + (k & 3) * 4;
}

static_assert(sizeof(Smem) + 1024 <= 232448, "shared memory budget (227 KB) exceeded");

struct TcParams {
  SolveParams sp;
  long long* timing;  // debug only (PIO_ALS_TC_TIMING=1): [grid][16 warps][8] cycle counters, else null
  float* dbg;    // debug only (PIO_ALS_TC_DEBUG=1): per local row ASLOT + KP floats (A as drained, b), else null
  float* out;    // split mode: per local row ASLOT + KP floats (packed lower triangle of the Gramian, then b); the rows
                 // are solved afterwards by als_solve_packed_kernel with every warp of the SM; null = solve in this kernel
  int out_row0;  // local row stored at out[0] (the buffer covers one tile of rows)
};

template <bool IMPLICIT>
__global__ void __launch_bounds__(NTHREADS, 1) als_solve_tc_kernel(const TcParams tp) {
  // direct cast (no integer round-trip) so the compiler keeps the shared address space: LDS/STS, not generic LD/ST
  extern __shared__ __align__(1024) unsigned char smem_raw[];
  Smem& sm = *reinterpret_cast<Smem*>(smem_raw);
  if (threadIdx.x == 0 && (s32(smem_raw) & 127u) != 0u) __trap();   // the stage ring is laid out for 128-byte alignment
  const SolveParams& p = tp.sp;
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;

  if (tid == 0) {
    for (int i = 0; i < NSTAGE; ++i) {
      mbar_init(&sm.full[i], 1);
    }
    sm.consumed = 0;
    for (int i = 0; i < NRAW; ++i) {
      mbar_init(&sm.rawfull[i], 32);   // every lane of the gather warp: cp.async.mbarrier.arrive.noinc
      mbar_init(&sm.rawempty[i], 1);
    }
    for (int t = 0; t < NTEAM; ++t)
      for (int bf = 0; bf < 2; ++bf) {
        mbar_init(&sm.descfull[t][bf], 1);
        mbar_init(&sm.teamdone[t][bf], NSLOT);
        mbar_init(&sm.bfull[t][bf], 1);
      }
    fence_barrier_init();
  }
  __syncthreads();

  long long tacc[8] = {0, 0, 0, 0, 0, 0, 0, 0};
  // per-role cycle counters are compiled in only with -DPIO_TC_TIMING=1 (tools/tc_timing.py); the default build carries no
  // instrumentation in the hot loops
  const bool timing = PIO_TC_TIMING && tp.timing != nullptr;
  long long t0_ = 0;
#define T_BEGIN() do { if (timing) t0_ = clock64(); } while (0)
#define T_END(i) do { if (timing) tacc[i] += clock64() - t0_; } while (0)
  const long long tstart_ = timing ? clock64() : 0;

  if (warp == 0) {
    // ================= scheduler =================
    // Warp-parallel: lane li = t*4+s (< 12) keeps the state of row lane (team t, slot s) in registers; every control
    // decision is warp-uniform.  Static row assignment (no atomics): rows are degree-sorted; groups of 12 consecutive
    // rows are dealt to the CTAs in snake order, lane li of this CTA takes row  g*12 + li  of its k-th group g.  The row
    // pointers of a lane's NEXT row are prefetched while the current one is processed.
    const int per_cta = NTEAM * NSLOT;
    const int nrows = p.row_end - p.row_begin;
    const int ngroups = (nrows + per_cta - 1) / per_cta;
    const int G = (int)gridDim.x;
    auto row_of = [&](int k) -> int {
      const long long g = (long long)k * G + ((k & 1) ? (G - 1 - (int)blockIdx.x) : (int)blockIdx.x);
      if (lane >= per_cta || g >= ngroups) return -1;
      const long long r = (long long)p.row_begin + g * per_cta + lane;
      return r < p.row_end ? (int)r : -1;
    };
    int my_row = -1, my_k = 0;
    long long my_pos = 0, my_end = 0;
    bool my_first = false;
    int nx_row = row_of(0);
    long long nx_beg = 0, nx_end = 0;
    if (nx_row >= 0) { nx_beg = p.ptr[nx_row]; nx_end = p.ptr[nx_row + 1]; }
    uint32_t exited = 0;
    uint32_t nbp = 0;                // batches published per team, 8 bits each (only the low two bits are ever used)
    uint32_t it = 0;                 // global stage counter: stages are produced and consumed in publish order
    auto nb_of = [&](int t) -> int { return (int)((nbp >> (8 * t)) & 3u); };
    // publish the next batch of team t; returns false when the team has nothing left (an exit descriptor is published)
    auto build = [&](int t) -> bool {
      const int nbt = nb_of(t);
      const int bf = nbt & 1;
      T_BEGIN();
      mbar_wait(&sm.teamdone[t][bf], ((nbt >> 1) & 1) ^ 1);
      T_END(0);
      T_BEGIN();
      BatchDesc& d = sm.desc[t][bf];
      const bool mine = lane < per_cta && (lane >> 2) == t;
      int len = 0;
      long long beg = 0;
      if (mine) {
        if (my_row >= 0 && my_pos >= my_end) my_row = -1;
        if (my_row < 0 && nx_row >= 0) {
          my_row = nx_row;
          my_pos = nx_beg;
          my_end = nx_end;
          my_first = true;
          ++my_k;
          nx_row = row_of(my_k);   // prefetch the pointers of the row after this one
          if (nx_row >= 0) { nx_beg = __ldg(p.ptr + nx_row); nx_end = __ldg(p.ptr + nx_row + 1); }
        }
        const int s = lane & 3;
        if (my_row >= 0) {
          long long e = my_pos + SEG;
          if (e > my_end) e = my_end;
          len = (int)(e - my_pos);
          beg = my_pos;
          d.row[s] = my_row;
          d.first[s] = my_first ? 1 : 0;
          d.last[s] = e == my_end;
          my_first = false;
          my_pos = e;
        } else {
          d.row[s] = -1;
          d.first[s] = 0;
          d.last[s] = 0;
        }
      }
      const int nst = (len + STAGE_RATINGS - 1) / STAGE_RATINGS;
      int n_[NSLOT], l_[NSLOT];
      long long b_[NSLOT];
#pragma unroll
      for (int s = 0; s < NSLOT; ++s) {
        n_[s] = __shfl_sync(0xffffffffu, nst, t * NSLOT + s);
        l_[s] = __shfl_sync(0xffffffffu, len, t * NSLOT + s);
        b_[s] = __shfl_sync(0xffffffffu, beg, t * NSLOT + s);
      }
      const int ns = n_[0] + n_[1] + n_[2] + n_[3];
      for (int e = lane; e < ns; e += 32) {   // the flat stage list, one entry per lane and pass
        int s = 0, q = e;
#pragma unroll
        for (int k = 0; k < NSLOT - 1; ++k)
          if (s == k && q >= n_[k]) { q -= n_[k]; s = k + 1; }
        const int ls = s == 0 ? l_[0] : (s == 1 ? l_[1] : (s == 2 ? l_[2] : l_[3]));
        const int nn = s == 0 ? n_[0] : (s == 1 ? n_[1] : (s == 2 ? n_[2] : n_[3]));
        const long long bs = s == 0 ? b_[0] : (s == 1 ? b_[1] : (s == 2 ? b_[2] : b_[3]));
        StageEnt se;
        se.beg = bs + (long long)q * STAGE_RATINGS;
        const int v = ls - q * STAGE_RATINGS;
        se.valid = v < STAGE_RATINGS ? v : STAGE_RATINGS;
        se.info = s | (q == nn - 1 ? 4 : 0) | (q == 0 ? 16 : 0) | (e == ns - 1 ? 8 : 0);
        d.st[e] = se;
      }
      const bool any = ns > 0;
      if (lane == 0) {
        d.nstages = ns;
        d.exit = any ? 0 : 1;
        d.stage0 = it;
      }
      it += (uint32_t)ns;
      __syncwarp();
      if (lane == 0) mbar_arrive(&sm.descfull[t][bf]);
      nbp = (nbp & ~(0xffu << (8 * t))) | ((((nbp >> (8 * t)) + 1u) & 3u) << (8 * t));
      if (!any) exited |= 1u << t;
      T_END(3);
      return any;
    };
    // teams in round-robin order, skipping those that have exited (the producers walk the descriptors in the same
    // order); build() waits until the team's descriptor buffer is free, i.e. its batch before last is solved
    int cursor = 0;
    while (true) {
      int t = -1;
      for (int k = 0; k < NTEAM && t < 0; ++k)
        if (!((exited >> ((cursor + k) % NTEAM)) & 1u)) t = (cursor + k) % NTEAM;
      if (t < 0) break;
      cursor = (t + 1) % NTEAM;
      build(t);
    }
    __syncwarp();
  } else if (warp < TEAM0) {
    // ================= producers =================
    // warp 1 = gather warp: walks the scheduler's stage lists and, per stage, starts one 256-byte cp.async.bulk
    //          copy per rating into the raw ring (completion counted on rawfull[]); source indices are loaded
    //          two stages ahead into a register shift queue.
    // converters: converter cw owns the stages whose number inside their segment is cw mod NCONV: it waits for the
    //          raw rows, scales, splits hi/lo and writes all three K-blocks of the wgmma tiles (three independent
    //          pieces of work per dependency chain), then hands the stage to the team that consumes it.
    // cursor over the published stage lists (scalars only)
    uint32_t c_ex = 0, c_par = 0;
    int c_cur = 0, c_t = 0, c_b = 0, c_i = -1, c_n = 0;
    bool c_done = false;
    auto next_batch = [&](bool blocking) -> bool {   // -> first stage of the next batch; false if finished / not published yet
      while (true) {
        int nt = -1;
#pragma unroll
        for (int k = 0; k < NTEAM; ++k) {
          const int cand = (c_cur + k) % NTEAM;
          if (nt < 0 && !((c_ex >> cand) & 1u)) nt = cand;
        }
        if (nt < 0) { c_done = true; return false; }
        const uint32_t cnt = (c_par >> (2 * nt)) & 3u;   // batches of team nt consumed so far, mod 4
        const int nbf = (int)(cnt & 1u);
        const uint32_t pb = (cnt >> 1) & 1u;
        if (blocking) mbar_wait(&sm.descfull[nt][nbf], pb);
        else if (!mbar_test(&sm.descfull[nt][nbf], pb)) return false;
        c_par = (c_par & ~(3u << (2 * nt))) | (((cnt + 1u) & 3u) << (2 * nt));
        c_cur = (nt + 1) % NTEAM;
        if (sm.desc[nt][nbf].exit) { c_ex |= 1u << nt; continue; }
        c_t = nt;
        c_b = nbf;
        c_n = sm.desc[nt][nbf].nstages;
        c_i = 0;
        return true;
      }
    };
    auto advance = [&](bool blocking) -> bool {
      if (c_done) return false;
      if (c_i >= 0 && c_i + 1 < c_n) { ++c_i; return true; }
      return next_batch(blocking);
    };
    if (warp < CONV0) {
      // ---------------- gather warps: warp gw issues every stage with (stage number % NGATHER == gw) ----------------
      // queue of this warp's next two stages (global stage number, beg, valid, source index) in registers; q0 is issued next
      const int gw = warp - 1;
      long long qbeg0 = 0, qbeg1 = 0;
      int qval0 = -1, qval1 = -1;      // valid count; -1 = empty queue slot
      int qidx0 = -1, qidx1 = -1;
      uint32_t qn0 = 0, qn1 = 0;
      uint32_t n_seen = 0;             // stages walked so far (all warps' stages)
      bool more = true;
      // pull this warp's next stage and start its index load; the look-ahead never blocks on a descriptor (the scheduler
      // may hold the next batch back until the MMAs of the current one - which need the stage still queued here - are issued)
      auto fetch = [&](uint32_t& qn, long long& qb, int& qv, int& qi, bool blocking) {
        qv = -1;
        while (more) {
          T_BEGIN();
          const bool ok = advance(blocking);
          T_END(0);
          if (!ok) {
            if (c_done) more = false;
            return;
          }
          const uint32_t n = n_seen++;
          if ((n % NGATHER) != (uint32_t)gw) continue;
          const StageEnt se = sm.desc[c_t][c_b].st[c_i];
          qn = n;
          qb = se.beg;
          qv = se.valid;
          qi = -1;
          if (lane < se.valid) qi = __ldg(p.idx + se.beg + lane);
          return;
        }
      };
      while (true) {
        if (qval0 < 0) {
          if (qval1 >= 0) { qn0 = qn1; qbeg0 = qbeg1; qval0 = qval1; qidx0 = qidx1; qval1 = -1; }
          else fetch(qn0, qbeg0, qval0, qidx0, true);    // nothing pending in this warp: safe to block
          if (qval0 < 0) break;                          // finished
        }
        if (qval1 < 0) fetch(qn1, qbeg1, qval1, qidx1, false);
        const int rs = qn0 % NRAW;
        T_BEGIN();
        // the slot's previous use (stage qn0 - NRAW) must have been loaded by its converter; waiting for the consumption of
        // stage qn0 - 2 NRAW first keeps this wait less than one lap ahead of the slot, so its parity is unambiguous
        wait_count(&sm.consumed, qn0 + 1 - 2 * NRAW);
        mbar_wait(&sm.rawempty[rs], ((qn0 / NRAW) & 1) ^ 1);   // the converter is done with this raw slot
        T_END(1);
        T_BEGIN();
        // lane = (row parity, 16-byte chunk): one LDGSTS moves two whole 256-byte rows per warp instruction
#pragma unroll
        for (int i = 0; i < STAGE_RATINGS / 2; ++i) {
          const int r = 2 * i + (lane >> 4);
          const int si = __shfl_sync(0xffffffffu, qidx0, r);
          if (2 * i < qval0 && si >= 0)
            cp_async16(&sm.raw[rs][r * RAW_ROW + (lane & 15) * 16], p.src + (size_t)si * KP + (lane & 15) * 4);
        }
        if (lane < qval0) cp_async4(&sm.rawval[rs][lane], p.val + qbeg0 + lane);
        cp_async_mbar_arrive_noinc(&sm.rawfull[rs]);
        T_END(2);
        qval0 = -1;
      }
    } else {
      // ---------------- converters ----------------
      const int cw = warp - CONV0;
      // lane -> (rating kr inside a K-block, source float4 groups sg_j = sgb + 4 j): a quarter-warp holds 4 ratings
      // (kr%4 = 0..3) x 2 halves of one 32-byte chunk -> its 8 STS.128 hit 8 distinct 16-byte bank groups
      const int kr = ((lane >> 3) & 1) * 4 + (lane & 3);
      const int sgb = ((lane >> 2) & 1) + 2 * (lane >> 4);
      uint32_t it = 0;   // global stage counter (wgmma ring + raw ring)
      uint32_t qs = 0;   // stage number inside the current segment: decides the owner, so that the grouping of a row's
                         // right-hand-side partial sums depends on the row alone (not on what else this CTA processes)
      float bacc[4][4];
#pragma unroll
      for (int j = 0; j < 4; ++j)
#pragma unroll
        for (int c = 0; c < 4; ++c) bacc[j][c] = 0.f;
      while (true) {
        T_BEGIN();
        const bool ok = advance(true);
        T_END(0);
        if (!ok) break;
        const StageEnt se = sm.desc[c_t][c_b].st[c_i];
        if (se.info & 16) qs = 0;
        const bool mine = (qs % NCONV) == (uint32_t)cw;
        ++qs;
        if (mine) {
          const int rs = it % NRAW;
          const int st = it % NSTAGE;
          T_BEGIN();
          wait_count(&sm.consumed, it + 1 - NRAW);             // stage it - NRAW has landed (keeps the parity below unambiguous)
          mbar_wait(&sm.rawfull[rs], (it / NRAW) & 1);           // gathered rows have landed
          T_END(1);
          T_BEGIN();
          // all shared-memory loads of the stage first (12 independent LDS.128 + 3 ratings), then arithmetic + stores
          float4 y[STAGE_KB][4];
          float cv[STAGE_KB];
#pragma unroll
          for (int kb = 0; kb < STAGE_KB; ++kb) {
            const int r = kb * KB_RATINGS + kr;                  // rating inside the stage
            const bool live = r < se.valid;
            cv[kb] = live ? sm.rawval[rs][r] : 0.f;
            const unsigned char* rrow = &sm.raw[rs][r * RAW_ROW];
#pragma unroll
            for (int j = 0; j < 4; ++j) {
              y[kb][j] = make_float4(0.f, 0.f, 0.f, 0.f);
              if (live) y[kb][j] = *reinterpret_cast<const float4*>(rrow + (sgb + 4 * j) * 16);
            }
          }
          // the raw slot is in registers now: hand it back to the gather warps before converting
          __syncwarp();
          if (lane == 0) mbar_arrive(&sm.rawempty[rs]);
          T_END(3);
          T_BEGIN();
          wait_count(&sm.consumed, it + 1 - NSTAGE);            // wgmma stage is free: stage it - NSTAGE consumed
          T_END(2);
          T_BEGIN();
#pragma unroll
          for (int kb = 0; kb < STAGE_KB; ++kb) {
            if (kb * KB_RATINGS < se.valid) {
              const float cval = cv[kb];
              float wb, sc;
              if (IMPLICIT) {
                const float c1 = p.alpha * fabsf(cval);
                wb = cval > 0.f ? 1.f + c1 : 0.f;
                sc = sqrtf(c1);
              } else {
                wb = cval;
                sc = 1.f;
              }
              unsigned char* kbp = &sm.stage[st][0] + kb * KB_BYTES;
#pragma unroll
              for (int j = 0; j < 4; ++j) {
                const int sg = sgb + 4 * j;
                // features 4sg..4sg+3 of rating kr: four 4-byte stores 16 bytes apart; over the warp the rating halves
                // (144 B = 4 banks apart), feature groups (288 B = 8 banks) and sgb parity (64 B = 16 banks) spread
                // the 32 lanes over 32 distinct banks
                const int off = tile_off(4 * sg, kr);
                const float4 yy = y[kb][j];
                bacc[j][0] = fmaf(wb, yy.x, bacc[j][0]);
                bacc[j][1] = fmaf(wb, yy.y, bacc[j][1]);
                bacc[j][2] = fmaf(wb, yy.z, bacc[j][2]);
                bacc[j][3] = fmaf(wb, yy.w, bacc[j][3]);
                float4 x = yy;
                if (IMPLICIT) { x.x *= sc; x.y *= sc; x.z *= sc; x.w *= sc; }
                float4 hi, lo;
                hi.x = tf32_round(x.x); hi.y = tf32_round(x.y); hi.z = tf32_round(x.z); hi.w = tf32_round(x.w);
                lo.x = x.x - hi.x; lo.y = x.y - hi.y; lo.z = x.z - hi.z; lo.w = x.w - hi.w;
                float* ph = reinterpret_cast<float*>(kbp + off);
                float* pl = reinterpret_cast<float*>(kbp + TILE_BYTES + off);
                ph[0] = hi.x; ph[4] = hi.y; ph[8] = hi.z; ph[12] = hi.w;
                pl[0] = lo.x; pl[4] = lo.y; pl[8] = lo.z; pl[12] = lo.w;
              }
            }
          }
          fence_proxy_async();
          __syncwarp();
          if (lane == 0) mbar_arrive(&sm.full[st]);       // -> MMA issuer
          T_END(4);
        }
        ++it;
        if (se.info & 4) {
          // end of a segment: every converter reduces its share of b over the 8 rating lanes, then the shares are added
          const int sslot = se.info & 3;
#pragma unroll
          for (int j = 0; j < 4; ++j)
#pragma unroll
            for (int c = 0; c < 4; ++c) {
              float v = bacc[j][c];
              v += __shfl_xor_sync(0xffffffffu, v, 1);
              v += __shfl_xor_sync(0xffffffffu, v, 2);
              v += __shfl_xor_sync(0xffffffffu, v, 8);
              bacc[j][c] = v;
            }
          named_bar_sync(1, NCONV * 32);  // bpart free (previous segment's sum was read)
          if (kr == 0) {
#pragma unroll
            for (int j = 0; j < 4; ++j)
              *reinterpret_cast<float4*>(&sm.bpart[cw][(sgb + 4 * j) * 4]) = make_float4(bacc[j][0], bacc[j][1], bacc[j][2], bacc[j][3]);
          }
          named_bar_sync(1, NCONV * 32);
          if (cw == 0) {
            for (int c = lane; c < KP; c += 32) {
              float acc = sm.bpart[0][c];
#pragma unroll
              for (int w = 1; w < NCONV; ++w) acc += sm.bpart[w][c];   // fixed order
              sm.bstage[c_t][c_b][sslot][c] = acc;
            }
            if (se.info & 8) {   // every right-hand side of this batch is in bstage[t][buf]
              __syncwarp();
              if (lane == 0) mbar_arrive(&sm.bfull[c_t][c_b]);
            }
          }
#pragma unroll
          for (int j = 0; j < 4; ++j)
#pragma unroll
            for (int c = 0; c < 4; ++c) bacc[j][c] = 0.f;
        }
      }
    }
  } else {
    // ================= teams: wgmma + solve =================
    const int t = (warp - TEAM0) / 4;
    const int slot = (warp - TEAM0) % 4;     // the row this warp solves
    const int wq = warp & 3;                 // rank of this warp in its warpgroup: accumulator rows 16wq..16wq+15
    const int barid = 2 + t;
    float acc[32];
#pragma unroll
    for (int i = 0; i < 32; ++i) acc[i] = 0.f;
    // accumulator -> A slot (packed lower triangle, as chol_solve_warp<PACKED_IN> reads it), overwriting for the first
    // stage of a row, adding otherwise.  Fragment of m64n64: acc[i] is row 16wq + lane/4 + 8((i/2)%2), column
    // 8(i/4) + 2(lane%4) + i%2; every element has one owner thread, so the adds need no synchronisation.
    auto drain = [&](float* as, bool overwrite) {
#pragma unroll
      for (int i = 0; i < 32; ++i) {
        const int r = 16 * wq + (lane >> 2) + 8 * ((i >> 1) & 1);
        const int c = 8 * (i >> 2) + 2 * (lane & 3) + (i & 1);
        if (c > r) continue;
        const int o = r < H ? r * (r + 1) / 2 + c : (c < H ? OFF21 + (r - H) * L21S + c : OFF22 + (r - H) * (r - H + 1) / 2 + (c - H));
        as[o] = overwrite ? acc[i] : as[o] + acc[i];
      }
    };
    int nb = 0;
    while (true) {
      const int bf = nb & 1;
      const uint32_t ph = (nb >> 1) & 1;
      T_BEGIN();
      mbar_wait(&sm.descfull[t][bf], ph);
      T_END(0);
      const BatchDesc& d = sm.desc[t][bf];
      if (d.exit) break;
      // every warp of the team must have finished solving the previous batch before any A slot is overwritten
      named_bar_sync(barid, 128);
      // this batch's turn: every earlier stage has been consumed (by the other teams), so the slot of each of its stages
      // is at most one lap ahead and the parity wait on full[] below is unambiguous
      wait_count(&sm.consumed, d.stage0);
      __syncwarp();
      // ---- the batch's stages in order: slot 0's segment, then slot 1's, ...; every stage's sum goes into its slot's A
      // (fp32 adds in stage order: deterministic)
      const int nst = d.nstages;
      for (int i = 0; i < nst; ++i) {
        const uint32_t g = d.stage0 + (uint32_t)i;
        const int st = (int)(g % NSTAGE);
        const int valid = d.st[i].valid;
        const int info = d.st[i].info;
        T_BEGIN();
        mbar_wait(&sm.full[st], (g / NSTAGE) & 1);
        __syncwarp();   // wgmma is warp-synchronous: reconverge after the polling loop
        T_END(1);
        T_BEGIN();
        const int nkb = (valid + KB_RATINGS - 1) / KB_RATINGS;
        const uint32_t base = s32(&sm.stage[st][0]);
        wgmma_fence();
        for (int kb = 0; kb < nkb; ++kb) {   // the small cross terms first; the first wgmma of the stage starts from zero
          const uint64_t dh = make_desc(base + kb * KB_BYTES);
          const uint64_t dl = make_desc(base + kb * KB_BYTES + TILE_BYTES);
          wgmma_tf32(acc, dl, dh, kb == 0 ? 0u : 1u);                      // lo hi^T
          wgmma_tf32(acc, dh, dl, 1u);                                     // hi lo^T
        }
        for (int kb = 0; kb < nkb; ++kb) {
          const uint64_t dh = make_desc(base + kb * KB_BYTES);
          wgmma_tf32(acc, dh, dh, 1u);                                     // hi hi^T
        }
        wgmma_commit();
        wgmma_wait_all();
#pragma unroll
        for (int j = 0; j < 32; ++j) acc_fence(acc[j]);
        named_bar_sync(barid, 128);                                      // no warp of the team reads the stage any more
        if (wq == 0 && lane == 0) st_release(&sm.consumed, g + 1);
        drain(&sm.aslot[t][info & 3][0], (info & 16) && d.first[info & 3] != 0);
        T_END(2);
      }
      __syncwarp();
      // right-hand side of this segment
      T_BEGIN();
      mbar_wait(&sm.bfull[t][bf], ph);
      T_END(3);
      {
        const int tt = (warp - TEAM0) % 4 * 32 + lane;  // 0..127 within the team
        for (int o = tt; o < NSLOT * KP; o += 128) {
          const int s = o / KP, c = o % KP;
          if (d.row[s] >= 0) sm.bslot[t][s][c] = d.first[s] ? sm.bstage[t][bf][s][c] : sm.bslot[t][s][c] + sm.bstage[t][bf][s][c];
        }
      }
      T_BEGIN();
      named_bar_sync(barid, 128);
      T_END(4);
      T_BEGIN();
      // ---- solve
      const int r = d.row[slot];
      if (r >= 0 && d.last[slot] && tp.dbg) {
        float* o = tp.dbg + (size_t)r * (ASLOT + KP);
        for (int c = lane; c < ASLOT; c += 32) o[c] = sm.aslot[t][slot][c];
        for (int c = lane; c < KP; c += 32) o[ASLOT + c] = sm.bslot[t][slot][c];
        __syncwarp();
      }
      if (r >= 0 && d.last[slot] && tp.out) {
        // split mode: hand the finished normal equations to the solver kernel (coalesced 16-byte stores)
        float4* o4 = reinterpret_cast<float4*>(tp.out + (size_t)(r - tp.out_row0) * (ASLOT + KP));
        const float4* a4 = reinterpret_cast<const float4*>(&sm.aslot[t][slot][0]);
        for (int c = lane; c < ASLOT / 4; c += 32) o4[c] = a4[c];
        const float4* b4 = reinterpret_cast<const float4*>(&sm.bslot[t][slot][0]);
        if (lane < KP / 4) o4[ASLOT / 4 + lane] = b4[lane];
      } else if (r >= 0 && d.last[slot]) {
        const float ridge = p.lambda * p.nreg[r];
        chol_solve_warp<KP, 8, 72, IMPLICIT, true>(&sm.aslot[t][slot][0], &sm.bslot[t][slot][0], p.yty, ridge, p.k,
                                                   &sm.colbuf[t * NSLOT + slot][0], &sm.dinv[t * NSLOT + slot][0],
                                                   p.dst + (size_t)(p.dst_row_offset + r) * KP, p.fail);
      }
      __syncwarp();
      T_END(5);
      if (lane == 0) mbar_arrive(&sm.teamdone[t][bf]);
      ++nb;
    }
  }
  if (timing && lane == 0) {
    tacc[7] = clock64() - tstart_;
    for (int i = 0; i < 8; ++i) tp.timing[((size_t)blockIdx.x * 16 + warp) * 8 + i] = tacc[i];
  }
}

// ---- split mode, second half: one warp per row solves the normal equations the tensor-core kernel left in `in`
// (ASLOT + KP floats per local row). 128-thread CTAs, four per SM by registers: all 16 resident warps factorise.
constexpr int SOLVE_WARPS = 4;
constexpr int SOLVE_SMEM_PER_WARP = ASLOT + KP + 2 * KP + KP;   // slot, b, column double buffer, 1/diag
template <bool IMPLICIT>
__global__ void __launch_bounds__(SOLVE_WARPS * 32, 3) als_solve_packed_kernel(const SolveParams p, const float* __restrict__ in, int in_row0) {
  extern __shared__ __align__(16) float solve_smem[];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  float* slot = solve_smem + warp * SOLVE_SMEM_PER_WARP;
  float* bv = slot + ASLOT;
  float* colbuf = bv + KP;
  float* dinv = colbuf + 2 * KP;
  const int nwarps = gridDim.x * SOLVE_WARPS;
  for (int r = p.row_begin + blockIdx.x * SOLVE_WARPS + warp; r < p.row_end; r += nwarps) {
    const float4* src = reinterpret_cast<const float4*>(in + (size_t)(r - in_row0) * (ASLOT + KP));
    float4* dst4 = reinterpret_cast<float4*>(slot);
    for (int c = lane; c < (ASLOT + KP) / 4; c += 32) cp_async16(dst4 + c, src + c);
    cp_async_commit();
    cp_async_wait<0>();
    __syncwarp();
    chol_solve_warp<KP, 8, 72, IMPLICIT, true>(slot, bv, p.yty, p.lambda * p.nreg[r], p.k, colbuf, dinv,
                                               p.dst + (size_t)(p.dst_row_offset + r) * KP, p.fail);
    __syncwarp();
  }
}

// what the host launcher needs to know about this role partition
struct Api {
  using Params = TcParams;
  static constexpr int kPerCta = NTEAM * NSLOT;       // rows in flight per CTA (one group of the static assignment)
  static constexpr int kThreads = NTHREADS;
  static constexpr size_t kSmem = sizeof(Smem) + 1024;
  static constexpr int kRowFloats = ASLOT + KP;       // split mode / debug dump: floats per row
  static constexpr int kSolveWarps = SOLVE_WARPS;
  static constexpr size_t kSolveSmem = sizeof(float) * SOLVE_WARPS * SOLVE_SMEM_PER_WARP;
  static void (*kernel(bool imp))(const TcParams) { return imp ? als_solve_tc_kernel<true> : als_solve_tc_kernel<false>; }
  static void (*solver(bool imp))(const SolveParams, const float*, int) {
    return imp ? als_solve_packed_kernel<true> : als_solve_packed_kernel<false>;
  }
};

}  // namespace TC_NS
}  // namespace pio
