// pio_als.cu -- C-ABI implementation (see include/pio_als.h for the reference interfaces each
// entry point replaces).  Host orchestration only; all arithmetic is in the CUDA kernels of
// als_kernels.cuh / sort_scan.cuh / topk.cuh.  Which kernels a half-step or a scoring call runs, and with
// what geometry, is planned by solve_plan.h and score_plan.h; this file executes the plans.  No CPU
// fallback: without a usable sm_90 device every computing entry point returns PIO_ALS_ERR_CUDA.
#include "../../include/pio_als.h"

#include <cuda_runtime.h>
#include <dlfcn.h>
#include <math.h>
#include <nccl.h>
#include <stdarg.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

#include <chrono>
#include <algorithm>
#include <deque>
#include <exception>
#include <map>
#include <mutex>
#include <string>
#include <type_traits>
#include <vector>

#include "als_kernels.cuh"
#include "als_mma_kernel.cuh"
#include "als_pair_kernel.cuh"
// the wgmma half-step kernel; the header is parametrised by the role partition of its sixteen warps: 2 gather +
// 5 converter warps + 2 teams (one warpgroup each, so that one team consumes stages while the other solves).  Six
// wgmma stages and seven raw stages fill the 227 KB of shared memory a block may use.
#define TC_NS tc
#define TC_NTEAM 2
#define TC_NCONV 5
#define TC_NGATHER 2
#define TC_NSTAGE 6
#define TC_NRAW 7
#include "als_tc_kernel.cuh"
#undef TC_NS
#undef TC_NTEAM
#undef TC_NCONV
#undef TC_NGATHER
#undef TC_NSTAGE
#undef TC_NRAW
#include "sort_scan.cuh"
#include "topk.cuh"
#include "score_plan.h"
#include "solve_plan.h"
#include "ids_encode.cuh"
#include "events_scan.cuh"
#include "events_fold.cuh"
#include "cooc.cuh"

namespace pio {

static thread_local std::string g_create_error;

static int ceil_log2(uint64_t n) {
  int b = 0;
  while (b < 63 && (1ull << b) < n) ++b;
  return b < 1 ? 1 : b;
}
static int pad_rank(int k) { return k <= 16 ? 16 : k <= 32 ? 32 : k <= 64 ? 64 : 128; }

// ---------------------------------------------------------------------------------------------
// NCCL through dlopen: the library has no link-time NCCL dependency and shares whichever libnccl
// the host process already loaded (torch's bundled one under torchrun, the system one under a JVM).
// ---------------------------------------------------------------------------------------------
struct NcclApi {
  void* lib = nullptr;
  ncclResult_t (*GetUniqueId)(ncclUniqueId*) = nullptr;
  ncclResult_t (*CommInitRank)(ncclComm_t*, int, ncclUniqueId, int) = nullptr;
  ncclResult_t (*AllGather)(const void*, void*, size_t, ncclDataType_t, ncclComm_t, cudaStream_t) = nullptr;
  ncclResult_t (*AllReduce)(const void*, void*, size_t, ncclDataType_t, ncclRedOp_t, ncclComm_t, cudaStream_t) = nullptr;
  ncclResult_t (*Send)(const void*, size_t, ncclDataType_t, int, ncclComm_t, cudaStream_t) = nullptr;
  ncclResult_t (*Recv)(void*, size_t, ncclDataType_t, int, ncclComm_t, cudaStream_t) = nullptr;
  ncclResult_t (*GroupStart)() = nullptr;
  ncclResult_t (*GroupEnd)() = nullptr;
  ncclResult_t (*CommDestroy)(ncclComm_t) = nullptr;
  const char* (*GetErrorString)(ncclResult_t) = nullptr;
  bool ok = false;
};
static NcclApi& nccl_api() {
  static NcclApi api;
  static std::once_flag once;
  std::call_once(once, [] {
    void* lib = dlopen("libnccl.so.2", RTLD_NOW | RTLD_NOLOAD | RTLD_GLOBAL);
    if (!lib) lib = dlopen("libnccl.so.2", RTLD_NOW | RTLD_GLOBAL);
    if (!lib) lib = dlopen("libnccl.so", RTLD_NOW | RTLD_GLOBAL);
    if (!lib) return;
    api.lib = lib;
    api.GetUniqueId = (decltype(api.GetUniqueId))dlsym(lib, "ncclGetUniqueId");
    api.CommInitRank = (decltype(api.CommInitRank))dlsym(lib, "ncclCommInitRank");
    api.AllGather = (decltype(api.AllGather))dlsym(lib, "ncclAllGather");
    api.AllReduce = (decltype(api.AllReduce))dlsym(lib, "ncclAllReduce");
    api.Send = (decltype(api.Send))dlsym(lib, "ncclSend");
    api.Recv = (decltype(api.Recv))dlsym(lib, "ncclRecv");
    api.GroupStart = (decltype(api.GroupStart))dlsym(lib, "ncclGroupStart");
    api.GroupEnd = (decltype(api.GroupEnd))dlsym(lib, "ncclGroupEnd");
    api.CommDestroy = (decltype(api.CommDestroy))dlsym(lib, "ncclCommDestroy");
    api.GetErrorString = (decltype(api.GetErrorString))dlsym(lib, "ncclGetErrorString");
    api.ok = api.GetUniqueId && api.CommInitRank && api.AllGather && api.CommDestroy && api.AllReduce && api.Send &&
             api.Recv && api.GroupStart && api.GroupEnd;
  });
  return api;
}

// ---------------------------------------------------------------------------------------------
// small kernels of the ingest / model plumbing
// ---------------------------------------------------------------------------------------------
__global__ void validate_coo_kernel(const int* u, const int* i, long long n, int nu, int ni, int* bad) {
  const long long e = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (e < n && (u[e] < 0 || u[e] >= nu || i[e] < 0 || i[e] >= ni)) atomicAdd(bad, 1);
}
__global__ void make_keys_ext_kernel(const int* u, const int* i, long long n, int bits_i, uint64_t* keys,
                                     uint32_t* pay) {
  const long long e = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (e < n) {
    keys[e] = ((uint64_t)(uint32_t)u[e] << bits_i) | (uint64_t)(uint32_t)i[e];
    pay[e] = (uint32_t)e;
  }
}
__global__ void head_flags_kernel(const uint64_t* keys, long long n, uint32_t* flag) {
  const long long e = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (e < n) flag[e] = (e == 0 || keys[e] != keys[e - 1]) ? 1u : 0u;
}
// one thread per run head: fold the run in event order (sum) or pick the latest event (keep-last)
__global__ void dedup_compact_kernel(const uint64_t* keys, const uint32_t* pay, const uint32_t* pos,
                                     long long n, int bits_i, const float* rating, const long long* ts,
                                     int mode, int* ou, int* oi, float* orr) {
  const long long e = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (e >= n) return;
  const uint64_t key = keys[e];
  if (e > 0 && keys[e - 1] == key) return;
  float acc;
  if (mode == PIO_ALS_DEDUP_SUM) {
    acc = 0.f;
    for (long long t = e; t < n && keys[t] == key; ++t) acc += rating[pay[t]];
  } else {
    long long best_t = ts ? ts[pay[e]] : 0;
    uint32_t best_p = pay[e];
    for (long long t = e + 1; t < n && keys[t] == key; ++t) {
      const uint32_t pp = pay[t];
      const long long tt = ts ? ts[pp] : 0;
      if (tt >= best_t) { best_t = tt; best_p = pp; }  // payload order == event order (stable sort)
    }
    acc = rating[best_p];
  }
  const uint32_t o = pos[e];
  ou[o] = (int)(key >> bits_i);
  oi[o] = (int)(key & ((1ull << bits_i) - 1ull));
  orr[o] = acc;
}
__global__ void degree_kernel(const int* u, const int* i, const float* r, long long n, uint32_t* du,
                              uint32_t* di, uint32_t* pu, uint32_t* pi) {
  const long long e = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (e >= n) return;
  atomicAdd(&du[u[e]], 1u);
  atomicAdd(&di[i[e]], 1u);
  if (r[e] > 0.f) {
    atomicAdd(&pu[u[e]], 1u);
    atomicAdd(&pi[i[e]], 1u);
  }
}
__global__ void degree_keys_kernel(const uint32_t* deg, int n, uint64_t* keys, uint32_t* pay) {
  const int r = blockIdx.x * blockDim.x + threadIdx.x;
  if (r < n) {
    keys[r] = (uint64_t)(0xFFFFFFFFu - deg[r]);
    pay[r] = (uint32_t)r;
  }
}
// sorted position p -> internal id: rows are dealt to ranks in snake order so every rank gets
// the same number of rows and a near-equal share of the ratings; a rank's rows stay
// degree-descending.
__global__ void assign_internal_kernel(const uint32_t* order, int n, int W, int R, int* perm, int* inv, int* rpos,
                                       int* p2i) {
  const int p = blockIdx.x * blockDim.x + threadIdx.x;
  if (p >= n) return;
  const int row = (int)order[p];
  const int blk = p / W, pos = p % W;
  const int rk = (blk & 1) ? (W - 1 - pos) : pos;
  const int internal = rk * R + blk;
  perm[row] = internal;
  inv[internal] = row;
  rpos[row] = p;       // degree-rank position: independent of the number of GPUs
  p2i[p] = internal;
}
// sharded ingest: destination rank of every event (by user residue for the dedup pass, by row owner for the CSR passes)
__global__ void dest_mod_kernel(const int* u, long long n, int W, uint64_t* keys, uint32_t* pay) {
  const long long e = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (e < n) {
    keys[e] = (uint64_t)((uint32_t)u[e] % (uint32_t)W);
    pay[e] = (uint32_t)e;
  }
}
__global__ void dest_owner_kernel(const int* rowext, long long n, const int* perm, int R, uint64_t* keys, uint32_t* pay) {
  const long long e = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (e < n) {
    keys[e] = (uint64_t)(perm[rowext[e]] / R);
    pay[e] = (uint32_t)e;
  }
}
template <class T>
__global__ void gather_by_index_kernel(const T* in, const uint32_t* idx, long long n, T* out) {
  const long long e = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (e < n) out[e] = in[idx[e]];
}
__global__ void fill_int_kernel(int* a, long long n, int v) {
  const long long e = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (e < n) a[e] = v;
}
// key = (internal row, degree-rank position of the column): inside a row the ratings are ordered by a
// quantity that does not depend on the sharding, so the fp32 summation order -- and hence every bit of the
// result -- is the same on 1, 2, 4 or 8 GPUs.
__global__ void make_keys_int_kernel(const int* rowext, const int* colext, long long n, const int* perm_row,
                                     const int* rpos_col, int bits_col, uint64_t* keys, uint32_t* pay) {
  const long long e = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (e < n) {
    keys[e] = ((uint64_t)(uint32_t)perm_row[rowext[e]] << bits_col) | (uint64_t)(uint32_t)rpos_col[colext[e]];
    pay[e] = (uint32_t)e;
  }
}
__global__ void build_ptr_kernel(const uint64_t* keys, long long n, int bits_col, int n_rows, long long* ptr) {
  const long long e = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (e >= n) return;
  const int r = (int)(keys[e] >> bits_col);
  const int rp = e == 0 ? -1 : (int)(keys[e - 1] >> bits_col);
  for (int rr = rp + 1; rr <= r; ++rr) ptr[rr] = e;
  if (e == n - 1)
    for (int rr = r + 1; rr <= n_rows; ++rr) ptr[rr] = n;
}
__global__ void extract_csr_kernel(const uint64_t* keys, const uint32_t* pay, const float* rating, long long b,
                                   long long cnt, int bits_col, const int* p2i_col, int* idx, float* val) {
  const long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= cnt) return;
  idx[t] = p2i_col[(int)(keys[b + t] & ((1ull << bits_col) - 1ull))];
  val[t] = rating[pay[b + t]];
}
__global__ void local_rows_kernel(const long long* ptr_full, int row0, int R, long long base, const int* inv,
                                  const uint32_t* deg, const uint32_t* npos, int implicit, long long* ptr,
                                  float* nreg, int* counts /* [0]=active [1]=heavy */, int heavy_t) {
  const int r = blockIdx.x * blockDim.x + threadIdx.x;
  if (r > R) return;
  ptr[r] = ptr_full[row0 + r] - base;
  if (r == R) return;
  const int ext = inv[row0 + r];
  float nr = 0.f;
  if (ext >= 0) {
    const uint32_t d = deg[ext];
    nr = implicit ? (float)npos[ext] : (float)d;
    if (d > 0) atomicAdd(&counts[0], 1);
    if (d > (uint32_t)heavy_t) atomicAdd(&counts[1], 1);
  }
  nreg[r] = nr;
}
__global__ void scatter_init_kernel(const float* ext_f, int n, int k, int kp, const int* perm, const uint32_t* deg,
                                    float* F) {
  const long long o = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (o >= (long long)n * kp) return;
  const int r = (int)(o / kp), c = (int)(o % kp);
  float v = 0.f;
  if (c < k && deg[r] > 0) v = ext_f[(size_t)r * k + c];
  F[(size_t)perm[r] * kp + c] = v;
}
__device__ __forceinline__ uint64_t splitmix64_dev(uint64_t x) {
  x += 0x9E3779B97F4A7C15ull;
  uint64_t z = x;
  z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9ull;
  z = (z ^ (z >> 27)) * 0x94D049BB133111EBull;
  return z ^ (z >> 31);
}
// unit-norm Gaussian rows from the counter hash (mirrors synth.py synth_init_factors)
__global__ void hash_init_kernel(int n, int k, int kp, uint64_t seed, int side, const int* perm,
                                 const uint32_t* deg, float* F) {
  const int r = blockIdx.x * blockDim.x + threadIdx.x;
  if (r >= n) return;
  float* row = F + (size_t)perm[r] * kp;
  if (deg[r] == 0) {
    for (int c = 0; c < kp; ++c) row[c] = 0.f;
    return;
  }
  const uint64_t s = seed ^ 0xA5A5A5A55A5A5A5Aull;
  double nrm = 0.0;
  for (int c = 0; c < k; ++c) {
    const uint64_t ctr = ((uint64_t)r * (uint64_t)k + (uint64_t)c) * 2ull + ((uint64_t)side << 62);
    const uint64_t h1 = splitmix64_dev(s ^ ctr), h2 = splitmix64_dev(s ^ (ctr + 1ull));
    const double u1 = ((double)(h1 >> 11) + 1.0) * (1.0 / 9007199254740992.0);
    const double u2 = (double)(h2 >> 11) * (1.0 / 9007199254740992.0);
    const float g = (float)(sqrt(-2.0 * log(u1)) * cos(2.0 * 3.14159265358979323846 * u2));
    row[c] = g;
    nrm += (double)g * (double)g;
  }
  float nf = (float)sqrt(nrm);
  if (nf == 0.f) nf = 1.f;
  for (int c = 0; c < k; ++c) row[c] = row[c] / nf;
  for (int c = k; c < kp; ++c) row[c] = 0.f;
}
__global__ void gather_factors_kernel(const float* F, int n, int k, int kp, const int* perm, float* out) {
  const long long o = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (o >= (long long)n * k) return;
  const int r = (int)(o / k), c = (int)(o % k);
  out[o] = F[(size_t)perm[r] * kp + c];
}
__global__ void has_kernel(const uint32_t* deg, int n, uint8_t* has) {
  const int r = blockIdx.x * blockDim.x + threadIdx.x;
  if (r < n) has[r] = deg[r] > 0 ? 1 : 0;
}
// internal row -> external id if the row owns a factor, else -1 (candidate table for top-k)
__global__ void cand_ext_kernel(const int* inv, const uint32_t* deg, int n_internal, int* out) {
  const int r = blockIdx.x * blockDim.x + threadIdx.x;
  if (r >= n_internal) return;
  const int ext = inv[r];
  out[r] = (ext >= 0 && deg[ext] > 0) ? ext : -1;
}
__global__ void gather_rows_kernel(const float* F, int kp, const int* rows_ext, int n, const int* perm,
                                   const uint32_t* deg, int n_ext, float* out, uint8_t* valid) {
  const int q = blockIdx.x;
  const int r = rows_ext[q];
  const bool ok = r >= 0 && r < n_ext && deg[r] > 0;
  for (int c = threadIdx.x; c < kp; c += blockDim.x) out[(size_t)q * kp + c] = ok ? F[(size_t)perm[r] * kp + c] : 0.f;
  if (threadIdx.x == 0 && valid) valid[q] = ok ? 1 : 0;
  (void)n;
}
// low-latency serving: the (few) row ids travel in the kernel parameters, no host-to-device copy
struct IdList {
  int v[40];
};
__global__ void gather_rows_ids_kernel(const float* F, int kp, IdList ids, const int* perm, const uint32_t* deg, int n_ext,
                                       float* out, uint8_t* valid) {
  const int q = blockIdx.x;
  const int r = ids.v[q];
  const bool ok = r >= 0 && r < n_ext && deg[r] > 0;
  for (int c = threadIdx.x; c < kp; c += blockDim.x) out[(size_t)q * kp + c] = ok ? F[(size_t)perm[r] * kp + c] : 0.f;
  if (threadIdx.x == 0 && valid) valid[q] = ok ? 1 : 0;
}
__global__ void copy_rows_kernel(const float* src, int kp, const int* rows, float* out) {
  const int v = blockIdx.x;
  for (int c = threadIdx.x; c < kp; c += blockDim.x) out[(size_t)v * kp + c] = src[(size_t)rows[v] * kp + c];
}
__global__ void synth_kernel(int nu, int ni, long long n, uint64_t seed, int implicit, long long start, int* u,
                             int* it, float* r) {
  const long long e = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (e >= n) return;
  const uint64_t base = (uint64_t)(start + e) * 4ull;
  const uint64_t h1 = splitmix64_dev(seed ^ (base + 1ull));
  const uint64_t h2 = splitmix64_dev(seed ^ (base + 2ull));
  const uint64_t h3 = splitmix64_dev(seed ^ (base + 3ull));
  u[e] = (int)(h1 % (uint64_t)nu);
  const double uu = (double)(h2 >> 11) * (1.0 / 9007199254740992.0);
  long long item = (long long)floor(__dmul_rn(__dmul_rn((double)ni, uu), uu));
  if (item > ni - 1) item = ni - 1;
  it[e] = (int)item;
  if (implicit) {
    int tz = h3 == 0 ? 64 : __ffsll((long long)h3) - 1;
    if (tz > 9) tz = 9;
    r[e] = (float)(1 + tz);
  } else {
    r[e] = (float)(1 + (int)(h3 % 5ull));
  }
}

// ---------------------------------------------------------------------------------------------
// handle
// ---------------------------------------------------------------------------------------------
struct Side {
  int n = 0;           // external rows
  int R = 0;           // rows owned per rank
  int n_internal = 0;  // world * R
  int bits = 1;        // bits of an internal id
  int* perm = nullptr;       // [n] external row -> internal id
  int* inv = nullptr;        // [n_internal]
  int* rpos = nullptr;       // [n] external row -> degree-rank position
  int* p2i = nullptr;        // [n] degree-rank position -> internal id
  uint32_t* deg = nullptr;   // [n]
  uint32_t* npos = nullptr;  // [n]
  long long* ptr = nullptr;  // [R+1]
  int* idx = nullptr;
  float* val = nullptr;
  long long nnz_local = 0;
  float* nreg = nullptr;     // [R]
  float* F = nullptr;        // [n_internal][KP]
  int* cand_ext = nullptr;   // [n_internal]
  int n_active = 0, n_heavy = 0;
  SidePlan plan;             // kernel, heavy-row threshold and part length of this side (solve_plan.h)
  // parts of the n_heavy longest local rows
  long long* part_beg = nullptr;
  long long* part_end = nullptr;
  int* row_part_ptr = nullptr;   // [n_heavy + 1]
  float* partial = nullptr;      // [n_parts][SLOT + KP]
  int n_parts = 0;
  std::vector<int> h_row_part_ptr;   // host copy (rank 65..128 walks its rows in tiles)
};

enum EvKind { EV_SOLVE = 0, EV_GRAM = 1, EV_COMM = 2, EV_SOLVE_USER = 3, EV_NKIND = 4 };   // EV_SOLVE = item half-step
struct EvPair {
  cudaEvent_t a, b;
  int kind;
};

}  // namespace pio

using namespace pio;

struct pio_als_handle {
  pio_als_config cfg;
  int KP = 0;
  cudaStream_t stream = nullptr;
  Side U, I;
  float* yty = nullptr;
  double* gram_partial = nullptr;
  double* gram_gsum = nullptr;   // [GRAM_GROUPS][KP*KP] class sums of the YtY partials (slot order, GramMap)
  const Side* gram_side = nullptr;   // the side whose YtY currently sits in `yty` (nullptr: none / stale)
  cudaEvent_t ev_gram = nullptr;
  int gram_blocks = 0;
  int* d_fail = nullptr;
  int* d_counts = nullptr;
  // pair kernel FP16 split scale: [0] max |source factors| of the current half-step, [1] max |rating| (ingest); float bits
  unsigned* d_absmax = nullptr;
  long long* d_timing = nullptr;  // PIO_ALS_TC_TIMING=1: per-warp cycle counters of the last tensor-core launch
  float* d_dbg = nullptr;     // PIO_ALS_TC_DEBUG=1: A/b dump of the last tensor-core half-step
  size_t dbg_rows = 0;
  SolveSwitches sw;           // the solve's environment switches (solve_plan.h)
  // half-step pipeline (pair-kernel sides): long rows (parts + finish) run on `aux` next to the whole rows on `stream`;
  // the destination rows are cut into sw.n_pieces local ranges and the all-gather of a finished range runs on
  // `comm_st` while the next range is solved (world_size > 1)
  cudaStream_t aux = nullptr, comm_st = nullptr;
  cudaEvent_t ev_start = nullptr, ev_heavy = nullptr, ev_piece[8] = {}, ev_comm = nullptr;
  bool pieces_done = false;   // the last launch_solve recorded ev_piece[] / ev_heavy (pair path)
  // low-latency serving (few queries, topk <= 128): a persistent device arena and a mapped pinned host arena -- no
  // allocation, no staging copies, results written by the merge kernel straight into host memory
  bool trace_on = false;      // PIO_ALS_INGEST_TRACE
  std::chrono::steady_clock::time_point t_prev;
  unsigned char* srv_dev = nullptr;
  size_t srv_dev_cap = 0;
  unsigned char* srv_host = nullptr;       // cudaHostAlloc(mapped)
  unsigned char* srv_host_dev = nullptr;   // its device address
  size_t srv_host_cap = 0;
  unsigned* srv_counter = nullptr;         // arrival counter of score_one_kernel (zero between calls)
  unsigned srv_seq = 0;                    // sequence number of the last fused single-query call
  bool serve_fused = true;                 // PIO_ALS_SERVE_FUSED=0: single queries take the three-launch path
  bool score_blocked = true;               // PIO_ALS_SCORE_BLOCKED=0: batched recommend on the one-item-per-thread kernel
  bool serve_trace = false;                // PIO_ALS_SERVE_TRACE=1: per-phase device timestamps of every fused call on stderr
  float* tc_out = nullptr;    // wgmma split mode: normal equations of one tile of rows ([rows][ASLOT + KP])
  size_t tc_out_rows = 0;
  bool have_ratings = false, have_init = false, trained = false;
  ncclComm_t comm = nullptr;
  std::string err;
  pio_als_stats st{};
  double phase_ms[8] = {0, 0, 0, 0, 0, 0, 0, 0};  // pio_als_get_phase_ms
  std::deque<EvPair> ev_pool;  // deque: references stay valid while the pool grows
  size_t ev_used = 0;
  std::mutex mu;
  int sm_count = 0;
};

namespace pio {

static int fail(pio_als_handle* h, int code, const char* fmt, ...) {
  char buf[512];
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(buf, sizeof buf, fmt, ap);
  va_end(ap);
  if (h) h->err = buf;
  else g_create_error = buf;
  return code;
}
// PIO_ALS_INGEST_TRACE=1: wall-clock milliseconds per ingest phase (stream drained at every mark) on stderr
static void tmark(pio_als_handle* h, const char* what) {
  if (!h->trace_on) return;
  cudaStreamSynchronize(h->stream);
  const auto now = std::chrono::steady_clock::now();
  fprintf(stderr, "[pio_als ingest r%d] %-34s %8.3f ms\n", h->cfg.world_rank, what,
          std::chrono::duration<double, std::milli>(now - h->t_prev).count());
  h->t_prev = now;
}
#define CK(h, call)                                                                              \
  do {                                                                                           \
    cudaError_t e_ = (call);                                                                     \
    if (e_ != cudaSuccess)                                                                       \
      return fail(h, PIO_ALS_ERR_CUDA, "%s failed: %s (%s:%d)", #call, cudaGetErrorString(e_), \
                  __FILE__, __LINE__);                                                           \
  } while (0)
#define LAUNCHED(h) (++(h)->st.kernel_launches)

static inline unsigned nblk(long long n, int t) { return (unsigned)((n + t - 1) / t); }

template <class T>
static cudaError_t dalloc(pio_als_handle* h, T** p, size_t n) {
  return cudaMallocAsync((void**)p, (n ? n : 1) * sizeof(T), h->stream);
}
template <class T>
static void dfree(pio_als_handle* h, T*& p) {
  if (p) cudaFreeAsync((void*)p, h->stream);
  p = nullptr;
}

// Device temporaries of one API call: released (stream-ordered) on every exit path, including the early error returns
// of CK().
struct Scratch {
  pio_als_handle* h;
  std::vector<void*> ptrs;
  explicit Scratch(pio_als_handle* h_) : h(h_) {}
  Scratch(const Scratch&) = delete;
  Scratch& operator=(const Scratch&) = delete;
  template <class T>
  cudaError_t alloc(T** p, size_t n) {
    const cudaError_t e = dalloc(h, p, n);
    if (e == cudaSuccess) ptrs.push_back((void*)*p);
    return e;
  }
  ~Scratch() {
    for (void* q : ptrs) cudaFreeAsync(q, h->stream);
  }
};

static void free_side(pio_als_handle* h, Side& s, bool keep_factors) {
  dfree(h, s.perm); dfree(h, s.inv); dfree(h, s.rpos); dfree(h, s.p2i); dfree(h, s.deg); dfree(h, s.npos); dfree(h, s.ptr);
  dfree(h, s.idx); dfree(h, s.val); dfree(h, s.nreg); dfree(h, s.cand_ext);
  dfree(h, s.part_beg); dfree(h, s.part_end); dfree(h, s.row_part_ptr); dfree(h, s.partial);
  s.n_parts = 0;
  s.h_row_part_ptr.clear();
  if (!keep_factors) dfree(h, s.F);
}

static EvPair& next_ev(pio_als_handle* h, int kind) {
  if (h->ev_used == h->ev_pool.size()) {
    EvPair p;
    cudaEventCreate(&p.a);
    cudaEventCreate(&p.b);
    p.kind = kind;
    h->ev_pool.push_back(p);
  }
  EvPair& p = h->ev_pool[h->ev_used++];
  p.kind = kind;
  return p;
}

// ---- ingest ---------------------------------------------------------------------------------
static int build_side(pio_als_handle* h, Side& row, const Side& col, const int* rowext, const int* colext,
                      const float* rating, long long nnz, long long nnz_global) {
  // nnz ratings are present on this rank (all of them in replicated mode, those of the rows it owns in sharded mode);
  // nnz_global = ratings after dedup over all ranks (kernel choice must agree on every rank)
  cudaStream_t st = h->stream;
  const int W = h->cfg.world_size, rk = h->cfg.world_rank;
  Scratch tmp(h);
  uint64_t *ka = nullptr, *kb = nullptr;
  uint32_t *va = nullptr, *vb = nullptr;
  CK(h, tmp.alloc(&ka, (size_t)nnz));
  CK(h, tmp.alloc(&kb, (size_t)nnz));
  CK(h, tmp.alloc(&va, (size_t)nnz));
  CK(h, tmp.alloc(&vb, (size_t)nnz));
  bool in_b = false;
  if (nnz > 0) {
    make_keys_int_kernel<<<nblk(nnz, 256), 256, 0, st>>>(rowext, colext, nnz, row.perm, col.rpos, col.bits, ka, va);
    LAUNCHED(h);
    CK(h, radix_sort_pairs(ka, va, kb, vb, (size_t)nnz, row.bits + col.bits, st, &in_b, &h->st.kernel_launches));
  }
  tmark(h, "  side: keys + radix sort");
  const uint64_t* ks = in_b ? kb : ka;
  const uint32_t* vs = in_b ? vb : va;
  long long* ptr_full = nullptr;
  CK(h, tmp.alloc(&ptr_full, (size_t)row.n_internal + 1));
  CK(h, cudaMemsetAsync(ptr_full, 0, sizeof(long long) * ((size_t)row.n_internal + 1), st));
  if (nnz > 0) {
    build_ptr_kernel<<<nblk(nnz, 256), 256, 0, st>>>(ks, nnz, col.bits, row.n_internal, ptr_full);
    LAUNCHED(h);
  }
  long long be[2];
  CK(h, cudaMemcpyAsync(&be[0], ptr_full + (size_t)rk * row.R, sizeof(long long), cudaMemcpyDeviceToHost, st));
  CK(h, cudaMemcpyAsync(&be[1], ptr_full + (size_t)(rk + 1) * row.R, sizeof(long long), cudaMemcpyDeviceToHost, st));
  CK(h, cudaStreamSynchronize(st));
  row.nnz_local = be[1] - be[0];
  if (row.nnz_local >= (1ll << 31))
    return fail(h, PIO_ALS_ERR_ARG, "more than 2^31-1 ratings on one GPU (%lld); use more GPUs", row.nnz_local);
  CK(h, dalloc(h, &row.idx, (size_t)row.nnz_local));
  CK(h, dalloc(h, &row.val, (size_t)row.nnz_local));
  CK(h, dalloc(h, &row.ptr, (size_t)row.R + 1));
  CK(h, dalloc(h, &row.nreg, (size_t)row.R));
  if (row.nnz_local > 0) {
    extract_csr_kernel<<<nblk(row.nnz_local, 256), 256, 0, st>>>(ks, vs, rating, be[0], row.nnz_local, col.bits,
                                                                 col.p2i, row.idx, row.val);
    LAUNCHED(h);
  }
  tmark(h, "  side: ptr + extract csr");
  CK(h, cudaMemsetAsync(h->d_counts, 0, 2 * sizeof(int), st));
  row.plan = plan_side(h->sw, h->KP, row.n, nnz_global);
  local_rows_kernel<<<nblk(row.R + 1, 256), 256, 0, st>>>(ptr_full, rk * row.R, row.R, be[0], row.inv, row.deg,
                                                           row.npos, h->cfg.implicit_prefs, row.ptr, row.nreg,
                                                           h->d_counts, row.plan.heavy_t);
  LAUNCHED(h);
  int counts[2];
  CK(h, cudaMemcpyAsync(counts, h->d_counts, sizeof counts, cudaMemcpyDeviceToHost, st));
  CK(h, cudaStreamSynchronize(st));
  row.n_active = counts[0];
  row.n_heavy = counts[1];
  tmark(h, "  side: local rows");
  if (row.n_heavy > 0) {
    // cut the heavy rows (local rows [0, n_heavy), longest first) into parts of part_len ratings
    std::vector<long long> hp((size_t)row.n_heavy + 1);
    CK(h, cudaMemcpyAsync(hp.data(), row.ptr, sizeof(long long) * hp.size(), cudaMemcpyDeviceToHost, st));
    CK(h, cudaStreamSynchronize(st));
    std::vector<long long> pb, pe;
    std::vector<int> rpp((size_t)row.n_heavy + 1);
    const int part_len = row.plan.part_len;
    for (int r = 0; r < row.n_heavy; ++r) {
      rpp[r] = (int)pb.size();
      for (long long b = hp[r]; b < hp[r + 1]; b += part_len) {
        pb.push_back(b);
        pe.push_back(b + part_len < hp[r + 1] ? b + part_len : hp[r + 1]);
      }
    }
    rpp[row.n_heavy] = (int)pb.size();
    row.n_parts = (int)pb.size();
    row.h_row_part_ptr = rpp;
    tmark(h, "  side: parts of long rows");
    CK(h, dalloc(h, &row.part_beg, pb.size()));
    CK(h, dalloc(h, &row.part_end, pe.size()));
    CK(h, dalloc(h, &row.row_part_ptr, rpp.size()));
    CK(h, cudaMemcpyAsync(row.part_beg, pb.data(), sizeof(long long) * pb.size(), cudaMemcpyHostToDevice, st));
    CK(h, cudaMemcpyAsync(row.part_end, pe.data(), sizeof(long long) * pe.size(), cudaMemcpyHostToDevice, st));
    CK(h, cudaMemcpyAsync(row.row_part_ptr, rpp.data(), sizeof(int) * rpp.size(), cudaMemcpyHostToDevice, st));
    CK(h, cudaStreamSynchronize(st));
  }
  (void)W;
  return PIO_ALS_OK;
}

static int rank_rows(pio_als_handle* h, Side& s) {
  cudaStream_t st = h->stream;
  Scratch tmp(h);
  uint64_t *ka = nullptr, *kb = nullptr;
  uint32_t *va = nullptr, *vb = nullptr;
  CK(h, tmp.alloc(&ka, (size_t)s.n));
  CK(h, tmp.alloc(&kb, (size_t)s.n));
  CK(h, tmp.alloc(&va, (size_t)s.n));
  CK(h, tmp.alloc(&vb, (size_t)s.n));
  degree_keys_kernel<<<nblk(s.n, 256), 256, 0, st>>>(s.deg, s.n, ka, va);
  LAUNCHED(h);
  bool in_b = false;
  CK(h, radix_sort_pairs(ka, va, kb, vb, (size_t)s.n, 32, st, &in_b, &h->st.kernel_launches));
  fill_int_kernel<<<nblk(s.n_internal, 256), 256, 0, st>>>(s.inv, s.n_internal, -1);
  LAUNCHED(h);
  assign_internal_kernel<<<nblk(s.n, 256), 256, 0, st>>>(in_b ? vb : va, s.n, h->cfg.world_size, s.R, s.perm, s.inv,
                                                         s.rpos, s.p2i);
  LAUNCHED(h);
  return PIO_ALS_OK;
}

// ---- sharded ingest: all-to-all exchange of event arrays ------------------------------------------------------------
// The n events on this rank go to the ranks named by the sort keys (destination rank, payload = event index; built by the
// caller in ka/va).  Events keep their order per destination and arrive concatenated in source-rank order, so a global
// event order (rank r's slice precedes rank r + 1's) survives.  The received arrays are allocated in `keep`.
struct XArr {
  const void* in;
  void** out;
  size_t elem;
};
static int exchange_events(pio_als_handle* h, Scratch& keep, uint64_t* ka, uint32_t* va, uint64_t* kb, uint32_t* vb,
                           long long n, XArr* arrs, int na, long long* n_out) {
  cudaStream_t st = h->stream;
  NcclApi& nc = nccl_api();
  const int W = h->cfg.world_size, me = h->cfg.world_rank;
  Scratch tmp(h);
  bool in_b = false;
  if (n > 0) CK(h, radix_sort_pairs(ka, va, kb, vb, (size_t)n, ceil_log2((uint64_t)W), st, &in_b, &h->st.kernel_launches));
  const uint64_t* ks = in_b ? kb : ka;
  const uint32_t* vs = in_b ? vb : va;
  long long *d_off = nullptr, *d_cnt = nullptr, *d_all = nullptr;
  CK(h, tmp.alloc(&d_off, (size_t)W + 1));
  CK(h, tmp.alloc(&d_cnt, (size_t)W));
  CK(h, tmp.alloc(&d_all, (size_t)W * W));
  CK(h, cudaMemsetAsync(d_off, 0, sizeof(long long) * (W + 1), st));
  if (n > 0) {
    build_ptr_kernel<<<nblk(n, 256), 256, 0, st>>>(ks, n, 0, W, d_off);
    LAUNCHED(h);
  }
  std::vector<long long> off(W + 1), all((size_t)W * W);
  CK(h, cudaMemcpyAsync(off.data(), d_off, sizeof(long long) * (W + 1), cudaMemcpyDeviceToHost, st));
  CK(h, cudaStreamSynchronize(st));
  std::vector<long long> cnt(W);
  for (int p = 0; p < W; ++p) cnt[p] = off[p + 1] - off[p];
  CK(h, cudaMemcpyAsync(d_cnt, cnt.data(), sizeof(long long) * W, cudaMemcpyHostToDevice, st));
  if (nc.AllGather(d_cnt, d_all, (size_t)W, ncclInt64, h->comm, st) != ncclSuccess)
    return fail(h, PIO_ALS_ERR_COMM, "ncclAllGather (exchange counts) failed");
  CK(h, cudaMemcpyAsync(all.data(), d_all, sizeof(long long) * W * W, cudaMemcpyDeviceToHost, st));
  CK(h, cudaStreamSynchronize(st));
  tmark(h, "  exchange: sort by rank + counts");
  std::vector<long long> roff(W + 1, 0);
  for (int src = 0; src < W; ++src) roff[src + 1] = roff[src] + all[(size_t)src * W + me];
  const long long nrecv = roff[W];
  if (nrecv >= (1ll << 32)) return fail(h, PIO_ALS_ERR_ARG, "more than 2^32-1 events on one rank after the exchange");
  // gather every array into destination order, then ONE grouped send/recv for all arrays and peers
  std::vector<unsigned char*> sendbufs(na, nullptr), recvbufs(na, nullptr);
  for (int a = 0; a < na; ++a) {
    if (!arrs[a].in) { *arrs[a].out = nullptr; continue; }
    CK(h, tmp.alloc(&sendbufs[a], (size_t)(n > 0 ? n : 1) * arrs[a].elem));
    CK(h, keep.alloc(&recvbufs[a], (size_t)(nrecv > 0 ? nrecv : 1) * arrs[a].elem));
    if (n > 0) {
      if (arrs[a].elem == 4)
        gather_by_index_kernel<uint32_t><<<nblk(n, 256), 256, 0, st>>>((const uint32_t*)arrs[a].in, vs, n, (uint32_t*)sendbufs[a]);
      else
        gather_by_index_kernel<uint64_t><<<nblk(n, 256), 256, 0, st>>>((const uint64_t*)arrs[a].in, vs, n, (uint64_t*)sendbufs[a]);
      LAUNCHED(h);
    }
    *arrs[a].out = recvbufs[a];
  }
  if (nc.GroupStart() != ncclSuccess) return fail(h, PIO_ALS_ERR_COMM, "ncclGroupStart failed");
  for (int a = 0; a < na; ++a) {
    if (!arrs[a].in) continue;
    for (int p = 0; p < W; ++p) {
      const long long sc = cnt[p], rc_ = all[(size_t)p * W + me];
      if (sc > 0 && nc.Send(sendbufs[a] + (size_t)off[p] * arrs[a].elem, (size_t)sc * arrs[a].elem, ncclInt8, p, h->comm, st) != ncclSuccess)
        return fail(h, PIO_ALS_ERR_COMM, "ncclSend failed");
      if (rc_ > 0 && nc.Recv(recvbufs[a] + (size_t)roff[p] * arrs[a].elem, (size_t)rc_ * arrs[a].elem, ncclInt8, p, h->comm, st) != ncclSuccess)
        return fail(h, PIO_ALS_ERR_COMM, "ncclRecv failed");
    }
  }
  if (nc.GroupEnd() != ncclSuccess) return fail(h, PIO_ALS_ERR_COMM, "ncclGroupEnd failed");
  CK(h, cudaStreamSynchronize(st));
  tmark(h, "  exchange: gather + send/recv");
  *n_out = nrecv;
  return PIO_ALS_OK;
}

// sharded == false: the arrays hold ALL events (every rank passes the same COO and keeps the rows it owns).
// sharded == true (world_size > 1): the arrays hold this rank's slice of the events; ratings are routed to the owners of
// their user row and of their item row by NCCL send/recv, degrees are all-reduced; no rank ever holds the full COO.
static int ingest_device(pio_als_handle* h, const int* d_user, const int* d_item, const float* d_rating,
                         long long nnz, int dedup, const long long* d_ts, bool sharded) {
  cudaStream_t st = h->stream;
  const int W = h->cfg.world_size;
  sharded = sharded && W > 1;
  if (nnz <= 0 && !sharded)
    return fail(h, PIO_ALS_ERR_ARG, "ratings cannot be empty (the templates require(!ratings.take(1).isEmpty))");
  if (nnz < 0) return fail(h, PIO_ALS_ERR_ARG, "nnz < 0");
  if (nnz >= (1ll << 32)) return fail(h, PIO_ALS_ERR_ARG, "nnz must be < 2^32 per call");
  if (dedup < 0 || dedup > 2) return fail(h, PIO_ALS_ERR_ARG, "bad dedup_mode %d", dedup);
  free_side(h, h->U, true);
  free_side(h, h->I, true);
  h->have_ratings = false;
  Side& U = h->U;
  Side& I = h->I;
  U.n = h->cfg.n_users;
  I.n = h->cfg.n_items;
  U.R = (U.n + W - 1) / W;
  I.R = (I.n + W - 1) / W;
  U.n_internal = U.R * W;
  I.n_internal = I.R * W;
  U.bits = ceil_log2((uint64_t)U.n_internal);
  I.bits = ceil_log2((uint64_t)I.n_internal);

  h->trace_on = getenv("PIO_ALS_INGEST_TRACE") != nullptr;
  h->t_prev = std::chrono::steady_clock::now();
  auto mark = [&](const char* what) { tmark(h, what); };
  CK(h, cudaMemsetAsync(h->d_fail, 0, sizeof(int), st));
  if (nnz > 0) {
    validate_coo_kernel<<<nblk(nnz, 256), 256, 0, st>>>(d_user, d_item, nnz, U.n, I.n, h->d_fail);
    LAUNCHED(h);
  }
  int bad = 0;
  CK(h, cudaMemcpyAsync(&bad, h->d_fail, sizeof(int), cudaMemcpyDeviceToHost, st));
  CK(h, cudaStreamSynchronize(st));
  if (bad) return fail(h, PIO_ALS_ERR_ARG, "%d ratings have a user/item index out of range", bad);

  mark("validate");
  Scratch tmp(h);   // everything temporary: released on every exit path, including the CK() early returns
  // 0. sharded + dedup: first bring all events of a user to one rank (user mod W), keeping the event order
  const int* su = d_user;
  const int* si = d_item;
  const float* sr = d_rating;
  const long long* sts = d_ts;
  long long ns = nnz;
  if (sharded && dedup != PIO_ALS_DEDUP_NONE) {
    Scratch xs(h);
    uint64_t *ka = nullptr, *kb = nullptr;
    uint32_t *va = nullptr, *vb = nullptr;
    CK(h, xs.alloc(&ka, (size_t)nnz)); CK(h, xs.alloc(&kb, (size_t)nnz));
    CK(h, xs.alloc(&va, (size_t)nnz)); CK(h, xs.alloc(&vb, (size_t)nnz));
    if (nnz > 0) {
      dest_mod_kernel<<<nblk(nnz, 256), 256, 0, st>>>(d_user, nnz, W, ka, va);
      LAUNCHED(h);
    }
    void *xu = nullptr, *xi = nullptr, *xr = nullptr, *xt = nullptr;
    XArr arrs[4] = {{d_user, &xu, 4}, {d_item, &xi, 4}, {d_rating, &xr, 4},
                    {dedup == PIO_ALS_DEDUP_KEEP_LAST ? (const void*)d_ts : nullptr, &xt, 8}};
    int rc = exchange_events(h, tmp, ka, va, kb, vb, nnz, arrs, 4, &ns);
    if (rc) return rc;
    su = (const int*)xu; si = (const int*)xi; sr = (const float*)xr; sts = (const long long*)xt;
  }

  mark("exchange by user residue");
  // 1. optional dedup of repeated (user,item) pairs (all copies of a pair are on this rank)
  const int* cu = su;
  const int* ci = si;
  const float* cr = sr;
  long long n2 = ns;
  if (dedup != PIO_ALS_DEDUP_NONE && ns > 0) {
    Scratch ds(h);
    uint64_t *ka = nullptr, *kb = nullptr;
    uint32_t *va = nullptr, *vb = nullptr;
    CK(h, ds.alloc(&ka, (size_t)ns)); CK(h, ds.alloc(&kb, (size_t)ns));
    CK(h, ds.alloc(&va, (size_t)ns)); CK(h, ds.alloc(&vb, (size_t)ns));
    const int bu = ceil_log2((uint64_t)U.n), bi = ceil_log2((uint64_t)I.n);
    make_keys_ext_kernel<<<nblk(ns, 256), 256, 0, st>>>(su, si, ns, bi, ka, va);
    LAUNCHED(h);
    bool in_b = false;
    CK(h, radix_sort_pairs(ka, va, kb, vb, (size_t)ns, bu + bi, st, &in_b, &h->st.kernel_launches));
    const uint64_t* ks = in_b ? kb : ka;
    const uint32_t* vs = in_b ? vb : va;
    uint32_t* flag = nullptr;
    CK(h, ds.alloc(&flag, (size_t)ns));
    head_flags_kernel<<<nblk(ns, 256), 256, 0, st>>>(ks, ns, flag);
    LAUNCHED(h);
    uint32_t last_flag = 0, last_pos = 0;
    CK(h, cudaMemcpyAsync(&last_flag, flag + ns - 1, sizeof(uint32_t), cudaMemcpyDeviceToHost, st));
    CK(h, scan_exclusive_u32(flag, flag, (size_t)ns, st, &h->st.kernel_launches));
    CK(h, cudaMemcpyAsync(&last_pos, flag + ns - 1, sizeof(uint32_t), cudaMemcpyDeviceToHost, st));
    CK(h, cudaStreamSynchronize(st));
    n2 = (long long)last_pos + last_flag;
    int *du_ = nullptr, *di_ = nullptr;
    float* dr_ = nullptr;
    CK(h, tmp.alloc(&du_, (size_t)n2));
    CK(h, tmp.alloc(&di_, (size_t)n2));
    CK(h, tmp.alloc(&dr_, (size_t)n2));
    dedup_compact_kernel<<<nblk(ns, 256), 256, 0, st>>>(ks, vs, flag, ns, bi, sr, sts, dedup, du_, di_, dr_);
    LAUNCHED(h);
    cu = du_;
    ci = di_;
    cr = dr_;
  }

  mark("dedup");
  // 2. degrees, positive-rating counts (sharded: summed over the ranks)
  for (Side* s : {&U, &I}) {
    CK(h, dalloc(h, &s->deg, (size_t)s->n));
    CK(h, dalloc(h, &s->npos, (size_t)s->n));
    CK(h, dalloc(h, &s->perm, (size_t)s->n));
    CK(h, dalloc(h, &s->inv, (size_t)s->n_internal));
    CK(h, dalloc(h, &s->rpos, (size_t)s->n));
    CK(h, dalloc(h, &s->p2i, (size_t)s->n));
    CK(h, cudaMemsetAsync(s->deg, 0, sizeof(uint32_t) * s->n, st));
    CK(h, cudaMemsetAsync(s->npos, 0, sizeof(uint32_t) * s->n, st));
  }
  if (n2 > 0) {
    degree_kernel<<<nblk(n2, 256), 256, 0, st>>>(cu, ci, cr, n2, U.deg, I.deg, U.npos, I.npos);
    LAUNCHED(h);
  }
  // max |rating| (sharded: over all ranks): bounds sqrt(c1) in the pair kernel's FP16 split scale
  CK(h, cudaMemsetAsync(h->d_absmax + 1, 0, sizeof(unsigned), st));
  if (n2 > 0) {
    pr::abs_max_kernel<<<std::min(nblk(n2, 256), 4u * h->sm_count), 256, 0, st>>>(cr, n2, h->d_absmax + 1);
    LAUNCHED(h);
  }
  long long n2_global = n2;
  if (sharded) {
    NcclApi& nc = nccl_api();   // only multi-GPU jobs touch NCCL (a single-GPU process must not load libnccl at all)
    long long* d_n = nullptr;
    CK(h, tmp.alloc(&d_n, 1));
    CK(h, cudaMemcpyAsync(d_n, &n2, sizeof(long long), cudaMemcpyHostToDevice, st));
    if (nc.GroupStart() != ncclSuccess) return fail(h, PIO_ALS_ERR_COMM, "ncclGroupStart failed");   // one launch for the six
    for (Side* s : {&U, &I}) {
      if (nc.AllReduce(s->deg, s->deg, (size_t)s->n, ncclUint32, ncclSum, h->comm, st) != ncclSuccess ||
          nc.AllReduce(s->npos, s->npos, (size_t)s->n, ncclUint32, ncclSum, h->comm, st) != ncclSuccess)
        return fail(h, PIO_ALS_ERR_COMM, "ncclAllReduce (degrees) failed");
    }
    if (nc.AllReduce(d_n, d_n, 1, ncclInt64, ncclSum, h->comm, st) != ncclSuccess ||
        nc.AllReduce(h->d_absmax + 1, h->d_absmax + 1, 1, ncclUint32, ncclMax, h->comm, st) != ncclSuccess)
      return fail(h, PIO_ALS_ERR_COMM, "ncclAllReduce (nnz, rating maximum) failed");
    if (nc.GroupEnd() != ncclSuccess) return fail(h, PIO_ALS_ERR_COMM, "ncclGroupEnd failed");
    CK(h, cudaMemcpyAsync(&n2_global, d_n, sizeof(long long), cudaMemcpyDeviceToHost, st));
    CK(h, cudaStreamSynchronize(st));
    if (n2_global <= 0)
      return fail(h, PIO_ALS_ERR_ARG, "ratings cannot be empty (the templates require(!ratings.take(1).isEmpty))");
  }
  h->st.nnz = n2_global;

  mark("degrees (+ all-reduce)");
  // 3. renumber rows: degree-descending, dealt to ranks (the same on every rank)
  int rc = rank_rows(h, U);
  if (rc) return rc;
  rc = rank_rows(h, I);
  if (rc) return rc;

  mark("rank rows");
  // 4. the two CSR orientations in internal numbering (only this rank's rows are kept)
  if (!sharded) {
    rc = build_side(h, U, I, cu, ci, cr, n2, n2_global);
    if (rc) return rc;
    mark("build user side");
    rc = build_side(h, I, U, ci, cu, cr, n2, n2_global);
    if (rc) return rc;
    mark("build item side");
  } else {
    struct { Side* row; Side* col; const int* rowext; const int* colext; } jobs[2] = {{&U, &I, cu, ci}, {&I, &U, ci, cu}};
    for (auto& j : jobs) {
      Scratch xs(h), recv(h);
      uint64_t *ka = nullptr, *kb = nullptr;
      uint32_t *va = nullptr, *vb = nullptr;
      CK(h, xs.alloc(&ka, (size_t)n2)); CK(h, xs.alloc(&kb, (size_t)n2));
      CK(h, xs.alloc(&va, (size_t)n2)); CK(h, xs.alloc(&vb, (size_t)n2));
      if (n2 > 0) {
        dest_owner_kernel<<<nblk(n2, 256), 256, 0, st>>>(j.rowext, n2, j.row->perm, j.row->R, ka, va);
        LAUNCHED(h);
      }
      void *xrow = nullptr, *xcol = nullptr, *xr = nullptr;
      XArr arrs[3] = {{j.rowext, &xrow, 4}, {j.colext, &xcol, 4}, {cr, &xr, 4}};
      long long ne = 0;
      rc = exchange_events(h, recv, ka, va, kb, vb, n2, arrs, 3, &ne);
      if (rc) return rc;
      mark("exchange by row owner");
      rc = build_side(h, *j.row, *j.col, (const int*)xrow, (const int*)xcol, (const float*)xr, ne, n2_global);
      if (rc) return rc;
      mark("build side");
    }
  }

  // 5. factor matrices (zero: rows without ratings must stay zero) and candidate tables
  for (Side* s : {&U, &I}) {
    if (!s->F) {
      CK(h, dalloc(h, &s->F, (size_t)s->n_internal * h->KP));
      h->have_init = false;
    }
    CK(h, dalloc(h, &s->cand_ext, (size_t)s->n_internal));
    cand_ext_kernel<<<nblk(s->n_internal, 256), 256, 0, st>>>(s->inv, s->deg, s->n_internal, s->cand_ext);
    LAUNCHED(h);
  }
  h->have_init = false;
  CK(h, cudaStreamSynchronize(st));
  mark("factor buffers");
  h->st.n_users_active = U.n_active;
  h->st.n_items_active = I.n_active;
  if (W > 1) {
    // n_active per rank is local; the global counts are not needed by the library
    h->st.n_users_active = -1;
    h->st.n_items_active = -1;
  }
  h->have_ratings = true;
  h->trained = false;
  return PIO_ALS_OK;
}

static int init_hash(pio_als_handle* h) {
  cudaStream_t st = h->stream;
  CK(h, cudaMemsetAsync(h->U.F, 0, sizeof(float) * (size_t)h->U.n_internal * h->KP, st));
  CK(h, cudaMemsetAsync(h->I.F, 0, sizeof(float) * (size_t)h->I.n_internal * h->KP, st));
  hash_init_kernel<<<nblk(h->U.n, 128), 128, 0, st>>>(h->U.n, h->cfg.rank, h->KP, (uint64_t)h->cfg.seed, 0, h->U.perm,
                                                      h->U.deg, h->U.F);
  LAUNCHED(h);
  hash_init_kernel<<<nblk(h->I.n, 128), 128, 0, st>>>(h->I.n, h->cfg.rank, h->KP, (uint64_t)h->cfg.seed, 1, h->I.perm,
                                                      h->I.deg, h->I.F);
  LAUNCHED(h);
  h->have_init = true;
  return PIO_ALS_OK;
}

// ---- solve dispatch ---------------------------------------------------------------------------
// solve_plan.h decides which kernels a half-step runs and with what geometry; launch_solve_cfg executes that plan.
using Cfg16 = SolveCfg<16, 4, 25, 8>;
using Cfg32 = SolveCfg<32, 8, 25, 4>;
using Cfg64 = SolveCfg<64, 8, 7, 8>;
using Cfg128 = SolveCfg<128, 8, 2, 9>;

// the planner's copy of each kernel's launch geometry
static_assert(fp32_rows_per_cta(16) == Cfg16::NG && fp32_rows_per_cta(32) == Cfg32::NG &&
              fp32_rows_per_cta(64) == Cfg64::NG && fp32_rows_per_cta(128) == Cfg128::NG, "SolveCfg::NG");
static_assert(Cfg16::WARP_CHOL && Cfg32::WARP_CHOL && Cfg64::WARP_CHOL && Cfg128::LS_PARTIAL,
              "als_finish_kernel runs one warp per row below KP 128, and KP 128 takes the LS128 route");
static_assert(MMA_ROWS_PER_CTA == mm::WARPS, "mm::WARPS");
static_assert(TC_ROWS_PER_CTA == tc::Api::kPerCta && TC_SOLVE_ROWS_PER_CTA == tc::Api::kSolveWarps, "tc::Api");
static_assert(LS128_FINISH_ROWS_PER_CTA == FIN128_WARPS, "FIN128_WARPS");
// a part boundary never splits a chunk of any kernel or a wgmma stage; the pair part length stays a multiple of its chunk
static_assert(PART % Cfg16::CH == 0 && PART % Cfg32::CH == 0 && PART % Cfg64::CH == 0 && PART % Cfg128::CH == 0 &&
              PART % mm::CH == 0 && PART % tc::STAGE_RATINGS == 0, "PART");
static_assert(PAIR_PART % pr::CH == 0 && pr::CH == 8, "PAIR_PART and PIO_ALS_PART round to multiples of pr::CH");

// cudaFuncSetAttribute(MaxDynamicSharedMemorySize) SETS a kernel's limit on the current device, it does not raise it.  A
// kernel launched from several call sites therefore needs one record of the limit in place, shared by all handles and
// threads of the process: this one only ever raises it, per kernel and device.  carveout: also ask once for the
// largest shared-memory carveout.
static int ensure_dyn_smem(pio_als_handle* h, const void* kernel, size_t bytes, bool carveout = false) {
  struct Rec {
    size_t bytes = 0;
    bool carveout = false;
  };
  static std::mutex mu;
  static std::map<std::pair<const void*, int>, Rec> recs;
  std::lock_guard<std::mutex> lk(mu);
  Rec& r = recs[std::make_pair(kernel, h->cfg.device)];
  if (r.bytes < bytes) {
    CK(h, cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)bytes));
    r.bytes = bytes;
  }
  if (carveout && !r.carveout) {
    CK(h, cudaFuncSetAttribute(kernel, cudaFuncAttributePreferredSharedMemoryCarveout, 100));
    r.carveout = true;
  }
  return PIO_ALS_OK;
}

// Every launch of a half-step's solve goes through here: raise the kernel's dynamic shared-memory limit, launch on `st`,
// count the launch and fail on a launch error.
template <typename... KArgs, typename... Args>
static int solve_launch(pio_als_handle* h, void (*kernel)(KArgs...), int grid, int block, size_t smem, bool carveout,
                        cudaStream_t st, Args... args) {
  const int rc = ensure_dyn_smem(h, (const void*)kernel, smem, carveout);
  if (rc) return rc;
  kernel<<<grid, block, smem, st>>>(args...);
  LAUNCHED(h);
  ++h->st.solve_launches;
  CK(h, cudaGetLastError());
  return PIO_ALS_OK;
}

// the pair kernel with PIO_ALS_PAIR_WARPS warps per CTA
static void (*pair_kernel(int warps, bool imp))(const SolveParams, int) {
  switch (warps) {
    case 1: return imp ? pr::als_solve_pair_kernel<true, 1> : pr::als_solve_pair_kernel<false, 1>;
    case 2: return imp ? pr::als_solve_pair_kernel<true, 2> : pr::als_solve_pair_kernel<false, 2>;
    case 6: return imp ? pr::als_solve_pair_kernel<true, 6> : pr::als_solve_pair_kernel<false, 6>;
    case 12: return imp ? pr::als_solve_pair_kernel<true, 12> : pr::als_solve_pair_kernel<false, 12>;
    default: return imp ? pr::als_solve_pair_kernel<true, 4> : pr::als_solve_pair_kernel<false, 4>;
  }
}

// Buffers of the wgmma kernel, before its first launch of a half-step: the PIO_ALS_TC_TIMING / PIO_ALS_TC_DEBUG dumps
// and, in split mode (PIO_ALS_TC_SPLIT=1, off by default), the normal equations of one tile of rows, which a second
// kernel solves with every warp of the SM (the one-warp 64x64 Cholesky is latency-bound, so more solver warps per SM
// can help where the fused solves do not overlap the MMAs well).
static int tc_buffers(pio_als_handle* h, const Side& dst, tc::Api::Params* tp) {
  using A = tc::Api;
  tp->dbg = nullptr;
  tp->timing = nullptr;
  tp->out = nullptr;
  tp->out_row0 = 0;
  if (h->sw.tc_timing) {
    if (!h->d_timing) CK(h, cudaMalloc((void**)&h->d_timing, (size_t)h->sm_count * 16 * 8 * sizeof(long long)));
    cudaMemsetAsync(h->d_timing, 0, (size_t)h->sm_count * 16 * 8 * sizeof(long long), h->stream);
    tp->timing = h->d_timing;
  }
  if (h->sw.tc_debug) {
    if (h->dbg_rows < (size_t)dst.R) {
      if (h->d_dbg) cudaFree(h->d_dbg);
      CK(h, cudaMalloc((void**)&h->d_dbg, (size_t)dst.R * A::kRowFloats * sizeof(float)));
      h->dbg_rows = dst.R;
    }
    cudaMemsetAsync(h->d_dbg, 0, (size_t)dst.R * A::kRowFloats * sizeof(float), h->stream);
    tp->dbg = h->d_dbg;
  }
  if (h->sw.tc_split) {
    const int nlight = dst.n_active - dst.n_heavy;
    const size_t need = (size_t)(nlight < TC_TILE_ROWS ? nlight : TC_TILE_ROWS);
    if (h->tc_out_rows < need) {
      if (h->tc_out) cudaFree(h->tc_out);
      h->tc_out = nullptr;
      h->tc_out_rows = 0;
      CK(h, cudaMalloc((void**)&h->tc_out, need * A::kRowFloats * sizeof(float)));
      h->tc_out_rows = need;
    }
  }
  return PIO_ALS_OK;
}

template <class Cfg>
static int launch_solve_cfg(pio_als_handle* h, Side& dst, const Side& src) {
  SolveParams p0;
  p0.ptr = dst.ptr;
  p0.idx = dst.idx;
  p0.val = dst.val;
  p0.src = src.F;
  p0.dst = dst.F;
  p0.yty = h->yty;
  p0.nreg = dst.nreg;
  p0.fail = h->d_fail;
  p0.lambda = (float)h->cfg.lambda;
  p0.alpha = (float)h->cfg.alpha;
  p0.k = h->cfg.rank;
  p0.dst_row_offset = h->cfg.world_rank * dst.R;
  p0.absmax = h->d_absmax;
  p0.wl_beg = nullptr;
  p0.wl_end = nullptr;
  p0.partial = nullptr;
  p0.n_items = 0;
  const bool imp = h->cfg.implicit_prefs != 0;
  const SolvePlan plan = plan_half_step(h->sw, dst.plan, Cfg::KP, h->sm_count, dst.R, dst.n_active, dst.n_heavy,
                                        dst.n_parts, dst.h_row_part_ptr);
  const bool pair = dst.plan.kernel == SOLVE_PAIR;
  if (pair) cudaEventRecord(h->ev_start, h->stream);
  if (plan.partial_parts > 0 && !dst.partial) {
    const size_t floats = pair ? pr::PART_FLOATS : Cfg::PART_FLOATS;
    CK(h, cudaMallocAsync((void**)&dst.partial, sizeof(float) * (size_t)plan.partial_parts * floats, h->stream));
    if (pair) cudaEventRecord(h->ev_start, h->stream);
  }
  if (plan.n_aux > 0) cudaStreamWaitEvent(h->aux, h->ev_start, 0);
  // pair path: ev_heavy once the long rows are launched on aux, ev_piece[c] once the rows of piece c are launched (the
  // all-gather of a piece starts when its rows are done)
  size_t next_piece = 0;
  auto record_events = [&](int issued) {
    if (pair && issued == plan.n_aux) cudaEventRecord(h->ev_heavy, h->aux);
    for (; next_piece < plan.piece_after.size() && plan.piece_after[next_piece] == issued; ++next_piece)
      cudaEventRecord(h->ev_piece[next_piece], h->stream);
  };
  record_events(0);
  const int warps = h->sw.pair_warps;
  tc::Api::Params tp;
  bool tc_ready = false;
  for (size_t i = 0; i < plan.launches.size(); ++i) {
    const SolveLaunch& L = plan.launches[i];
    const cudaStream_t st = L.aux ? h->aux : h->stream;
    const int nrows = L.row_end - L.row_begin;
    SolveParams p = p0;
    if (L.stage == STAGE_ROWS || L.stage == STAGE_TC_SOLVE) {
      p.row_begin = L.row_begin;
      p.row_end = L.row_end;
    } else {   // work-list stages: parts [wl_off, wl_off + wl_count) of the heavy rows
      p.wl_beg = dst.part_beg + L.wl_off;
      p.wl_end = dst.part_end + L.wl_off;
      p.partial = dst.partial;
      p.n_items = L.wl_count;
      p.row_begin = 0;
      p.row_end = dst.n_heavy;
    }
    auto fp32 = [&] {
      return solve_launch(h, imp ? als_solve_kernel<Cfg, true> : als_solve_kernel<Cfg, false>, L.grid, Cfg::NT,
                          Cfg::smem_bytes(), false, st, p);
    };
    auto pair_items = [&](int n_items) {
      return solve_launch(h, pair_kernel(warps, imp), L.grid, 32 * warps, pr::smem_bytes(warps), true, st, p, n_items);
    };
    int rc = PIO_ALS_OK;
    switch (L.stage) {
      case STAGE_PARTS:
        rc = pair ? pair_items(L.wl_count) : fp32();
        break;
      case STAGE_FINISH:
        rc = pair ? solve_launch(h, imp ? pr::als_finish_pair_kernel<true> : pr::als_finish_pair_kernel<false>, L.grid,
                                 32, pr::smem_bytes(1), true, st, p, dst.row_part_ptr, nrows)
                  : solve_launch(h, imp ? als_finish_kernel<Cfg, true> : als_finish_kernel<Cfg, false>, L.grid,
                                 32 * FINISH_ROWS_PER_CTA, sizeof(float) * 4 * (Cfg::SLOT + 4 * Cfg::KP), false, st, p,
                                 dst.row_part_ptr, nrows);
        break;
      case STAGE_LS128_TILE:
        rc = fp32();
        break;
      case STAGE_LS128_FINISH:
        rc = solve_launch(h, imp ? als_finish_ls128_kernel<true> : als_finish_ls128_kernel<false>, L.grid,
                          32 * FIN128_WARPS, sizeof(float) * (size_t)FIN128_FLOATS * FIN128_WARPS, false, st, p,
                          dst.row_part_ptr, L.row_begin, nrows, L.wl_off);
        break;
      case STAGE_ROWS:
        switch (dst.plan.kernel) {
          case SOLVE_PAIR:
            rc = pair_items(nrows);
            break;
          case SOLVE_MMA:
            rc = solve_launch(h, imp ? mm::als_solve_mma_kernel<true> : mm::als_solve_mma_kernel<false>, L.grid, mm::NT,
                              mm::SMEM_BYTES, false, st, p);
            break;
          case SOLVE_WGMMA:
            if (!tc_ready) {
              rc = tc_buffers(h, dst, &tp);
              if (rc) return rc;
              tc_ready = true;
            }
            tp.sp = p;
            tp.out = h->sw.tc_split ? h->tc_out : nullptr;
            tp.out_row0 = L.row_begin;
            rc = solve_launch(h, tc::Api::kernel(imp), L.grid, tc::Api::kThreads, tc::Api::kSmem, false, st, tp);
            break;
          default:
            rc = fp32();
        }
        break;
      case STAGE_TC_SOLVE:
        rc = solve_launch(h, tc::Api::solver(imp), L.grid, 32 * tc::Api::kSolveWarps, tc::Api::kSolveSmem, false, st, p,
                          (const float*)h->tc_out, L.row_begin);
        break;
    }
    if (rc) return rc;
    record_events((int)i + 1);
  }
  if (pair) {
    cudaStreamWaitEvent(h->stream, h->ev_heavy, 0);   // the half-step ends when both streams are done
    h->pieces_done = true;
  }
  return PIO_ALS_OK;
}

static int launch_solve(pio_als_handle* h, Side& dst, const Side& src) {
  switch (h->KP) {
    case 16: return launch_solve_cfg<Cfg16>(h, dst, src);
    case 32: return launch_solve_cfg<Cfg32>(h, dst, src);
    case 64: return launch_solve_cfg<Cfg64>(h, dst, src);
    default: return launch_solve_cfg<Cfg128>(h, dst, src);
  }
}

// YtY (implicit feedback): als_kernels.cuh GramMap.  gram_sharded(): every rank owns whole classes (world size 2, 4, 8).
static bool gram_sharded(const pio_als_handle* h) { return h->cfg.world_size > 1 && GRAM_GROUPS % h->cfg.world_size == 0; }
static void gram_layout(const pio_als_handle* h, GramMap& m, int& my_groups, int& slot0) {
  const bool shard = gram_sharded(h);
  const int W = shard ? h->cfg.world_size : 1, me = shard ? h->cfg.world_rank : 0;
  my_groups = GRAM_GROUPS / W;
  slot0 = me * my_groups;
  int seen[GRAM_GROUPS] = {}, mine = 0;
  for (int g = 0; g < GRAM_GROUPS; ++g) {
    const int blk = g / W, pos = g % W;
    const int owner = (blk & 1) ? (W - 1 - pos) : pos;      // assign_internal_kernel's dealing, positions 0 .. 7
    m.slot_of[g] = owner * my_groups + seen[owner]++;
    if (owner == me) m.cls[mine++] = g;
  }
  for (int lg = mine; lg < GRAM_GROUPS; ++lg) m.cls[lg] = 0;
}
// phase A: block partials and slot sums of this rank's classes (sharded: from its own rows only)
static int gram_local(pio_als_handle* h, const Side& s) {
  GramMap m;
  int my_groups, slot0;
  gram_layout(h, m, my_groups, slot0);
  const int bpg = h->gram_blocks / GRAM_GROUPS, n = h->KP * h->KP, grid = my_groups * bpg;
  switch (h->KP) {
    case 16: gram_partial_kernel<16><<<grid, GRAM_THREADS, 0, h->stream>>>(s.F, s.p2i, s.n, h->gram_partial, slot0, bpg, m); break;
    case 32: gram_partial_kernel<32><<<grid, GRAM_THREADS, 0, h->stream>>>(s.F, s.p2i, s.n, h->gram_partial, slot0, bpg, m); break;
    case 64: gram_partial_kernel<64><<<grid, GRAM_THREADS, 0, h->stream>>>(s.F, s.p2i, s.n, h->gram_partial, slot0, bpg, m); break;
    default: gram_partial_kernel<128><<<grid, GRAM_THREADS, 0, h->stream>>>(s.F, s.p2i, s.n, h->gram_partial, slot0, bpg, m); break;
  }
  LAUNCHED(h);
  gram_group_kernel<<<dim3(nblk(n, 128), my_groups), 128, 0, h->stream>>>(h->gram_partial, bpg, n, slot0, h->gram_gsum);
  LAUNCHED(h);
  CK(h, cudaGetLastError());
  return PIO_ALS_OK;
}
// phase B: (sharded) all-gather of the slot sums on `comm_stream`, then the class sums in class order on the main stream
static int gram_exchange(pio_als_handle* h, cudaStream_t comm_stream) {
  if (!gram_sharded(h)) return PIO_ALS_OK;
  const int n = h->KP * h->KP, my_groups = GRAM_GROUPS / h->cfg.world_size;
  const size_t cnt = (size_t)my_groups * n;
  if (nccl_api().AllGather(h->gram_gsum + (size_t)h->cfg.world_rank * cnt, h->gram_gsum, cnt, ncclDouble, h->comm, comm_stream) !=
      ncclSuccess)
    return fail(h, PIO_ALS_ERR_COMM, "ncclAllGather (YtY class sums) failed");
  return PIO_ALS_OK;
}
static int gram_reduce(pio_als_handle* h, const Side& s) {
  GramMap m;
  int my_groups, slot0;
  gram_layout(h, m, my_groups, slot0);
  const int n = h->KP * h->KP;
  gram_reduce_kernel<<<nblk(n, 256), 256, 0, h->stream>>>(h->gram_gsum, n, h->yty, m);
  LAUNCHED(h);
  CK(h, cudaGetLastError());
  h->gram_side = &s;
  return PIO_ALS_OK;
}

// One half-iteration: dst := argmin given src.  `more` = another half-step follows in this run: then YtY of the fresh dst
// factors is prepared here -- on 2 / 4 / 8 GPUs from the rank's own rows while the last pieces of the factor all-gather
// are still in flight, its 8 x KP^2 doubles exchanged on the communication stream right behind them.
static int half_step(pio_als_handle* h, Side& dst, const Side& src, bool more) {
  cudaStream_t st = h->stream;
  const bool implicit = h->cfg.implicit_prefs != 0;
  if (implicit && h->gram_side != &src) {     // first half-step of a run, or the factors were set from outside
    const EvPair e = next_ev(h, EV_GRAM);
    cudaEventRecord(e.a, st);
    int grc = gram_local(h, src);
    if (!grc) grc = gram_exchange(h, st);
    if (!grc) grc = gram_reduce(h, src);
    if (grc) return grc;
    cudaEventRecord(e.b, st);
  }
  {
    const EvPair e = next_ev(h, &dst == &h->U ? EV_SOLVE_USER : EV_SOLVE);
    cudaEventRecord(e.a, st);
    h->pieces_done = false;
    if (h->gram_side == &dst) h->gram_side = nullptr;
    if (dst.plan.kernel == SOLVE_PAIR) {
      // max |source factors| over the full replica (the same on every rank): the pair kernel's FP16 split scale
      const long long n = (long long)src.n_internal * h->KP;
      CK(h, cudaMemsetAsync(h->d_absmax, 0, sizeof(unsigned), st));
      pr::abs_max_kernel<<<4 * h->sm_count, 256, 0, st>>>(src.F, n, h->d_absmax);
      LAUNCHED(h);
    }
    const int rc = launch_solve(h, dst, src);
    if (rc) return rc;
    cudaEventRecord(e.b, st);
  }
  const bool prep = implicit && more;
  bool gram_pending = false;      // class sums computed, exchange + reduce still to do
  if (h->cfg.world_size > 1) {
    NcclApi& nc = nccl_api();
    const int W = h->cfg.world_size, me = h->cfg.world_rank;
    const EvPair e = next_ev(h, EV_COMM);
    if (h->pieces_done && h->sw.n_pieces > 1) {
      // all-gather piece by piece on the communication stream: piece c = local rows [R c / C, R (c + 1) / C) of every
      // rank, exchanged as soon as its rows are solved (grouped send/recv: NVSwitch gives every pair full bandwidth)
      cudaStream_t sc = h->comm_st;
      const int C = h->sw.n_pieces;
      bool first = true;
      for (int c = 0; c < C; ++c) {
        const long long lo = (long long)dst.R * c / C, hi = (long long)dst.R * (c + 1) / C;
        if (hi <= lo) continue;
        cudaStreamWaitEvent(sc, h->ev_piece[c], 0);
        if (lo < dst.n_heavy) cudaStreamWaitEvent(sc, h->ev_heavy, 0);
        if (first) { cudaEventRecord(e.a, st); first = false; }   // comm time reported = what is NOT hidden behind the solve
        const size_t cnt = (size_t)(hi - lo) * h->KP;
        if (nc.GroupStart() != ncclSuccess) return fail(h, PIO_ALS_ERR_COMM, "ncclGroupStart failed");
        for (int p = 0; p < W; ++p) {
          if (p == me) continue;
          if (nc.Send(dst.F + ((size_t)me * dst.R + lo) * h->KP, cnt, ncclFloat, p, h->comm, sc) != ncclSuccess ||
              nc.Recv(dst.F + ((size_t)p * dst.R + lo) * h->KP, cnt, ncclFloat, p, h->comm, sc) != ncclSuccess)
            return fail(h, PIO_ALS_ERR_COMM, "ncclSend/ncclRecv (factor pieces) failed");
        }
        if (nc.GroupEnd() != ncclSuccess) return fail(h, PIO_ALS_ERR_COMM, "ncclGroupEnd failed");
      }
      if (prep && gram_sharded(h)) {
        // the rank's own rows are final on the main stream once the heavy-row finish has joined it
        if (dst.n_heavy > 0) cudaStreamWaitEvent(st, h->ev_heavy, 0);
        const EvPair g = next_ev(h, EV_GRAM);
        cudaEventRecord(g.a, st);
        const int grc = gram_local(h, dst);
        if (grc) return grc;
        cudaEventRecord(g.b, st);
        cudaEventRecord(h->ev_gram, st);
        cudaStreamWaitEvent(sc, h->ev_gram, 0);
        const int xrc = gram_exchange(h, sc);
        if (xrc) return xrc;
        gram_pending = true;
      }
      cudaEventRecord(e.b, sc);
      cudaEventRecord(h->ev_comm, sc);
      cudaStreamWaitEvent(st, h->ev_comm, 0);
    } else {
      cudaEventRecord(e.a, st);
      const size_t cnt = (size_t)dst.R * h->KP;
      ncclResult_t r = nc.AllGather(dst.F + (size_t)me * cnt, dst.F, cnt, ncclFloat, h->comm, st);
      if (r != ncclSuccess)
        return fail(h, PIO_ALS_ERR_COMM, "ncclAllGather failed: %s", nc.GetErrorString ? nc.GetErrorString(r) : "?");
      cudaEventRecord(e.b, st);
    }
  }
  if (prep) {
    const EvPair e = next_ev(h, EV_GRAM);
    cudaEventRecord(e.a, st);
    int grc = PIO_ALS_OK;
    if (!gram_pending) {
      grc = gram_local(h, dst);
      if (!grc) grc = gram_exchange(h, st);
    }
    if (!grc) grc = gram_reduce(h, dst);
    if (grc) return grc;
    cudaEventRecord(e.b, st);
  }
  return PIO_ALS_OK;
}

}  // namespace pio

// =============================================================================================
// C ABI
// =============================================================================================
extern "C" {

int pio_als_abi_version(void) { return PIO_ALS_ABI_VERSION; }

int pio_als_device_count(void) {
  int n = 0;
  if (cudaGetDeviceCount(&n) != cudaSuccess) return PIO_ALS_ERR_CUDA;
  int ok = 0;
  for (int d = 0; d < n; ++d) {
    cudaDeviceProp pr;
    if (cudaGetDeviceProperties(&pr, d) == cudaSuccess && pr.major == 9 && pr.minor == 0) ++ok;
  }
  return ok;
}

int pio_als_nccl_unique_id(uint8_t out_id[128]) {
  NcclApi& a = nccl_api();
  if (!a.ok) return fail(nullptr, PIO_ALS_ERR_COMM, "libnccl.so.2 not loadable");
  ncclUniqueId id;
  if (a.GetUniqueId(&id) != ncclSuccess) return fail(nullptr, PIO_ALS_ERR_COMM, "ncclGetUniqueId failed");
  static_assert(sizeof(ncclUniqueId) == 128, "ncclUniqueId size");
  memcpy(out_id, &id, 128);
  return PIO_ALS_OK;
}

const char* pio_als_last_error(const pio_als_handle* h) { return h ? h->err.c_str() : g_create_error.c_str(); }

static int create_common(pio_als_handle* h) {
  int ndev = 0;
  cudaError_t ce = cudaGetDeviceCount(&ndev);
  if (ce != cudaSuccess || ndev == 0)
    return fail(nullptr, PIO_ALS_ERR_CUDA, "no CUDA device available (%s); this library has no CPU fallback",
                cudaGetErrorString(ce));
  if (h->cfg.device < 0 || h->cfg.device >= ndev) return fail(nullptr, PIO_ALS_ERR_ARG, "bad device %d", h->cfg.device);
  cudaDeviceProp pr;
  if (cudaGetDeviceProperties(&pr, h->cfg.device) != cudaSuccess) return fail(nullptr, PIO_ALS_ERR_CUDA, "cudaGetDeviceProperties");
  if (pr.major != 9 || pr.minor != 0)
    return fail(nullptr, PIO_ALS_ERR_CUDA, "device %d is sm_%d%d; this library is built for sm_90a (H100) only",
                h->cfg.device, pr.major, pr.minor);
  h->sm_count = pr.multiProcessorCount;
  h->st.sm_count = pr.multiProcessorCount;
  if (cudaSetDevice(h->cfg.device) != cudaSuccess) return fail(nullptr, PIO_ALS_ERR_CUDA, "cudaSetDevice");
  if (cudaStreamCreateWithFlags(&h->stream, cudaStreamNonBlocking) != cudaSuccess)
    return fail(nullptr, PIO_ALS_ERR_CUDA, "cudaStreamCreate");
  // keep freed blocks in the pool (ingest allocates and frees multi-GB scratch repeatedly)
  cudaMemPool_t pool;
  if (cudaDeviceGetDefaultMemPool(&pool, h->cfg.device) == cudaSuccess) {
    uint64_t thr = UINT64_MAX;
    cudaMemPoolSetAttribute(pool, cudaMemPoolAttrReleaseThreshold, &thr);
  }
  h->KP = pad_rank(h->cfg.rank);
  // the communication stream gets the highest priority: its few NCCL CTAs must not queue behind a grid that fills the
  // SMs (the YtY class sums run on the main stream next to the last pieces of the factor exchange)
  int prio_lo = 0, prio_hi = 0;
  cudaDeviceGetStreamPriorityRange(&prio_lo, &prio_hi);
  if (cudaStreamCreateWithFlags(&h->aux, cudaStreamNonBlocking) != cudaSuccess ||
      cudaStreamCreateWithPriority(&h->comm_st, cudaStreamNonBlocking, prio_hi) != cudaSuccess)
    return fail(nullptr, PIO_ALS_ERR_CUDA, "cudaStreamCreate");
  {
    cudaEvent_t* evs[5] = {&h->ev_start, &h->ev_heavy, &h->ev_comm, &h->ev_gram, nullptr};
    for (int i = 0; evs[i]; ++i)
      if (cudaEventCreateWithFlags(evs[i], cudaEventDisableTiming) != cudaSuccess) return fail(nullptr, PIO_ALS_ERR_CUDA, "cudaEventCreate");
    for (int i = 0; i < 8; ++i)
      if (cudaEventCreateWithFlags(&h->ev_piece[i], cudaEventDisableTiming) != cudaSuccess) return fail(nullptr, PIO_ALS_ERR_CUDA, "cudaEventCreate");
    if (const char* v = getenv("PIO_ALS_SERVE_FUSED")) h->serve_fused = atoi(v) != 0;
    if (const char* v = getenv("PIO_ALS_SERVE_TRACE")) h->serve_trace = atoi(v) != 0;
    if (const char* v = getenv("PIO_ALS_SCORE_BLOCKED")) h->score_blocked = atoi(v) != 0;
  }
  h->sw = read_solve_switches(getenv, h->KP, h->cfg.world_size);
  h->gram_blocks = GRAM_GROUPS * h->sm_count;   // a sharded run gives every rank whole groups: one CTA per SM at 8 GPUs
  if (cudaMallocAsync((void**)&h->yty, sizeof(float) * h->KP * h->KP, h->stream) != cudaSuccess ||
      cudaMallocAsync((void**)&h->gram_partial, sizeof(double) * (size_t)h->gram_blocks * h->KP * h->KP, h->stream) != cudaSuccess ||
      cudaMallocAsync((void**)&h->gram_gsum, sizeof(double) * (size_t)GRAM_GROUPS * h->KP * h->KP, h->stream) != cudaSuccess ||
      cudaMallocAsync((void**)&h->d_fail, sizeof(int), h->stream) != cudaSuccess ||
      cudaMallocAsync((void**)&h->d_counts, 4 * sizeof(int), h->stream) != cudaSuccess ||
      cudaMallocAsync((void**)&h->d_absmax, 2 * sizeof(unsigned), h->stream) != cudaSuccess)
    return fail(nullptr, PIO_ALS_ERR_CUDA, "device allocation failed");
  cudaMemsetAsync(h->yty, 0, sizeof(float) * h->KP * h->KP, h->stream);
  cudaMemsetAsync(h->d_fail, 0, sizeof(int), h->stream);
  return PIO_ALS_OK;
}

int pio_als_create(const pio_als_config* cfg, pio_als_handle** out) {
  if (!cfg || !out) return fail(nullptr, PIO_ALS_ERR_ARG, "null argument");
  *out = nullptr;
  if (cfg->abi_version != PIO_ALS_ABI_VERSION) return fail(nullptr, PIO_ALS_ERR_ARG, "abi_version mismatch");
  if (cfg->rank < 1 || cfg->rank > 128) return fail(nullptr, PIO_ALS_ERR_ARG, "rank must be in 1..128 (got %d)", cfg->rank);
  if (cfg->n_users < 1 || cfg->n_items < 1) return fail(nullptr, PIO_ALS_ERR_ARG, "n_users and n_items must be >= 1");
  if (cfg->world_size < 1 || cfg->world_rank < 0 || cfg->world_rank >= cfg->world_size)
    return fail(nullptr, PIO_ALS_ERR_ARG, "bad world_size/world_rank");
  if (!(cfg->lambda >= 0.0)) return fail(nullptr, PIO_ALS_ERR_ARG, "lambda must be >= 0");
  pio_als_handle* h = new pio_als_handle();
  h->cfg = *cfg;
  int rc = create_common(h);
  if (rc == PIO_ALS_OK && cfg->world_size > 1) {
    NcclApi& a = nccl_api();
    if (!a.ok) rc = fail(nullptr, PIO_ALS_ERR_COMM, "libnccl.so.2 not loadable");
    else {
      ncclUniqueId id;
      memcpy(&id, cfg->nccl_id, 128);
      ncclResult_t r = a.CommInitRank(&h->comm, cfg->world_size, id, cfg->world_rank);
      if (r != ncclSuccess) rc = fail(nullptr, PIO_ALS_ERR_COMM, "ncclCommInitRank failed: %s", a.GetErrorString ? a.GetErrorString(r) : "?");
    }
  }
  if (rc != PIO_ALS_OK) {
    pio_als_destroy(h);
    return rc;
  }
  *out = h;
  return PIO_ALS_OK;
}

void pio_als_destroy(pio_als_handle* h) {
  if (!h) return;
  if (h->stream) {
    cudaSetDevice(h->cfg.device);
    free_side(h, h->U, false);
    free_side(h, h->I, false);
    dfree(h, h->yty);
    dfree(h, h->gram_partial);
    dfree(h, h->gram_gsum);
    dfree(h, h->d_fail);
    dfree(h, h->d_counts);
    dfree(h, h->d_absmax);
    cudaStreamSynchronize(h->stream);
    if (h->tc_out) cudaFree(h->tc_out);
    if (h->d_dbg) cudaFree(h->d_dbg);
    if (h->d_timing) cudaFree(h->d_timing);
    for (auto& e : h->ev_pool) {
      cudaEventDestroy(e.a);
      cudaEventDestroy(e.b);
    }
    if (h->comm) nccl_api().CommDestroy(h->comm);
    if (h->ev_start) cudaEventDestroy(h->ev_start);
    if (h->ev_heavy) cudaEventDestroy(h->ev_heavy);
    if (h->ev_comm) cudaEventDestroy(h->ev_comm);
    if (h->ev_gram) cudaEventDestroy(h->ev_gram);
    for (int i = 0; i < 8; ++i)
      if (h->ev_piece[i]) cudaEventDestroy(h->ev_piece[i]);
    if (h->srv_dev) cudaFree(h->srv_dev);
    if (h->srv_host) cudaFreeHost(h->srv_host);
    if (h->srv_counter) cudaFree(h->srv_counter);
    if (h->aux) cudaStreamDestroy(h->aux);
    if (h->comm_st) cudaStreamDestroy(h->comm_st);
    cudaStreamDestroy(h->stream);
  }
  delete h;
}

static int set_ratings_impl(pio_als_handle* h, const int32_t* user, const int32_t* item, const float* rating, int64_t nnz,
                            int dedup_mode, const int64_t* ts, bool on_device, bool sharded) {
  if (!h) return PIO_ALS_ERR_ARG;
  const bool may_be_empty = sharded && h->cfg.world_size > 1;   // a rank's slice may be empty, the union may not
  if (nnz < 0 || (nnz == 0 && !may_be_empty))
    return fail(h, PIO_ALS_ERR_ARG, "ratings cannot be empty (the templates require(!ratings.take(1).isEmpty))");
  if (nnz > 0 && (!user || !item || !rating)) return fail(h, PIO_ALS_ERR_ARG, "null rating arrays");
  std::lock_guard<std::mutex> lk(h->mu);
  CK(h, cudaSetDevice(h->cfg.device));
  cudaStream_t st = h->stream;
  cudaEvent_t a, b;
  cudaEventCreate(&a);
  cudaEventCreate(&b);
  cudaEventRecord(a, st);
  int rc;
  {
    Scratch tmp(h);
    const int *du = user, *di = item;
    const float* dr = rating;
    const long long* dts = (const long long*)ts;
    auto stage = [&]() -> int {
      if (on_device || nnz == 0) return PIO_ALS_OK;
      int *tu = nullptr, *ti = nullptr;
      float* tr = nullptr;
      long long* tt = nullptr;
      CK(h, tmp.alloc(&tu, (size_t)nnz));
      CK(h, tmp.alloc(&ti, (size_t)nnz));
      CK(h, tmp.alloc(&tr, (size_t)nnz));
      CK(h, cudaMemcpyAsync(tu, user, sizeof(int) * nnz, cudaMemcpyHostToDevice, st));
      CK(h, cudaMemcpyAsync(ti, item, sizeof(int) * nnz, cudaMemcpyHostToDevice, st));
      CK(h, cudaMemcpyAsync(tr, rating, sizeof(float) * nnz, cudaMemcpyHostToDevice, st));
      if (ts && dedup_mode == PIO_ALS_DEDUP_KEEP_LAST) {
        CK(h, tmp.alloc(&tt, (size_t)nnz));
        CK(h, cudaMemcpyAsync(tt, ts, sizeof(long long) * nnz, cudaMemcpyHostToDevice, st));
      }
      du = tu; di = ti; dr = tr; dts = tt;
      return PIO_ALS_OK;
    };
    rc = stage();
    if (rc == PIO_ALS_OK) rc = ingest_device(h, du, di, dr, nnz, dedup_mode, dts, sharded);
  }
  cudaEventRecord(b, st);
  cudaEventSynchronize(b);
  float ms = 0;
  cudaEventElapsedTime(&ms, a, b);
  h->st.last_ingest_ms = ms;
  cudaEventDestroy(a);
  cudaEventDestroy(b);
  return rc;
}

int pio_als_set_ratings_coo_device(pio_als_handle* h, const int32_t* d_user, const int32_t* d_item,
                                   const float* d_rating, int64_t nnz, int dedup_mode, const int64_t* d_ts) {
  return set_ratings_impl(h, d_user, d_item, d_rating, nnz, dedup_mode, d_ts, true, false);
}

int pio_als_set_ratings_coo(pio_als_handle* h, const int32_t* user, const int32_t* item, const float* rating,
                            int64_t nnz, int dedup_mode, const int64_t* ts) {
  return set_ratings_impl(h, user, item, rating, nnz, dedup_mode, ts, false, false);
}

int pio_als_set_ratings_coo_sharded(pio_als_handle* h, const int32_t* user, const int32_t* item, const float* rating,
                                    int64_t nnz_local, int dedup_mode, const int64_t* ts) {
  return set_ratings_impl(h, user, item, rating, nnz_local, dedup_mode, ts, false, true);
}

int pio_als_set_ratings_coo_sharded_device(pio_als_handle* h, const int32_t* d_user, const int32_t* d_item,
                                           const float* d_rating, int64_t nnz_local, int dedup_mode, const int64_t* d_ts) {
  return set_ratings_impl(h, d_user, d_item, d_rating, nnz_local, dedup_mode, d_ts, true, true);
}

int pio_als_set_init(pio_als_handle* h, const float* user_factors, const float* item_factors) {
  if (!h) return PIO_ALS_ERR_ARG;
  std::lock_guard<std::mutex> lk(h->mu);
  if (!h->have_ratings) return fail(h, PIO_ALS_ERR_STATE, "set_init before set_ratings");
  if (!user_factors) return fail(h, PIO_ALS_ERR_ARG, "user_factors is null");
  CK(h, cudaSetDevice(h->cfg.device));
  cudaStream_t st = h->stream;
  const int k = h->cfg.rank;
  struct { Side* s; const float* f; } jobs[2] = {{&h->U, user_factors}, {&h->I, item_factors}};
  for (auto& j : jobs) {
    CK(h, cudaMemsetAsync(j.s->F, 0, sizeof(float) * (size_t)j.s->n_internal * h->KP, st));
    if (!j.f) continue;
    float* tmp = nullptr;
    CK(h, dalloc(h, &tmp, (size_t)j.s->n * k));
    CK(h, cudaMemcpyAsync(tmp, j.f, sizeof(float) * (size_t)j.s->n * k, cudaMemcpyHostToDevice, st));
    scatter_init_kernel<<<nblk((long long)j.s->n * h->KP, 256), 256, 0, st>>>(tmp, j.s->n, k, h->KP, j.s->perm, j.s->deg, j.s->F);
    LAUNCHED(h);
    dfree(h, tmp);
  }
  CK(h, cudaStreamSynchronize(st));
  h->have_init = true;
  return PIO_ALS_OK;
}

int pio_als_run(pio_als_handle* h, int n_iters) {
  if (!h) return PIO_ALS_ERR_ARG;
  std::lock_guard<std::mutex> lk(h->mu);
  if (!h->have_ratings) return fail(h, PIO_ALS_ERR_STATE, "run before set_ratings");
  if (n_iters < 0) return fail(h, PIO_ALS_ERR_ARG, "n_iters < 0");
  CK(h, cudaSetDevice(h->cfg.device));
  if (!h->have_init) {
    if (h->cfg.init_mode == PIO_ALS_INIT_HASH) {
      int rc = init_hash(h);
      if (rc) return rc;
    } else {
      return fail(h, PIO_ALS_ERR_STATE, "no initial factors: call pio_als_set_init or use PIO_ALS_INIT_HASH");
    }
  }
  cudaStream_t st = h->stream;
  h->ev_used = 0;
  CK(h, cudaMemsetAsync(h->d_fail, 0, sizeof(int), st));
  EvPair& tot = next_ev(h, -1);
  cudaEventRecord(tot.a, st);
  h->gram_side = nullptr;      // the factors may have been replaced since the last run
  for (int it = 0; it < n_iters; ++it) {
    int rc = half_step(h, h->I, h->U, true);                  // item factors from user factors
    if (rc) return rc;
    rc = half_step(h, h->U, h->I, it + 1 < n_iters);          // user factors from item factors
    if (rc) return rc;
  }
  cudaEventRecord(tot.b, st);
  int nfail = 0;
  CK(h, cudaMemcpyAsync(&nfail, h->d_fail, sizeof(int), cudaMemcpyDeviceToHost, st));
  CK(h, cudaStreamSynchronize(st));
  double ms[EV_NKIND] = {0, 0, 0, 0};
  float t = 0;
  for (size_t i = 0; i < h->ev_used; ++i) {
    EvPair& e = h->ev_pool[i];
    cudaEventElapsedTime(&t, e.a, e.b);
    if (e.kind >= 0) ms[e.kind] += t;
    else h->st.last_run_ms = t;
  }
  h->st.last_solve_ms = ms[EV_SOLVE] + ms[EV_SOLVE_USER];
  h->phase_ms[0] = ms[EV_SOLVE];
  h->phase_ms[1] = ms[EV_SOLVE_USER];
  h->phase_ms[2] = ms[EV_GRAM];
  h->phase_ms[3] = ms[EV_COMM];
  h->phase_ms[6] = (double)n_iters;
  h->st.last_gram_ms = ms[EV_GRAM];
  h->st.last_comm_ms = ms[EV_COMM];
  h->trained = true;
  if (nfail)
    return fail(h, PIO_ALS_ERR_NUMERIC, "%d normal equations were not positive definite (MLlib: dppsv info != 0)", nfail);
  return PIO_ALS_OK;
}

int pio_als_get_phase_ms(pio_als_handle* h, double out[8]) {
  if (!h || !out) return PIO_ALS_ERR_ARG;
  std::lock_guard<std::mutex> lk(h->mu);
  for (int i = 0; i < 8; ++i) out[i] = h->phase_ms[i];
  // kernel of the rows below the heavy-row threshold: 0 = FP32 (als_solve_kernel), 1 = wgmma, 2 = mma.sync, 3 = pair
  out[4] = phase_code(h->I.plan.kernel);
  out[5] = phase_code(h->U.plan.kernel);
  return PIO_ALS_OK;
}

int pio_als_get_factors(pio_als_handle* h, float* user_out, float* item_out, uint8_t* user_has, uint8_t* item_has) {
  if (!h) return PIO_ALS_ERR_ARG;
  std::lock_guard<std::mutex> lk(h->mu);
  if (!h->have_ratings && !h->trained) return fail(h, PIO_ALS_ERR_STATE, "no model");
  CK(h, cudaSetDevice(h->cfg.device));
  cudaStream_t st = h->stream;
  const int k = h->cfg.rank;
  struct { Side* s; float* f; uint8_t* has; } jobs[2] = {{&h->U, user_out, user_has}, {&h->I, item_out, item_has}};
  for (auto& j : jobs) {
    if (j.f) {
      float* tmp = nullptr;
      CK(h, dalloc(h, &tmp, (size_t)j.s->n * k));
      gather_factors_kernel<<<nblk((long long)j.s->n * k, 256), 256, 0, st>>>(j.s->F, j.s->n, k, h->KP, j.s->perm, tmp);
      LAUNCHED(h);
      CK(h, cudaMemcpyAsync(j.f, tmp, sizeof(float) * (size_t)j.s->n * k, cudaMemcpyDeviceToHost, st));
      dfree(h, tmp);
    }
    if (j.has) {
      uint8_t* tmp = nullptr;
      CK(h, dalloc(h, &tmp, (size_t)j.s->n));
      has_kernel<<<nblk(j.s->n, 256), 256, 0, st>>>(j.s->deg, j.s->n, tmp);
      LAUNCHED(h);
      CK(h, cudaMemcpyAsync(j.has, tmp, (size_t)j.s->n, cudaMemcpyDeviceToHost, st));
      dfree(h, tmp);
    }
  }
  CK(h, cudaStreamSynchronize(st));
  return PIO_ALS_OK;
}

int pio_als_train(pio_als_handle* h, const int32_t* user, const int32_t* item, const float* rating, int64_t nnz,
                  int dedup_mode, const int64_t* ts, const float* user_init, const float* item_init, int n_iters,
                  float* user_out, float* item_out, uint8_t* user_has, uint8_t* item_has) {
  int rc = pio_als_set_ratings_coo(h, user, item, rating, nnz, dedup_mode, ts);
  if (rc) return rc;
  if (user_init) {
    rc = pio_als_set_init(h, user_init, item_init);
    if (rc) return rc;
  }
  rc = pio_als_run(h, n_iters);
  if (rc) return rc;
  return pio_als_get_factors(h, user_out, item_out, user_has, item_has);
}

}  // extern "C"

// ---- top-k scoring: score_plan.h decides what runs, the helpers below launch it ----------------------------------------
namespace pio {
static int serve_reserve(pio_als_handle* h, size_t dev_bytes, size_t host_bytes) {
  if (h->srv_dev_cap < dev_bytes) {
    CK(h, cudaStreamSynchronize(h->stream));
    if (h->srv_dev) cudaFree(h->srv_dev);
    h->srv_dev = nullptr;
    h->srv_dev_cap = 0;
    CK(h, cudaMalloc((void**)&h->srv_dev, dev_bytes));
    h->srv_dev_cap = dev_bytes;
  }
  if (h->srv_host_cap < host_bytes) {
    CK(h, cudaStreamSynchronize(h->stream));
    if (h->srv_host) cudaFreeHost(h->srv_host);
    h->srv_host = nullptr;
    h->srv_host_cap = 0;
    CK(h, cudaHostAlloc((void**)&h->srv_host, host_bytes, cudaHostAllocMapped));
    CK(h, cudaHostGetDevicePointer((void**)&h->srv_host_dev, h->srv_host, 0));
    h->srv_host_cap = host_bytes;
  }
  return PIO_ALS_OK;
}
static inline size_t al256(size_t x) { return (x + 255) & ~(size_t)255; }

// the layout of a serving arena: blocks in call order, each starting on a 256-byte boundary
struct ArenaLayout {
  size_t bytes = 0;
  size_t take(size_t n) {
    const size_t at = bytes;
    bytes = al256(bytes + n);
    return at;
  }
};

// Every launch of a scoring call goes through here: raise the kernel's dynamic shared-memory limit when it takes any,
// launch on the handle's stream, count the launch, record which scoring kernel ran (path: its PIO_ALS_PATH_* bit, 0 for
// gathers, copies and merges) and fail on a launch error -- a kernel that never started would leave stale candidates
// behind.
template <typename... KArgs, typename... Args>
static int score_launch(pio_als_handle* h, void (*kernel)(KArgs...), dim3 grid, dim3 block, size_t smem, unsigned path,
                        Args... args) {
  if (smem) {
    const int rc = ensure_dyn_smem(h, (const void*)kernel, smem);
    if (rc) return rc;
  }
  kernel<<<grid, block, smem, h->stream>>>(args...);
  LAUNCHED(h);
  h->st.last_score_path |= path;
  CK(h, cudaGetLastError());
  return PIO_ALS_OK;
}

template <int N>
using IntC = std::integral_constant<int, N>;
// f(IntC<KP>()) for the handle's padded rank: the blocked and single-query kernels exist for KP 16, 32 and 64
template <class F>
static int with_kp(int kp, F&& f) {
  if (kp == 16) return f(IntC<16>());
  if (kp == 32) return f(IntC<32>());
  return f(IntC<64>());
}

static ScoreEnv score_env(const pio_als_handle* h) {
  return ScoreEnv{h->KP, h->sm_count, h->I.n_internal, h->serve_fused, h->score_blocked};
}

struct DevFilter {
  uint8_t* mask = nullptr;
  double* weight = nullptr;
};
// arena bytes of a call's item mask and weights (either may be absent)
static size_t filter_bytes(const pio_als_handle* h, const uint8_t* mask, const double* weight) {
  return al256(mask ? (size_t)h->I.n : 0) + al256(weight ? sizeof(double) * (size_t)h->I.n : 0);
}
// the call's item mask and weights on the device: in call scratch, or (tmp == nullptr) in the device arena at `at`
static int upload_filter(pio_als_handle* h, const uint8_t* mask, const double* weight, Scratch* tmp, size_t at, DevFilter* f) {
  const size_t n = (size_t)h->I.n;
  if (mask) {
    if (tmp) CK(h, tmp->alloc(&f->mask, n));
    else f->mask = h->srv_dev + at;
    CK(h, cudaMemcpyAsync(f->mask, mask, n, cudaMemcpyHostToDevice, h->stream));
  }
  if (weight) {
    if (tmp) CK(h, tmp->alloc(&f->weight, n));
    else f->weight = (double*)(h->srv_dev + at + al256(mask ? n : 0));
    CK(h, cudaMemcpyAsync(f->weight, weight, sizeof(double) * n, cudaMemcpyHostToDevice, h->stream));
  }
  return PIO_ALS_OK;
}

// where the merge writes: ids, scores and counts of every query, and the bounds of the next pass (multi-pass plans)
struct MergeOut {
  int* items = nullptr;
  float* scores = nullptr;
  int* count = nullptr;
  ScoreIdx* bound = nullptr;
};
// device results of n queries in call scratch
static int alloc_results(pio_als_handle* h, Scratch& tmp, int n, int topk, bool bound, MergeOut* o) {
  CK(h, tmp.alloc(&o->items, (size_t)n * topk));
  CK(h, tmp.alloc(&o->scores, (size_t)n * topk));
  CK(h, tmp.alloc(&o->count, (size_t)n));
  if (bound) CK(h, tmp.alloc(&o->bound, (size_t)n));
  return PIO_ALS_OK;
}
// device results to the caller: three copies and one synchronisation
static int deliver(pio_als_handle* h, const MergeOut& o, int n, int topk, int32_t* items, float* scores, int32_t* count) {
  cudaStream_t st = h->stream;
  CK(h, cudaMemcpyAsync(items, o.items, sizeof(int) * (size_t)n * topk, cudaMemcpyDeviceToHost, st));
  CK(h, cudaMemcpyAsync(scores, o.scores, sizeof(float) * (size_t)n * topk, cudaMemcpyDeviceToHost, st));
  if (count) CK(h, cudaMemcpyAsync(count, o.count, sizeof(int) * (size_t)n, cudaMemcpyDeviceToHost, st));
  CK(h, cudaStreamSynchronize(st));
  return PIO_ALS_OK;
}
// results of the serving paths, in the mapped host arena: ids, scores and counts of up to cap queries
struct MappedOut {
  size_t items, scores, count;
  MappedOut(ArenaLayout& host, int cap, int topk)
      : items(host.take(sizeof(int) * (size_t)cap * topk)), scores(host.take(sizeof(float) * (size_t)cap * topk)),
        count(host.take(sizeof(int) * (size_t)cap)) {}
  MergeOut dev(const pio_als_handle* h) const {
    MergeOut o;
    o.items = (int*)(h->srv_host_dev + items);
    o.scores = (float*)(h->srv_host_dev + scores);
    o.count = (int*)(h->srv_host_dev + count);
    return o;
  }
  // once the writer has finished
  void copy(const pio_als_handle* h, int n, int topk, int32_t* out_items, float* out_scores, int32_t* out_count) const {
    memcpy(out_items, h->srv_host + items, sizeof(int) * (size_t)n * topk);
    memcpy(out_scores, h->srv_host + scores, sizeof(float) * (size_t)n * topk);
    if (out_count) memcpy(out_count, h->srv_host + count, sizeof(int) * (size_t)n);
  }
};

// one launch of a pass: the query groups [g0, g0 + grid.y)
struct Chunk {
  dim3 grid;               // (gx, groups of this launch)
  int g0;                  // first group
  int q0, nq;              // first query and queries of these groups (plans with qpg > 0)
  int pk;                  // results of this pass
  const ScoreIdx* bound;   // bound of the first query (nullptr in the first pass)
  ScoreIdx* cand;          // candidate lists of the first query
};
// The passes of a plan: in each, the scoring launches (launch(chunk), at most p.chunk query groups each), then the
// merge of every query's candidate lists into the results; the last result of a full pass bounds the next one.
template <class Launch>
static int run_passes(pio_als_handle* h, const ScorePlan& p, int n_queries, int topk, ScoreIdx* cand, const MergeOut& out,
                      Launch&& launch) {
  for (int done = 0; done < topk; done += TK_MAXK) {
    const int pk = topk - done < TK_MAXK ? topk - done : TK_MAXK;
    if (done > 0) h->st.last_score_path |= PIO_ALS_PATH_MULTI_PASS;
    for (int g0 = 0; g0 < p.ngroups; g0 += p.chunk) {
      const int ng = p.ngroups - g0 < p.chunk ? p.ngroups - g0 : p.chunk;
      Chunk c;
      c.grid = dim3(p.gx, ng);
      c.g0 = g0;
      c.q0 = g0 * p.qpg;
      c.nq = n_queries - c.q0 < ng * p.qpg ? n_queries - c.q0 : ng * p.qpg;
      c.pk = pk;
      c.bound = done > 0 ? out.bound + c.q0 : nullptr;
      c.cand = cand + (size_t)c.q0 * p.lists * pk;
      const int rc = launch(c);
      if (rc) return rc;
    }
    // the candidate lists of a query are [lists][pk] entries, stored with stride pk
    const int rc = score_launch(h, topk_merge_kernel, dim3(n_queries), dim3(TK_THREADS), 0, 0, (const ScoreIdx*)cand,
                                p.lists * pk, pk, topk, done, out.items, out.scores, out.count, out.bound);
    if (rc) return rc;
  }
  return PIO_ALS_OK;
}

// the recommend kernel of the plan for the users of chunk c (xq / valid: the gathered user vectors)
static int launch_dot(pio_als_handle* h, const ScorePlan& p, const Chunk& c, const float* d_xq, const uint8_t* d_valid,
                      const DevFilter& f) {
  const float* xq = d_xq + (size_t)c.q0 * h->KP;
  if (p.kernel == PIO_ALS_PATH_DOT_BLOCKED)
    return with_kp(h->KP, [&](auto kp) {
      return score_launch(h, score_dot_blocked_kernel<decltype(kp)::value>, c.grid, dim3(p.threads), p.smem, p.kernel, h->I.F,
                          h->I.n_internal, xq, d_valid + c.q0, c.nq, h->I.cand_ext, f.mask, f.weight, c.pk, c.cand);
    });
  return score_launch(h, score_dot_topk_batched_kernel, c.grid, dim3(p.threads), p.smem, p.kernel, h->I.F, h->I.n_internal,
                      h->KP, xq, d_valid + c.q0, c.nq, h->I.cand_ext, f.mask, f.weight, c.bound, c.pk, c.cand);
}

// the query vectors of a similar batch on the device: the vectors (qf), the first query (q0, bins only) and the first
// vector (v0) of every bin / group, the query of every vector (vq) and the id list of every query (qptr / qid)
struct CosQueries {
  const float* qf;
  const int* q0;
  const int* v0;
  int n_bins;
  const int* vq;
  const long long* qptr;
  const int* qid;
  int keep;   // PIO_ALS_SIM_KEEP_QUERY_ITEMS
};
// the batch similar kernel of the plan for the bins / groups of chunk c
static int launch_cos(pio_als_handle* h, const ScorePlan& p, const Chunk& c, const CosQueries& q, const DevFilter& f) {
  if (p.kernel == PIO_ALS_PATH_COS_BLOCKED)
    return with_kp(h->KP, [&](auto kp) {
      return score_launch(h, score_cos_blocked_kernel<decltype(kp)::value>, c.grid, dim3(p.threads), p.smem, p.kernel, h->I.F,
                          h->I.n_internal, h->cfg.rank, q.qf, q.q0 + (size_t)c.g0 * DB_WPR, q.v0 + (size_t)c.g0 * DB_WPR,
                          q.n_bins - c.g0 * DB_WPR, q.vq, q.qptr, q.qid, h->I.cand_ext, f.mask, f.weight, q.keep, c.pk, c.cand);
    });
  return score_launch(h, score_cos_topk_multi_kernel, c.grid, dim3(p.threads), p.smem, p.kernel, h->I.F, h->I.n_internal,
                      h->KP, h->cfg.rank, q.qf, q.v0 + c.g0, q.vq, q.qptr + c.q0, q.qid, c.nq, h->I.cand_ext, f.mask, f.weight,
                      c.bound, q.keep, c.pk, c.cand);
}

// R2: n <= SB_QB users, topk <= TK_MAXK, in the serving arenas: three launches and one synchronisation
static int recommend_small(pio_als_handle* h, const ScorePlan& p, const int32_t* users, int n, int topk,
                           const uint8_t* item_mask, const double* item_weight, int32_t* out_items, float* out_scores,
                           int32_t* out_count) {
  const int KP = h->KP;
  ArenaLayout dev, host;
  const size_t o_xq = dev.take(sizeof(float) * SB_QB * KP), o_valid = dev.take(SB_QB),
               o_cand = dev.take(sizeof(ScoreIdx) * (size_t)SB_QB * p.gx * topk),
               o_filter = dev.take(filter_bytes(h, item_mask, item_weight));
  const MappedOut res(host, SB_QB, topk);
  int rc = serve_reserve(h, dev.bytes, host.bytes);
  if (rc) return rc;
  float* d_xq = (float*)(h->srv_dev + o_xq);
  uint8_t* d_valid = h->srv_dev + o_valid;
  DevFilter f;
  rc = upload_filter(h, item_mask, item_weight, nullptr, o_filter, &f);
  if (rc) return rc;
  IdList ids;
  for (int q = 0; q < n; ++q) ids.v[q] = users[q];
  rc = score_launch(h, gather_rows_ids_kernel, dim3(n), dim3(64), 0, 0, h->U.F, KP, ids, h->U.perm, h->U.deg, h->U.n, d_xq,
                    d_valid);
  if (rc) return rc;
  rc = run_passes(h, p, n, topk, (ScoreIdx*)(h->srv_dev + o_cand), res.dev(h),
                  [&](const Chunk& c) { return launch_dot(h, p, c, d_xq, d_valid, f); });
  if (rc) return rc;
  CK(h, cudaStreamSynchronize(h->stream));
  res.copy(h, n, topk, out_items, out_scores, out_count);
  return PIO_ALS_OK;
}

// S2: one similar() query with nq <= SM_NV items and topk <= TK_MAXK, in the serving arenas: query items without a factor
// enter as zero vectors (their cosine terms are exactly 0, like the reference skipping them), so no host round trip is
// needed to compact the query
static int similar_small(pio_als_handle* h, const ScorePlan& p, const int32_t* query_items, int nq, int topk,
                         const uint8_t* item_mask, const double* item_weight, int flags, int32_t* out_items,
                         float* out_scores, int32_t* out_count) {
  ArenaLayout dev, host;
  const size_t o_qf = dev.take(sizeof(float) * SM_NV * h->KP), o_cand = dev.take(sizeof(ScoreIdx) * (size_t)p.gx * topk),
               o_filter = dev.take(filter_bytes(h, item_mask, item_weight));
  // mapped host arena: results, then the tiny query description the kernel reads over PCIe
  const MappedOut res(host, 1, topk);
  const size_t ho_g = host.take(sizeof(int) * 2), ho_vq = host.take(sizeof(int) * SM_NV),
               ho_qp = host.take(sizeof(long long) * 2), ho_qid = host.take(sizeof(int) * SM_NV);
  int rc = serve_reserve(h, dev.bytes, host.bytes);
  if (rc) return rc;
  float* d_qf = (float*)(h->srv_dev + o_qf);
  DevFilter f;
  rc = upload_filter(h, item_mask, item_weight, nullptr, o_filter, &f);
  if (rc) return rc;
  int* hg = (int*)(h->srv_host + ho_g);
  int* hvq = (int*)(h->srv_host + ho_vq);
  long long* hqp = (long long*)(h->srv_host + ho_qp);
  int* hqid = (int*)(h->srv_host + ho_qid);
  hg[0] = 0; hg[1] = nq;
  hqp[0] = 0; hqp[1] = nq;
  IdList ids;
  for (int q = 0; q < nq; ++q) { ids.v[q] = query_items[q]; hvq[q] = 0; hqid[q] = query_items[q]; }
  rc = score_launch(h, gather_rows_ids_kernel, dim3(nq), dim3(64), 0, 0, h->I.F, h->KP, ids, h->I.perm, h->I.deg, h->I.n,
                    d_qf, (uint8_t*)nullptr);
  if (rc) return rc;
  const CosQueries q{d_qf, nullptr, (const int*)(h->srv_host_dev + ho_g), 1, (const int*)(h->srv_host_dev + ho_vq),
                     (const long long*)(h->srv_host_dev + ho_qp), (const int*)(h->srv_host_dev + ho_qid),
                     (flags & PIO_ALS_SIM_KEEP_QUERY_ITEMS) ? 1 : 0};
  rc = run_passes(h, p, 1, topk, (ScoreIdx*)(h->srv_dev + o_cand), res.dev(h),
                  [&](const Chunk& c) { return launch_cos(h, p, c, q, f); });
  if (rc) return rc;
  CK(h, cudaStreamSynchronize(h->stream));
  res.copy(h, 1, topk, out_items, out_scores, out_count);
  return PIO_ALS_OK;
}

// R1 / S1: ONE query in ONE launch (score_one_kernel): recommend for one user (cos = false, ids[0] = the user) or similar
// for nq <= S1_MAXNV query items.  The host waits on a sequence flag in the mapped arena instead of a stream
// synchronisation.
static int serve_one(pio_als_handle* h, const ScorePlan& p, bool cos, const int32_t* ids, int nq, int topk,
                     const uint8_t* item_mask, const double* item_weight, int flags, int32_t* out_items, float* out_scores,
                     int32_t* out_count) {
  cudaStream_t st = h->stream;
  ArenaLayout dev, host;
  const size_t o_cand = dev.take(sizeof(ScoreIdx) * (size_t)p.gx * topk),
               o_filter = dev.take(filter_bytes(h, item_mask, item_weight));
  const MappedOut res(host, 1, topk);
  const size_t ho_flag = host.take(sizeof(unsigned)), ho_trace = host.take(sizeof(unsigned long long) * 8);
  const bool fresh_host = h->srv_host_cap < host.bytes;
  int rc = serve_reserve(h, dev.bytes, host.bytes);
  if (rc) return rc;
  if (fresh_host) memset(h->srv_host, 0, h->srv_host_cap);
  if (!h->srv_counter) {
    CK(h, cudaMalloc((void**)&h->srv_counter, 256));
    CK(h, cudaMemsetAsync(h->srv_counter, 0, 256, st));
  }
  DevFilter f;
  rc = upload_filter(h, item_mask, item_weight, nullptr, o_filter, &f);
  if (rc) return rc;
  OneQuery qry;
  qry.nq = nq;
  for (int t = 0; t < S1_MAXNV; ++t) qry.ids[t] = t < nq ? ids[t] : -1;
  const unsigned seq = ++h->srv_seq ? h->srv_seq : ++h->srv_seq;   // never 0: a fresh arena reads 0
  volatile unsigned* flag = (volatile unsigned*)(h->srv_host + ho_flag);
  const MergeOut m = res.dev(h);
  unsigned* m_flag = (unsigned*)(h->srv_host_dev + ho_flag);
  unsigned long long* m_trace = h->serve_trace ? (unsigned long long*)(h->srv_host_dev + ho_trace) : nullptr;
  unsigned long long* g_thr = reinterpret_cast<unsigned long long*>(h->srv_counter + 2);
  ScoreIdx* d_cand = (ScoreIdx*)(h->srv_dev + o_cand);
  const int keep = (flags & PIO_ALS_SIM_KEEP_QUERY_ITEMS) ? 1 : 0;
  const Side& q = cos ? h->I : h->U;
  const auto launch = [&](auto c, auto nvp, auto kp) {
    return score_launch(h, score_one_kernel<decltype(c)::value, decltype(nvp)::value, decltype(kp)::value>, dim3(p.gx),
                        dim3(p.threads), p.smem, p.kernel, h->I.F, h->I.n_internal, h->cfg.rank, q.F, q.perm, q.deg, q.n, qry,
                        h->I.cand_ext, f.mask, f.weight, keep, topk, d_cand, h->srv_counter, g_thr, m.items, m.scores,
                        m.count, m_flag, seq, m_trace);
  };
  const auto t_call = std::chrono::steady_clock::now();
  rc = with_kp(h->KP, [&](auto kp) {
    if (!cos) return launch(std::false_type(), IntC<1>(), kp);
    if (p.nvp == 1) return launch(std::true_type(), IntC<1>(), kp);
    if (p.nvp == 2) return launch(std::true_type(), IntC<2>(), kp);
    if (p.nvp == 4) return launch(std::true_type(), IntC<4>(), kp);
    return launch(std::true_type(), IntC<8>(), kp);
  });
  if (rc) return rc;
  for (unsigned spins = 1; *flag != seq; ++spins) {
    if ((spins & 0x3FFFu) == 0) {   // a faulted kernel never writes the flag: ask the stream now and then
      const cudaError_t e = cudaStreamQuery(st);
      if (e != cudaErrorNotReady) {
        if (e != cudaSuccess) CK(h, e);
        if (*flag != seq) return fail(h, PIO_ALS_ERR_CUDA, "single-query kernel finished without publishing its result");
      }
    }
#if defined(__x86_64__)
    __builtin_ia32_pause();
#endif
  }
  __atomic_thread_fence(__ATOMIC_ACQUIRE);
  if (h->serve_trace) {
    const unsigned long long* t = (const unsigned long long*)(h->srv_host + ho_trace);
    const double host_us = std::chrono::duration<double, std::micro>(std::chrono::steady_clock::now() - t_call).count();
    fprintf(stderr, "pio serve trace: host launch->flag %.1f us; publishing CTA: query lookup %.1f us, first step %.1f us, rest of the scan "
            "%.1f us, cta merge + arrival %.1f us, list merge %.1f us, system fence %.1f us\n", host_us, (t[5] - t[0]) * 1e-3,
            (t[6] - t[5]) * 1e-3, (t[1] - t[6]) * 1e-3, (t[2] - t[1]) * 1e-3, (t[3] - t[2]) * 1e-3, (t[4] - t[3]) * 1e-3);
  }
  res.copy(h, 1, topk, out_items, out_scores, out_count);
  return PIO_ALS_OK;
}

// S3 / S4: a gathered similar batch (qf_all / valid: the vector of every query id and whether it owns a factor), its
// queries in the bins / groups q0 of the plan
static int similar_groups(pio_als_handle* h, const ScorePlan& p, const std::vector<int>& q0, const int64_t* q_ptr,
                          int n_queries, int topk, const std::vector<uint8_t>& valid, const float* d_qf_all,
                          const int* d_qid, const DevFilter& f, int flags, Scratch& tmp, int32_t* out_items,
                          float* out_scores, int32_t* out_count) {
  cudaStream_t st = h->stream;
  const int KP = h->KP;
  const bool bins = p.kernel == PIO_ALS_PATH_COS_BLOCKED;
  // the vectors that own a factor, bin / group after bin / group, query order kept: their row in qf_all, their query
  // (global in a bin, inside the group in S4) and the first vector of every bin / group
  std::vector<int> v0, vsrc, vq;
  for (size_t g = 0; g + 1 < q0.size(); ++g) {
    v0.push_back((int)vsrc.size());
    for (int j = q0[g]; j < q0[g + 1]; ++j)
      for (long long t = q_ptr[j]; t < q_ptr[j + 1]; ++t)
        if (valid[(size_t)(t - q_ptr[0])]) {
          vsrc.push_back((int)(t - q_ptr[0]));
          vq.push_back(bins ? j : j - q0[g]);
        }
  }
  v0.push_back((int)vsrc.size());
  std::vector<long long> rel((size_t)n_queries + 1);
  for (int j = 0; j <= n_queries; ++j) rel[j] = q_ptr[j] - q_ptr[0];
  const int nvec = (int)vsrc.size();
  const size_t nv1 = nvec > 0 ? (size_t)nvec : 1;
  int *d_q0 = nullptr, *d_v0 = nullptr, *d_vq = nullptr, *d_vsrc = nullptr;
  long long* d_qptr = nullptr;
  float* d_qfc = nullptr;
  ScoreIdx* d_cand = nullptr;
  if (bins) CK(h, tmp.alloc(&d_q0, q0.size()));
  CK(h, tmp.alloc(&d_v0, v0.size()));
  CK(h, tmp.alloc(&d_vq, nv1));
  CK(h, tmp.alloc(&d_vsrc, nv1));
  CK(h, tmp.alloc(&d_qptr, rel.size()));
  CK(h, tmp.alloc(&d_qfc, nv1 * KP));
  if (bins) CK(h, cudaMemcpyAsync(d_q0, q0.data(), sizeof(int) * q0.size(), cudaMemcpyHostToDevice, st));
  CK(h, cudaMemcpyAsync(d_v0, v0.data(), sizeof(int) * v0.size(), cudaMemcpyHostToDevice, st));
  CK(h, cudaMemcpyAsync(d_qptr, rel.data(), sizeof(long long) * rel.size(), cudaMemcpyHostToDevice, st));
  if (nvec > 0) {
    CK(h, cudaMemcpyAsync(d_vq, vq.data(), sizeof(int) * nvec, cudaMemcpyHostToDevice, st));
    CK(h, cudaMemcpyAsync(d_vsrc, vsrc.data(), sizeof(int) * nvec, cudaMemcpyHostToDevice, st));
    const int rc = score_launch(h, copy_rows_kernel, dim3(nvec), dim3(64), 0, 0, d_qf_all, KP, (const int*)d_vsrc, d_qfc);
    if (rc) return rc;
  }
  CK(h, tmp.alloc(&d_cand, (size_t)n_queries * p.lists * p.pass_k));
  MergeOut o;
  int rc = alloc_results(h, tmp, n_queries, topk, p.passes > 1, &o);
  if (rc) return rc;
  const CosQueries q{d_qfc, d_q0, d_v0, (int)q0.size() - 1, d_vq, d_qptr, d_qid, (flags & PIO_ALS_SIM_KEEP_QUERY_ITEMS) ? 1 : 0};
  rc = run_passes(h, p, n_queries, topk, d_cand, o, [&](const Chunk& c) { return launch_cos(h, p, c, q, f); });
  if (rc) return rc;
  return deliver(h, o, n_queries, topk, out_items, out_scores, out_count);
}

// S5: one similar() query with mask / weights already on the device; results to HOST out arrays (topk entries)
static int similar_one(pio_als_handle* h, const int32_t* query_items, int nq, int topk, const DevFilter& f, int flags,
                       int32_t* out_items, float* out_scores, int32_t* out_count) {
  for (int t = 0; t < topk; ++t) { out_items[t] = -1; out_scores[t] = 0.f; }
  if (out_count) *out_count = 0;
  if (nq == 0) return PIO_ALS_OK;
  cudaStream_t st = h->stream;
  const int KP = h->KP, k = h->cfg.rank;
  const int keep_query = (flags & PIO_ALS_SIM_KEEP_QUERY_ITEMS) ? 1 : 0;
  Scratch tmp(h);
  int* d_q = nullptr;
  float* d_qf = nullptr;
  uint8_t* d_valid = nullptr;
  CK(h, tmp.alloc(&d_q, (size_t)nq));
  CK(h, tmp.alloc(&d_qf, (size_t)nq * KP));
  CK(h, tmp.alloc(&d_valid, (size_t)nq));
  CK(h, cudaMemcpyAsync(d_q, query_items, sizeof(int) * nq, cudaMemcpyHostToDevice, st));
  int rc = score_launch(h, gather_rows_kernel, dim3(nq), dim3(64), 0, 0, h->I.F, KP, (const int*)d_q, nq, h->I.perm,
                        h->I.deg, h->I.n, d_qf, d_valid);
  if (rc) return rc;
  std::vector<uint8_t> valid(nq);
  CK(h, cudaMemcpyAsync(valid.data(), d_valid, (size_t)nq, cudaMemcpyDeviceToHost, st));
  CK(h, cudaStreamSynchronize(st));
  // compact the query vectors that own a factor (order preserved); all query ids stay excluded
  std::vector<int> keep;
  for (int q = 0; q < nq; ++q)
    if (valid[q]) keep.push_back(q);
  const int nqv = (int)keep.size();
  const ScorePlan p = plan_similar_query(score_env(h), nqv, nq, topk);
  if (p.route == ROUTE_NONE) return PIO_ALS_OK;
  float* d_qc = nullptr;
  CK(h, tmp.alloc(&d_qc, keep.size() * (size_t)KP));
  for (size_t j = 0; j < keep.size(); ++j)
    CK(h, cudaMemcpyAsync(d_qc + j * KP, d_qf + (size_t)keep[j] * KP, sizeof(float) * KP, cudaMemcpyDeviceToDevice, st));
  ScoreIdx* d_cand = nullptr;
  CK(h, tmp.alloc(&d_cand, (size_t)p.lists * p.pass_k));
  MergeOut o;
  rc = alloc_results(h, tmp, 1, topk, p.passes > 1, &o);
  if (rc) return rc;
  rc = run_passes(h, p, 1, topk, d_cand, o, [&](const Chunk& c) {
    return score_launch(h, p.kernel == PIO_ALS_PATH_COS_BATCHED ? score_cos_topk_batched_kernel : score_cos_topk_kernel,
                        c.grid, dim3(p.threads), p.smem, p.kernel, h->I.F, h->I.n_internal, KP, k, (const float*)d_qc,
                        (const int*)d_q, nq, nqv, h->I.cand_ext, f.mask, f.weight, c.bound, keep_query, c.pk, c.cand);
  });
  if (rc) return rc;
  int cnt = 0;
  rc = deliver(h, o, 1, topk, out_items, out_scores, &cnt);
  if (rc) return rc;
  if (out_count) *out_count = cnt;
  return PIO_ALS_OK;
}
}  // namespace pio

extern "C" {

// Scoring passes: at most TK_MAXK results per pass; a query asking for more runs further passes, each bounded by the last
// result of the one before (topk.cuh below_bound).
int pio_als_recommend(pio_als_handle* h, const int32_t* users, int n, int topk, const uint8_t* item_mask,
                      const double* item_weight, int32_t* out_items, float* out_scores, int32_t* out_count) {
  if (!h) return PIO_ALS_ERR_ARG;
  std::lock_guard<std::mutex> lk(h->mu);
  h->st.last_score_path = 0;   // also for a call that launches nothing
  if (n < 0 || topk < 1) return fail(h, PIO_ALS_ERR_ARG, "topk must be >= 1 and n >= 0");
  if (n == 0) return PIO_ALS_OK;
  if (!users || !out_items || !out_scores) return fail(h, PIO_ALS_ERR_ARG, "null argument");
  if (!h->U.F || !h->I.F || !h->I.cand_ext) return fail(h, PIO_ALS_ERR_STATE, "no model");
  CK(h, cudaSetDevice(h->cfg.device));
  const ScorePlan p = plan_recommend(score_env(h), n, topk);
  if (p.route == ROUTE_ONE)   // the serving case: one query, one launch
    return serve_one(h, p, false, users, 1, topk, item_mask, item_weight, 0, out_items, out_scores, out_count);
  if (p.route == ROUTE_ARENA)   // a few queries
    return recommend_small(h, p, users, n, topk, item_mask, item_weight, out_items, out_scores, out_count);
  cudaStream_t st = h->stream;
  const int KP = h->KP;
  Scratch tmp(h);
  int* d_users = nullptr;
  float* d_xq = nullptr;
  uint8_t* d_valid = nullptr;
  ScoreIdx* d_cand = nullptr;
  CK(h, tmp.alloc(&d_users, (size_t)n));
  CK(h, tmp.alloc(&d_xq, (size_t)n * KP));
  CK(h, tmp.alloc(&d_valid, (size_t)n));
  CK(h, tmp.alloc(&d_cand, (size_t)n * p.lists * p.pass_k));
  MergeOut o;
  int rc = alloc_results(h, tmp, n, topk, p.passes > 1, &o);
  if (rc) return rc;
  CK(h, cudaMemcpyAsync(d_users, users, sizeof(int) * n, cudaMemcpyHostToDevice, st));
  DevFilter f;
  rc = upload_filter(h, item_mask, item_weight, &tmp, 0, &f);
  if (rc) return rc;
  rc = score_launch(h, gather_rows_kernel, dim3(n), dim3(64), 0, 0, h->U.F, KP, (const int*)d_users, n, h->U.perm, h->U.deg,
                    h->U.n, d_xq, d_valid);
  if (rc) return rc;
  rc = run_passes(h, p, n, topk, d_cand, o, [&](const Chunk& c) { return launch_dot(h, p, c, d_xq, d_valid, f); });
  if (rc) return rc;
  return deliver(h, o, n, topk, out_items, out_scores, out_count);
}

int pio_als_similar_batch(pio_als_handle* h, const int64_t* q_ptr, const int32_t* q_items, int n_queries, int topk,
                          const uint8_t* item_mask, const double* item_weight, int flags, int32_t* out_items,
                          float* out_scores, int32_t* out_count) {
  if (!h) return PIO_ALS_ERR_ARG;
  std::lock_guard<std::mutex> lk(h->mu);
  h->st.last_score_path = 0;   // also for a call that launches nothing
  if (n_queries < 0 || topk < 1) return fail(h, PIO_ALS_ERR_ARG, "topk must be >= 1 and n_queries >= 0");
  if (n_queries == 0) return PIO_ALS_OK;
  if (!q_ptr || !out_items || !out_scores) return fail(h, PIO_ALS_ERR_ARG, "null argument");
  for (int j = 0; j < n_queries; ++j)
    if (q_ptr[j + 1] < q_ptr[j] || (q_ptr[j + 1] > q_ptr[j] && !q_items))
      return fail(h, PIO_ALS_ERR_ARG, "q_ptr must be non-decreasing offsets into q_items");
  if (!h->I.F || !h->I.cand_ext) return fail(h, PIO_ALS_ERR_STATE, "no model");
  CK(h, cudaSetDevice(h->cfg.device));
  const ScoreEnv env = score_env(h);
  const long long total = q_ptr[n_queries] - q_ptr[0];
  const ScorePlan p = plan_similar(env, n_queries, q_ptr[1] - q_ptr[0], total, topk);
  if (p.route == ROUTE_ONE)   // the serving case
    return serve_one(h, p, true, q_items + q_ptr[0], (int)(q_ptr[1] - q_ptr[0]), topk, item_mask, item_weight, flags,
                     out_items, out_scores, out_count);
  if (p.route == ROUTE_ARENA)
    return similar_small(h, p, q_items + q_ptr[0], (int)(q_ptr[1] - q_ptr[0]), topk, item_mask, item_weight, flags,
                         out_items, out_scores, out_count);
  cudaStream_t st = h->stream;
  Scratch tmp(h);
  DevFilter f;
  int rc = upload_filter(h, item_mask, item_weight, &tmp, 0, &f);
  if (rc) return rc;
  if (p.route == ROUTE_BATCH) {
    // all query item vectors in one gather; which of them own a factor decides the vector list of every query
    int* d_qid = nullptr;
    float* d_qf_all = nullptr;
    uint8_t* d_valid = nullptr;
    CK(h, tmp.alloc(&d_qid, (size_t)total));
    CK(h, tmp.alloc(&d_qf_all, (size_t)total * h->KP));
    CK(h, tmp.alloc(&d_valid, (size_t)total));
    CK(h, cudaMemcpyAsync(d_qid, q_items + q_ptr[0], sizeof(int) * total, cudaMemcpyHostToDevice, st));
    rc = score_launch(h, gather_rows_kernel, dim3((unsigned)total), dim3(64), 0, 0, h->I.F, h->KP, (const int*)d_qid,
                      (int)total, h->I.perm, h->I.deg, h->I.n, d_qf_all, d_valid);
    if (rc) return rc;
    std::vector<uint8_t> valid((size_t)total);
    CK(h, cudaMemcpyAsync(valid.data(), d_valid, (size_t)total, cudaMemcpyDeviceToHost, st));
    CK(h, cudaStreamSynchronize(st));
    std::vector<int> nvalid((size_t)n_queries, 0), q0;
    for (int j = 0; j < n_queries; ++j)
      for (long long t = q_ptr[j]; t < q_ptr[j + 1]; ++t) nvalid[j] += valid[(size_t)(t - q_ptr[0])] ? 1 : 0;
    const ScorePlan b = plan_similar_batch(env, nvalid, topk, &q0);
    if (b.route == ROUTE_BATCH)
      return similar_groups(h, b, q0, q_ptr, n_queries, topk, valid, d_qf_all, d_qid, f, flags, tmp, out_items, out_scores,
                            out_count);
  }
  for (int j = 0; j < n_queries; ++j) {   // S5: one query at a time
    int32_t cnt = 0;
    rc = similar_one(h, q_items + q_ptr[j], (int)(q_ptr[j + 1] - q_ptr[j]), topk, f, flags, out_items + (size_t)j * topk,
                     out_scores + (size_t)j * topk, &cnt);
    if (rc) return rc;
    if (out_count) out_count[j] = cnt;
  }
  CK(h, cudaStreamSynchronize(h->stream));
  return PIO_ALS_OK;
}

int pio_als_similar(pio_als_handle* h, const int32_t* query_items, int nq, int topk, const uint8_t* item_mask,
                    const double* item_weight, int flags, int32_t* out_items, float* out_scores, int32_t* out_count) {
  if (!h) return PIO_ALS_ERR_ARG;
  if (nq < 0) {
    std::lock_guard<std::mutex> lk(h->mu);
    h->st.last_score_path = 0;
    return fail(h, PIO_ALS_ERR_ARG, "nq < 0");
  }
  const int64_t ptr[2] = {0, nq};
  return pio_als_similar_batch(h, ptr, query_items, 1, topk, item_mask, item_weight, flags, out_items, out_scores, out_count);
}

// ---- persistence ------------------------------------------------------------------------------
struct ModelHeader {
  char magic[8];
  int32_t version, rank, implicit_prefs, n_users, n_items, reserved;
  double lambda, alpha;
};

int pio_als_save(pio_als_handle* h, const char* path) {
  if (!h || !path) return PIO_ALS_ERR_ARG;
  try {
    const size_t nu = h->cfg.n_users, ni = h->cfg.n_items, k = h->cfg.rank;
    std::vector<float> uf(nu * k), itf(ni * k);
    std::vector<uint8_t> uh(nu), ih(ni);
    int rc = pio_als_get_factors(h, uf.data(), itf.data(), uh.data(), ih.data());
    if (rc) return rc;
    FILE* f = fopen(path, "wb");
    if (!f) return fail(h, PIO_ALS_ERR_IO, "cannot open %s for writing", path);
    ModelHeader hd{};
    memcpy(hd.magic, "PIOALS01", 8);
    hd.version = 1;
    hd.rank = h->cfg.rank;
    hd.implicit_prefs = h->cfg.implicit_prefs;
    hd.n_users = h->cfg.n_users;
    hd.n_items = h->cfg.n_items;
    hd.lambda = h->cfg.lambda;
    hd.alpha = h->cfg.alpha;
    bool ok = fwrite(&hd, sizeof hd, 1, f) == 1 && fwrite(uh.data(), 1, nu, f) == nu && fwrite(ih.data(), 1, ni, f) == ni &&
              fwrite(uf.data(), sizeof(float), nu * k, f) == nu * k && fwrite(itf.data(), sizeof(float), ni * k, f) == ni * k;
    ok = (fclose(f) == 0) && ok;
    return ok ? PIO_ALS_OK : fail(h, PIO_ALS_ERR_IO, "short write to %s", path);
  } catch (const std::exception& e) {   // bad_alloc etc. must not cross the C boundary
    return fail(h, PIO_ALS_ERR_IO, "pio_als_save: %s", e.what());
  }
}

__global__ void load_side_kernel(const uint8_t* has, int n, int* perm, int* inv, uint32_t* deg, uint32_t* npos) {
  const int r = blockIdx.x * blockDim.x + threadIdx.x;
  if (r >= n) return;
  perm[r] = r;
  inv[r] = r;
  deg[r] = (!has || has[r]) ? 1u : 0u;
  npos[r] = deg[r];
}

int pio_als_model_import(const pio_als_config* cfg_in, const float* user_factors, const float* item_factors,
                         const uint8_t* user_has, const uint8_t* item_has, pio_als_handle** out) {
  if (!cfg_in || !out) return fail(nullptr, PIO_ALS_ERR_ARG, "null argument");
  *out = nullptr;
  if (!item_factors) return fail(nullptr, PIO_ALS_ERR_ARG, "item_factors is null");
  pio_als_config cfg = *cfg_in;
  cfg.world_size = 1;
  cfg.world_rank = 0;
  const bool item_only = cfg.n_users == 0 && !user_factors;
  if (item_only) cfg.n_users = 1;   // an item-only model (similarproduct) carries one factor-less placeholder user
  else if (!user_factors) return fail(nullptr, PIO_ALS_ERR_ARG, "user_factors is null but n_users > 0");
  pio_als_handle* h = nullptr;
  int rc = pio_als_create(&cfg, &h);
  if (rc) return rc;
  cudaStream_t st = h->stream;
  const size_t k = (size_t)cfg.rank;
  const uint8_t zero = 0;
  struct { Side* s; size_t n; const uint8_t* has; const float* fac; } jobs[2] = {
      {&h->U, (size_t)cfg.n_users, item_only ? &zero : user_has, user_factors}, {&h->I, (size_t)cfg.n_items, item_has, item_factors}};
  auto body = [&]() -> int {
    for (auto& j : jobs) {
      Side& s = *j.s;
      s.n = (int)j.n;
      s.R = s.n;
      s.n_internal = s.n;
      s.bits = ceil_log2((uint64_t)s.n);
      CK(h, dalloc(h, &s.perm, j.n)); CK(h, dalloc(h, &s.inv, j.n)); CK(h, dalloc(h, &s.deg, j.n));
      CK(h, dalloc(h, &s.npos, j.n)); CK(h, dalloc(h, &s.cand_ext, j.n));
      CK(h, dalloc(h, &s.F, j.n * (size_t)h->KP));
      Scratch tmp(h);
      uint8_t* dh = nullptr;
      float* dfac = nullptr;
      if (j.has) {
        CK(h, tmp.alloc(&dh, j.n));
        CK(h, cudaMemcpyAsync(dh, j.has, j.n, cudaMemcpyHostToDevice, st));
      }
      load_side_kernel<<<nblk(s.n, 256), 256, 0, st>>>(dh, s.n, s.perm, s.inv, s.deg, s.npos);
      LAUNCHED(h);
      if (j.fac) {
        CK(h, tmp.alloc(&dfac, j.n * k));
        CK(h, cudaMemcpyAsync(dfac, j.fac, sizeof(float) * j.n * k, cudaMemcpyHostToDevice, st));
        scatter_init_kernel<<<nblk((long long)s.n * h->KP, 256), 256, 0, st>>>(dfac, s.n, (int)k, h->KP, s.perm, s.deg, s.F);
        LAUNCHED(h);
      } else {
        CK(h, cudaMemsetAsync(s.F, 0, sizeof(float) * j.n * (size_t)h->KP, st));
      }
      cand_ext_kernel<<<nblk(s.n, 256), 256, 0, st>>>(s.inv, s.deg, s.n, s.cand_ext);
      LAUNCHED(h);
      CK(h, cudaStreamSynchronize(st));   // the host sources may go away after this call
    }
    return PIO_ALS_OK;
  };
  rc = body();
  if (rc) {
    g_create_error = h->err;
    pio_als_destroy(h);
    return rc;
  }
  h->trained = true;
  *out = h;
  return PIO_ALS_OK;
}

int pio_als_load(const char* path, int device, pio_als_handle** out) {
  if (!path || !out) return fail(nullptr, PIO_ALS_ERR_ARG, "null argument");
  *out = nullptr;
  FILE* f = fopen(path, "rb");
  if (!f) return fail(nullptr, PIO_ALS_ERR_IO, "cannot open %s", path);
  ModelHeader hd;
  if (fread(&hd, sizeof hd, 1, f) != 1 || memcmp(hd.magic, "PIOALS01", 8) != 0 || hd.version != 1) {
    fclose(f);
    return fail(nullptr, PIO_ALS_ERR_IO, "%s is not a PIOALS01 model file", path);
  }
  // a corrupt header must not turn into a huge allocation: check the fields and the file size first
  if (hd.rank < 1 || hd.rank > 128 || hd.n_users < 1 || hd.n_items < 1) {
    fclose(f);
    return fail(nullptr, PIO_ALS_ERR_IO, "%s: corrupt header (rank %d, %d users, %d items)", path, hd.rank, hd.n_users, hd.n_items);
  }
  const size_t nu = hd.n_users, ni = hd.n_items, k = hd.rank;
  const long long expect = (long long)sizeof hd + (long long)(nu + ni) + (long long)sizeof(float) * (long long)((nu + ni) * k);
  if (fseek(f, 0, SEEK_END) != 0 || ftell(f) != expect || fseek(f, (long)sizeof hd, SEEK_SET) != 0) {
    fclose(f);
    return fail(nullptr, PIO_ALS_ERR_IO, "%s is truncated or has trailing bytes (expected %lld bytes)", path, expect);
  }
  try {
    std::vector<float> uf(nu * k), itf(ni * k);
    std::vector<uint8_t> uh(nu), ih(ni);
    bool ok = fread(uh.data(), 1, nu, f) == nu && fread(ih.data(), 1, ni, f) == ni &&
              fread(uf.data(), sizeof(float), nu * k, f) == nu * k && fread(itf.data(), sizeof(float), ni * k, f) == ni * k;
    fclose(f);
    f = nullptr;
    if (!ok) return fail(nullptr, PIO_ALS_ERR_IO, "%s is truncated", path);
    pio_als_config cfg{};
    cfg.abi_version = PIO_ALS_ABI_VERSION;
    cfg.rank = hd.rank;
    cfg.implicit_prefs = hd.implicit_prefs;
    cfg.n_users = hd.n_users;
    cfg.n_items = hd.n_items;
    cfg.device = device;
    cfg.world_size = 1;
    cfg.lambda = hd.lambda;
    cfg.alpha = hd.alpha;
    return pio_als_model_import(&cfg, uf.data(), itf.data(), uh.data(), ih.data(), out);
  } catch (const std::exception& e) {
    if (f) fclose(f);
    return fail(nullptr, PIO_ALS_ERR_IO, "pio_als_load: %s", e.what());
  }
}

/* debug only (not in pio_als.h): copies the A/b dump of the last tensor-core half-step (rows in internal order) */
__attribute__((visibility("default"))) int pio_als_debug_dump(pio_als_handle* h, float* out, long long n_floats) {
  if (!h || !h->d_dbg) return PIO_ALS_ERR_STATE;
  cudaStreamSynchronize(h->stream);
  size_t n = h->dbg_rows * (tc::ASLOT + tc::KP);
  if ((size_t)n_floats < n) n = (size_t)n_floats;
  return cudaMemcpy(out, h->d_dbg, n * sizeof(float), cudaMemcpyDeviceToHost) == cudaSuccess ? PIO_ALS_OK : PIO_ALS_ERR_CUDA;
}

__attribute__((visibility("default"))) int pio_als_debug_timing(pio_als_handle* h, long long* out, long long n) {
  if (!h || !h->d_timing) return PIO_ALS_ERR_STATE;
  cudaStreamSynchronize(h->stream);
  size_t m = (size_t)h->sm_count * 16 * 8;
  if ((size_t)n < m) m = (size_t)n;
  return cudaMemcpy(out, h->d_timing, m * sizeof(long long), cudaMemcpyDeviceToHost) == cudaSuccess ? PIO_ALS_OK : PIO_ALS_ERR_CUDA;
}

#define CK0(call)                                                                                         \
  do {                                                                                                    \
    cudaError_t e_ = (call);                                                                              \
    if (e_ != cudaSuccess) return fail(nullptr, PIO_ALS_ERR_CUDA, "%s failed: %s", #call, cudaGetErrorString(e_)); \
  } while (0)

/* debug only (not in pio_als.h): the lockstep Cholesky of als_lockstep.cuh on n dense SPD systems (A: n x N x N
 * row-major, b: n x N; HOST buffers), N = 64 or 128; x = (A + ridge I)^-1 b.  reps > 1 repeats fill + solve for timing
 * (ms_out = device time of the launch).  Used by tests/test_gpu_lockstep.py and tools/bench_solver.py. */
extern "C++" {
template <int N>
__global__ void __launch_bounds__(32) lockstep_probe_kernel(const float* __restrict__ A, const float* __restrict__ b, int n,
                                                            float ridge, float* __restrict__ x, int reps, int* fail) {
  using LL = LsLayout<N>;
  constexpr int LANES = N / 4, NM = 32 / LANES;
  extern __shared__ __align__(16) float sm[];
  float* bvec = sm + NM * LL::STRIDE;
  float* colbuf = bvec + NM * 80 + (N > 64 ? N : 0);
  const int lane = threadIdx.x & 31, grp = lane / LANES;
  for (int base = blockIdx.x * NM; base < n; base += gridDim.x * NM) {
    for (int rep = 0; rep < reps; ++rep) {
      for (int m = 0; m < NM; ++m) {
        const int mi = base + m;
        float* slot = sm + m * LL::STRIDE;
        for (int o = lane; o < N * N; o += 32) {
          const int r = o / N, c = o % N;
          if (c <= r) slot[LL::at(r, c)] = mi < n ? A[(size_t)mi * N * N + o] : (r == c ? 1.f : 0.f);
        }
        for (int o = lane; o < N; o += 32) bvec[m * (N > 64 ? N : 80) + o] = mi < n ? b[(size_t)mi * N + o] : 0.f;
      }
      __syncwarp();
      const int mine = base + grp;
      chol_lockstep<N, false>(sm + grp * LL::STRIDE, bvec + grp * (N > 64 ? N : 80), nullptr, ridge, N, colbuf + grp * 80,
                              x + (size_t)(mine < n ? mine : 0) * N, mine < n, fail);
      __syncwarp();
    }
  }
}
}  // extern "C++"

__attribute__((visibility("default"))) int pio_als_debug_lockstep(int device, int N, int n, const float* A, const float* b,
                                                                  float ridge, float* x, int reps, float* ms_out,
                                                                  int* fail_out) {
  if ((N != 64 && N != 128) || n < 1 || !A || !b || !x) return PIO_ALS_ERR_ARG;
  CK0(cudaSetDevice(device));
  float *dA = nullptr, *db = nullptr, *dx = nullptr;
  int* dfail = nullptr;
  CK0(cudaMalloc((void**)&dA, sizeof(float) * (size_t)n * N * N));
  CK0(cudaMalloc((void**)&db, sizeof(float) * (size_t)n * N));
  CK0(cudaMalloc((void**)&dx, sizeof(float) * (size_t)n * N));
  CK0(cudaMalloc((void**)&dfail, sizeof(int)));
  CK0(cudaMemset(dfail, 0, sizeof(int)));
  CK0(cudaMemcpy(dA, A, sizeof(float) * (size_t)n * N * N, cudaMemcpyHostToDevice));
  CK0(cudaMemcpy(db, b, sizeof(float) * (size_t)n * N, cudaMemcpyHostToDevice));
  const int nm = N == 64 ? 2 : 1;
  const size_t smem = sizeof(float) * (size_t)(nm * (N == 64 ? LsLayout<64>::STRIDE : LsLayout<128>::STRIDE) + 2 * 80 + 2 * 80 + 256);
  cudaDeviceProp pr_;
  CK0(cudaGetDeviceProperties(&pr_, device));
  int grid = (n + nm - 1) / nm;
  const int cap = pr_.multiProcessorCount * (N == 64 ? 12 : 6);
  if (grid > cap) grid = cap;
  cudaEvent_t e0, e1;
  cudaEventCreate(&e0);
  cudaEventCreate(&e1);
  if (N == 64) {
    CK0(cudaFuncSetAttribute(lockstep_probe_kernel<64>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    CK0(cudaFuncSetAttribute(lockstep_probe_kernel<64>, cudaFuncAttributePreferredSharedMemoryCarveout, 100));
    cudaEventRecord(e0);
    lockstep_probe_kernel<64><<<grid, 32, smem>>>(dA, db, n, ridge, dx, reps < 1 ? 1 : reps, dfail);
  } else {
    CK0(cudaFuncSetAttribute(lockstep_probe_kernel<128>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    CK0(cudaFuncSetAttribute(lockstep_probe_kernel<128>, cudaFuncAttributePreferredSharedMemoryCarveout, 100));
    cudaEventRecord(e0);
    lockstep_probe_kernel<128><<<grid, 32, smem>>>(dA, db, n, ridge, dx, reps < 1 ? 1 : reps, dfail);
  }
  cudaEventRecord(e1);
  CK0(cudaDeviceSynchronize());
  float ms = 0.f;
  cudaEventElapsedTime(&ms, e0, e1);
  if (ms_out) *ms_out = ms;
  CK0(cudaMemcpy(x, dx, sizeof(float) * (size_t)n * N, cudaMemcpyDeviceToHost));
  if (fail_out) CK0(cudaMemcpy(fail_out, dfail, sizeof(int), cudaMemcpyDeviceToHost));
  cudaEventDestroy(e0);
  cudaEventDestroy(e1);
  cudaFree(dA); cudaFree(db); cudaFree(dx); cudaFree(dfail);
  return PIO_ALS_OK;
}

int pio_als_get_stats(const pio_als_handle* h, pio_als_stats* out) {
  if (!h || !out) return PIO_ALS_ERR_ARG;
  *out = h->st;
  return PIO_ALS_OK;
}

int pio_als_synth_ratings_device(int device, int32_t n_users, int32_t n_items, int64_t nnz, int64_t seed, int implicit,
                                 int64_t start, int32_t* d_user, int32_t* d_item, float* d_rating) {
  if (cudaSetDevice(device) != cudaSuccess) return fail(nullptr, PIO_ALS_ERR_CUDA, "cudaSetDevice(%d) failed", device);
  if (nnz <= 0) return PIO_ALS_OK;
  synth_kernel<<<nblk(nnz, 256), 256>>>(n_users, n_items, nnz, (uint64_t)seed, implicit, start, d_user, d_item, d_rating);
  cudaError_t e = cudaDeviceSynchronize();
  if (e != cudaSuccess) return fail(nullptr, PIO_ALS_ERR_CUDA, "synth kernel: %s", cudaGetErrorString(e));
  return PIO_ALS_OK;
}

// ---- string ids -> dense indices (BiMap.stringInt) ---------------------------------------------------------------------
// The pipeline of ids_encode.cuh over n strings already on the device, on stream st (pio_ids_encode, pio_events_fold):
// d_index[e] = dense index of string e in order of first occurrence; d_first (nullable, n entries) [id] = position of
// the first occurrence of id; *n_unique.  0 < n < 2^32.
static int ids_encode_device(const uint8_t* d_bytes, const long long* d_off, int64_t n, cudaStream_t st, int* d_index,
                             long long* d_first, int64_t* n_unique) {
  uint64_t *ka = nullptr, *kb = nullptr;
  uint32_t *va = nullptr, *vb = nullptr, *f1 = nullptr, *f2 = nullptr, *run_start = nullptr, *head = nullptr, *ishead = nullptr,
           *firstpos = nullptr, *isfirst = nullptr;
  std::vector<void*> owned;
  auto A = [&](void** p, size_t bytes_) -> cudaError_t {
    cudaError_t e = cudaMalloc(p, bytes_ ? bytes_ : 1);
    if (e == cudaSuccess) owned.push_back(*p);
    return e;
  };
  struct Guard {
    std::vector<void*>& v;
    cudaStream_t s;
    ~Guard() {
      cudaStreamSynchronize(s);
      for (void* q : v) cudaFree(q);
    }
  } guard{owned, st};
  CK0(A((void**)&ka, 8 * (size_t)n)); CK0(A((void**)&kb, 8 * (size_t)n));
  CK0(A((void**)&va, 4 * (size_t)n)); CK0(A((void**)&vb, 4 * (size_t)n));
  CK0(A((void**)&f1, 4 * (size_t)n)); CK0(A((void**)&f2, 4 * (size_t)n));
  CK0(A((void**)&run_start, 4 * (size_t)n)); CK0(A((void**)&head, 4 * (size_t)n)); CK0(A((void**)&ishead, 4 * (size_t)n));
  CK0(A((void**)&firstpos, 4 * (size_t)n)); CK0(A((void**)&isfirst, 4 * (size_t)n));
  uint64_t mask = ~0ull;
  if (const char* hb = getenv("PIO_IDS_HASH_BITS")) {   // tests: a short hash makes different strings collide on purpose
    const int b = atoi(hb);
    if (b >= 1 && b < 64) mask = (1ull << b) - 1ull;
  }
  ids_hash_kernel<<<nblk(n, 256), 256, 0, st>>>(d_bytes, d_off, n, ka, va, mask);
  bool in_b = false;
  CK0(radix_sort_pairs(ka, va, kb, vb, (size_t)n, 64, st, &in_b, nullptr));
  const uint64_t* ks = in_b ? kb : ka;
  const uint32_t* vs = in_b ? vb : va;
  ids_runflag_kernel<<<nblk(n, 256), 256, 0, st>>>(ks, n, f1);
  CK0(scan_exclusive_u32(f1, f1, (size_t)n, st, nullptr));                 // f1 = run ids
  ids_runstart_kernel<<<nblk(n, 256), 256, 0, st>>>(ks, f1, n, run_start);
  ids_head_kernel<<<nblk(n, 256), 256, 0, st>>>(ks, vs, f1, run_start, d_bytes, d_off, n, head, ishead);
  uint32_t last_flag = 0, last_ex = 0;
  CK0(cudaMemcpyAsync(&last_flag, ishead + n - 1, 4, cudaMemcpyDeviceToHost, st));
  CK0(scan_exclusive_u32(ishead, f2, (size_t)n, st, nullptr));             // f2 = group ids (valid at heads)
  CK0(cudaMemcpyAsync(&last_ex, f2 + n - 1, 4, cudaMemcpyDeviceToHost, st));
  CK0(cudaMemsetAsync(isfirst, 0, 4 * (size_t)n, st));
  ids_firstpos_kernel<<<nblk(n, 256), 256, 0, st>>>(vs, ishead, f2, n, firstpos, isfirst);
  CK0(scan_exclusive_u32(isfirst, isfirst, (size_t)n, st, nullptr));       // ids by first occurrence
  ids_assign_kernel<<<nblk(n, 256), 256, 0, st>>>(vs, head, isfirst, n, d_index, d_first);
  CK0(cudaGetLastError());
  CK0(cudaStreamSynchronize(st));
  *n_unique = (int64_t)last_ex + last_flag;
  return PIO_ALS_OK;
}

int pio_ids_encode(int device, const uint8_t* bytes, const int64_t* offsets, int64_t n, int32_t* out_index,
                   int64_t* out_first, int32_t* out_n_unique) {
  if (n < 0 || !offsets || !out_index || !out_n_unique || (n > 0 && !bytes && offsets[n] > offsets[0]))
    return fail(nullptr, PIO_ALS_ERR_ARG, "bad pio_ids_encode arguments");
  *out_n_unique = 0;
  if (n == 0) return PIO_ALS_OK;
  if (n >= (1ll << 32)) return fail(nullptr, PIO_ALS_ERR_ARG, "n must be < 2^32");
  if (offsets[0] != 0) return fail(nullptr, PIO_ALS_ERR_ARG, "offsets[0] must be 0");
  CK0(cudaSetDevice(device));
  const size_t nb = (size_t)offsets[n];
  uint8_t* d_bytes = nullptr;
  long long *d_off = nullptr, *d_first = nullptr;
  int* d_out = nullptr;
  std::vector<void*> owned;
  auto A = [&](void** p, size_t bytes_) -> cudaError_t {
    cudaError_t e = cudaMalloc(p, bytes_ ? bytes_ : 1);
    if (e == cudaSuccess) owned.push_back(*p);
    return e;
  };
  struct Guard { std::vector<void*>& v; ~Guard() { for (void* q : v) cudaFree(q); } } guard{owned};
  CK0(A((void**)&d_bytes, nb));
  CK0(A((void**)&d_off, sizeof(long long) * (n + 1)));
  CK0(A((void**)&d_out, 4 * (size_t)n));
  CK0(A((void**)&d_first, 8 * (size_t)n));
  cudaStream_t st = 0;
  CK0(cudaMemcpyAsync(d_bytes, bytes, nb, cudaMemcpyHostToDevice, st));
  CK0(cudaMemcpyAsync(d_off, offsets, sizeof(long long) * (n + 1), cudaMemcpyHostToDevice, st));
  int64_t nuniq = 0;
  const int rc = ids_encode_device(d_bytes, d_off, n, st, d_out, out_first ? d_first : nullptr, &nuniq);
  if (rc != PIO_ALS_OK) return rc;
  CK0(cudaMemcpy(out_index, d_out, 4 * (size_t)n, cudaMemcpyDeviceToHost));
  if (out_first) CK0(cudaMemcpy(out_first, d_first, 8 * (size_t)nuniq, cudaMemcpyDeviceToHost));
  *out_n_unique = (int32_t)nuniq;
  return PIO_ALS_OK;
}

// ---- event file scan (PEventStore.findColumns; events_scan.cuh) --------------------------------------------------------
// Where the time of the last pio_events_scan on this thread went, summed over its chunks (pio_events_debug_timing).
struct EvTiming {
  double h2d_ms, kernel_ms, d2h_ms, stage_ms;   // device times (CUDA events); stage: host copy into pinned memory
  int64_t chunks;
};
static thread_local EvTiming g_ev_timing;
static_assert(PIO_EVENTS_MIN_EVENT_BYTES <= ev::MIN_MATCHED_BYTES, "capacity bound of pio_events_scan");

// End of the device chunk that starts at b: after the last terminator in [b, b + cap), never between the "\r" and "\n"
// of a CRLF; b when [b, b + cap) holds no usable terminator (the line at b is longer than a chunk).
static int64_t ev_cut(const uint8_t* t, int64_t n, int64_t b, int64_t cap) {
  if (n - b <= cap) return n;
  const int64_t lim = b + cap;
  for (int64_t p = lim - 1; p >= b; --p) {
    if (t[p] == '\n') return p + 1;
    if (t[p] == '\r' && t[p + 1] != '\n') return p + 1;   // p + 1 <= lim < n
  }
  return b;
}

// the tracked keys of pio_events_scan_keys and where their columns go (host buffers)
struct EvKeyArgs {
  const char* const* keys;
  int n;
  uint8_t* out_present;
  uint8_t* out_number;
  double* out_num;
  uint8_t* out_tok_bytes;
  int64_t* out_tok_off;
};

// pio_events_scan (ka == nullptr) and pio_events_scan_keys: one chunk loop, the kernels instantiated with KEYS = ka != 0
static int events_scan_impl(int device, const uint8_t* text, int64_t n_bytes, const pio_events_filter* f,
                            int64_t capacity, int64_t* out_line, int32_t* out_code, double* out_value, uint8_t* out_flags,
                            int64_t* out_time_us, uint8_t* out_eid_bytes, int64_t* out_eid_off, uint8_t* out_tid_bytes,
                            int64_t* out_tid_off, int64_t* out_n_events, int64_t fb_capacity, int64_t* out_fb_line,
                            int64_t* out_fb_begin, int64_t* out_fb_end, int64_t* out_n_fallback, int64_t* out_n_lines,
                            const EvKeyArgs* ka) {
  if (n_bytes < 0 || (n_bytes > 0 && !text) || !f || capacity < n_bytes / PIO_EVENTS_MIN_EVENT_BYTES + 1 ||
      fb_capacity < 0 || !out_line || !out_code || !out_value || !out_flags || !out_time_us || !out_eid_bytes ||
      !out_eid_off || !out_tid_bytes || !out_tid_off || !out_n_events || (fb_capacity > 0 && (!out_fb_line ||
      !out_fb_begin || !out_fb_end)) || !out_n_fallback || !out_n_lines)
    return fail(nullptr, PIO_ALS_ERR_ARG, "bad pio_events_scan arguments");
  if (f->n_event_names < 0 || (f->n_event_names > 0 && !f->event_names))
    return fail(nullptr, PIO_ALS_ERR_ARG, "bad event name list");
  for (int k = 0; k < f->n_event_names; ++k)
    if (!f->event_names[k]) return fail(nullptr, PIO_ALS_ERR_ARG, "event name %d is NULL", k);
  if (f->target_entity_type_mode < PIO_EVENTS_TARGET_ANY || f->target_entity_type_mode > PIO_EVENTS_TARGET_EQUALS ||
      (f->target_entity_type_mode == PIO_EVENTS_TARGET_EQUALS && !f->target_entity_type))
    return fail(nullptr, PIO_ALS_ERR_ARG, "bad target_entity_type_mode / target_entity_type");
  const int nk = ka ? ka->n : 0;
  *out_n_events = *out_n_fallback = *out_n_lines = 0;
  out_eid_off[0] = out_tid_off[0] = 0;
  if (ka) ka->out_tok_off[0] = 0;
  if (n_bytes == 0) return PIO_ALS_OK;
  CK0(cudaSetDevice(device));

  // the filter's strings, packed: entity type | target entity type | property | names...
  std::vector<uint8_t> fbytes;
  auto put = [&](const char* s) -> int {
    const size_t at = fbytes.size();
    fbytes.insert(fbytes.end(), s, s + strlen(s));
    return (int)at;
  };
  const int at_et = f->entity_type ? put(f->entity_type) : 0;
  const int len_et = f->entity_type ? (int)(fbytes.size() - at_et) : -1;
  const int at_tt = f->target_entity_type_mode == PIO_EVENTS_TARGET_EQUALS ? put(f->target_entity_type) : 0;
  const int len_tt = (int)fbytes.size() - at_tt;
  const int at_pr = f->property ? put(f->property) : 0;
  const int len_pr = f->property ? (int)(fbytes.size() - at_pr) : -1;
  std::vector<int> noff(1, (int)fbytes.size());
  for (int k = 0; k < f->n_event_names; ++k) {
    put(f->event_names[k]);
    noff.push_back((int)fbytes.size());
  }
  std::vector<int> koff(1, (int)fbytes.size());   // then the tracked keys
  for (int q = 0; q < nk; ++q) {
    put(ka->keys[q]);
    koff.push_back((int)fbytes.size());
  }

  int64_t cap = 64ll << 20;   // device chunk; PIO_EVENTS_DEVICE_CHUNK (bytes) lets tests straddle its boundaries
  if (const char* c = getenv("PIO_EVENTS_DEVICE_CHUNK")) {
    const long long v = atoll(c);
    if (v >= 1 && v <= (1ll << 30)) cap = v;
  }
  if (cap > n_bytes) cap = n_bytes;

  std::vector<void*> owned, pinned;
  cudaStream_t streams[2] = {nullptr, nullptr};
  // copy begin / end per staging slot, then on the scan stream: kernels before and after the line count, and the
  // device-to-host copies (pio_events_debug_timing)
  cudaEvent_t evs[10] = {};
  cudaEvent_t *h2d_begin = evs, *copied = evs + 2, &k0 = evs[4], &k1 = evs[5], &k2 = evs[6], &k3 = evs[7],
              &d0 = evs[8], &d1 = evs[9];
  struct Guard {
    std::vector<void*>& d;
    std::vector<void*>& p;
    cudaStream_t* s;
    cudaEvent_t* e;
    ~Guard() {
      for (int k = 0; k < 2; ++k)
        if (s[k]) cudaStreamSynchronize(s[k]);
      for (void* q : d) cudaFree(q);
      for (void* q : p) cudaFreeHost(q);
      for (int k = 0; k < 2; ++k)
        if (s[k]) cudaStreamDestroy(s[k]);
      for (int k = 0; k < 10; ++k)
        if (e[k]) cudaEventDestroy(e[k]);
    }
  } guard{owned, pinned, streams, evs};
  auto A = [&](void** p, size_t bytes_) -> cudaError_t {
    cudaError_t e = cudaMalloc(p, bytes_ ? bytes_ : 1);
    if (e == cudaSuccess) owned.push_back(*p);
    return e;
  };
  auto P = [&](void** p, size_t bytes_) -> cudaError_t {
    cudaError_t e = cudaHostAlloc(p, bytes_ ? bytes_ : 1, cudaHostAllocDefault);
    if (e == cudaSuccess) pinned.push_back(*p);
    return e;
  };
  for (int k = 0; k < 2; ++k) CK0(cudaStreamCreateWithFlags(&streams[k], cudaStreamNonBlocking));
  for (cudaEvent_t& e : evs) CK0(cudaEventCreate(&e));
  EvTiming& tm = g_ev_timing;
  tm = EvTiming{};
  bool use_smem = true;   // PIO_EVENTS_SMEM=0: the parse reads its lines from global memory (A/B measurements)
  if (const char* c = getenv("PIO_EVENTS_SMEM")) use_smem = atoi(c) != 0;
  if (use_smem)
    CK0(cudaFuncSetAttribute(ka ? ev_parse_smem_kernel<true> : ev_parse_smem_kernel<false>,
                             cudaFuncAttributeMaxDynamicSharedMemorySize, EV_SMEM_BYTES));
  cudaStream_t ex = streams[0], cp = streams[1];   // scan, host-to-device copies
  uint8_t *d_text[2] = {nullptr, nullptr}, *stage[2] = {nullptr, nullptr}, *d_scratch = nullptr, *d_fbytes = nullptr;
  uint32_t *d_flag = nullptr, *d_lid = nullptr, *d_tot = nullptr, *h_tot = nullptr;
  int *d_noff = nullptr, *d_koff = nullptr;
  for (int k = 0; k < 2; ++k) {
    CK0(A((void**)&d_text[k], (size_t)cap));
    CK0(P((void**)&stage[k], (size_t)cap));
  }
  CK0(A((void**)&d_scratch, (size_t)cap));
  CK0(A((void**)&d_flag, 4 * (size_t)cap));
  CK0(A((void**)&d_lid, 4 * (size_t)cap));
  CK0(A((void**)&d_fbytes, fbytes.size()));
  CK0(A((void**)&d_noff, sizeof(int) * noff.size()));
  CK0(A((void**)&d_tot, 4 * sizeof(uint32_t)));
  CK0(P((void**)&h_tot, 8 * sizeof(uint32_t)));
  if (!fbytes.empty()) CK0(cudaMemcpy(d_fbytes, fbytes.data(), fbytes.size(), cudaMemcpyHostToDevice));
  CK0(cudaMemcpy(d_noff, noff.data(), sizeof(int) * noff.size(), cudaMemcpyHostToDevice));
  CK0(A((void**)&d_koff, sizeof(int) * koff.size()));
  CK0(cudaMemcpy(d_koff, koff.data(), sizeof(int) * koff.size(), cudaMemcpyHostToDevice));
  ev::Filter df;
  df.entity_type = d_fbytes + at_et;
  df.entity_type_len = len_et;
  df.names = d_fbytes;
  df.name_off = d_noff;
  df.n_names = f->event_names ? f->n_event_names : -1;   // NULL: any name; an empty list: none
  df.target_mode = f->target_entity_type_mode;
  df.target = d_fbytes + at_tt;
  df.target_len = len_tt;
  df.prop = d_fbytes + at_pr;
  df.prop_len = len_pr;
  df.has_start = f->has_start != 0;
  df.has_until = f->has_until != 0;
  df.start_us = f->start_us;
  df.until_us = f->until_us;

  EvKeys K{};
  K.list.names = d_fbytes;
  K.list.off = d_koff;
  K.list.n = nk;

  EvBase base{0, 0, 0, 0};
  int64_t n_ev = 0, n_fb = 0, n_tok = 0;   // n_tok: token bytes so far   // n_fb counts every fallback line, also those beyond fb_capacity
  // lines longer than a chunk, found while cutting the next chunk: written after the current chunk's fallback lines so
  // that the fallback list stays in line order
  std::vector<int64_t> oversized;
  auto flush_oversized = [&]() {
    for (size_t k = 0; k < oversized.size(); k += 3) {
      if (n_fb < fb_capacity)
        out_fb_line[n_fb] = oversized[k], out_fb_begin[n_fb] = oversized[k + 1], out_fb_end[n_fb] = oversized[k + 2];
      ++n_fb;
    }
    oversized.clear();
  };
  // stage a chunk: host copy into pinned memory, then an asynchronous copy on cp.  The loop below calls it for chunk
  // k + 1 after it has launched the parse of chunk k, so that both copies run while the device parses.
  auto prefetch = [&](int slot, int64_t b, int64_t e) -> int {
    const auto h0 = std::chrono::steady_clock::now();
    memcpy(stage[slot], text + b, (size_t)(e - b));
    tm.stage_ms += std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now() - h0).count();
    CK0(cudaEventRecord(h2d_begin[slot], cp));
    CK0(cudaMemcpyAsync(d_text[slot], stage[slot], (size_t)(e - b), cudaMemcpyHostToDevice, cp));
    CK0(cudaEventRecord(copied[slot], cp));
    return PIO_ALS_OK;
  };
  auto ms = [](cudaEvent_t a, cudaEvent_t b) {
    float v = 0.f;
    cudaEventElapsedTime(&v, a, b);
    return (double)v;
  };
  // the next chunk [b, e) at or after pos; lines longer than a chunk become fallback lines on the way
  auto next_chunk = [&](int64_t pos, int64_t* b, int64_t* e) {
    for (;;) {
      if (pos >= n_bytes) {
        *b = *e = n_bytes;
        return;
      }
      const int64_t c = ev_cut(text, n_bytes, pos, cap);
      if (c > pos) {
        *b = pos, *e = c;
        return;
      }
      int64_t q = pos;   // a line longer than a chunk: the host parses it
      while (q < n_bytes && text[q] != '\n' && text[q] != '\r') ++q;
      oversized.insert(oversized.end(), {base.line, pos, q});
      ++base.line;
      if (q < n_bytes && text[q] == '\r' && q + 1 < n_bytes && text[q + 1] == '\n') ++q;
      pos = q < n_bytes ? q + 1 : q;
    }
  };

  int64_t cb, ce;
  next_chunk(0, &cb, &ce);
  flush_oversized();
  if (cb < ce && prefetch(0, cb, ce) != PIO_ALS_OK) return PIO_ALS_ERR_CUDA;
  for (int slot = 0; cb < ce; slot ^= 1) {
    const long long L = ce - cb;
    base.byte = cb;
    CK0(cudaStreamWaitEvent(ex, copied[slot], 0));
    const uint8_t* t = d_text[slot];
    CK0(cudaEventRecord(k0, ex));
    ev_start_flag_kernel<<<nblk(L, EV_THREADS), EV_THREADS, 0, ex>>>(t, L, d_flag);
    CK0(scan_exclusive_u32(d_flag, d_lid, (size_t)L, ex, nullptr));
    CK0(cudaMemcpyAsync(h_tot + 4, d_flag + L - 1, 4, cudaMemcpyDeviceToHost, ex));
    CK0(cudaMemcpyAsync(h_tot + 5, d_lid + L - 1, 4, cudaMemcpyDeviceToHost, ex));
    CK0(cudaEventRecord(k1, ex));
    CK0(cudaStreamSynchronize(ex));
    const long long nl = (long long)h_tot[4] + h_tot[5];
    const EvBase here = base;
    base.line += nl;

    std::vector<void*> chunk_mem;
    struct ChunkGuard {
      std::vector<void*>& v;
      cudaStream_t s;
      ~ChunkGuard() { for (void* q : v) cudaFreeAsync(q, s); }
    } chunk_guard{chunk_mem, ex};
    auto CA = [&](void** p, size_t bytes_) -> cudaError_t {
      cudaError_t e = cudaMallocAsync(p, bytes_ ? bytes_ : 1, ex);
      if (e == cudaSuccess) chunk_mem.push_back(*p);
      return e;
    };
    uint32_t* starts = nullptr;
    EvLines Ls;
    EvOut o;
    const size_t nls = (size_t)nl;
    CK0(CA((void**)&starts, 4 * (nls + 1)));
    uint32_t** u32s[8] = {&Ls.is_match, &Ls.is_fb, &Ls.eid_len, &Ls.tid_len, &Ls.match_pos, &Ls.fb_pos, &Ls.eid_pos,
                          &Ls.tid_pos};
    for (uint32_t** p : u32s) CK0(CA((void**)p, 4 * nls));
    CK0(CA((void**)&Ls.code, 4 * nls));
    CK0(CA((void**)&Ls.value, 8 * nls));
    CK0(CA((void**)&Ls.time_us, 8 * nls));
    CK0(CA((void**)&Ls.flags, nls));
    CK0(CA((void**)&o.line, 8 * nls));
    CK0(CA((void**)&o.code, 4 * nls));
    CK0(CA((void**)&o.value, 8 * nls));
    CK0(CA((void**)&o.flags, nls));
    CK0(CA((void**)&o.time_us, 8 * nls));
    CK0(CA((void**)&o.eid_off, 8 * nls));
    CK0(CA((void**)&o.tid_off, 8 * nls));
    CK0(CA((void**)&o.fb_line, 8 * nls));
    CK0(CA((void**)&o.fb_begin, 8 * nls));
    CK0(CA((void**)&o.fb_end, 8 * nls));
    CK0(CA((void**)&o.eid_bytes, (size_t)L));
    CK0(CA((void**)&o.tid_bytes, (size_t)L));
    if (ka) {
      const size_t nlk = nls * (size_t)nk;
      CK0(CA((void**)&K.present, nls));
      CK0(CA((void**)&K.number, nls));
      CK0(CA((void**)&K.num, 8 * nlk));
      CK0(CA((void**)&K.tok_b, 4 * nlk));
      CK0(CA((void**)&K.tok_e, 4 * nlk));
      CK0(CA((void**)&K.tok_len, 4 * nls));
      CK0(CA((void**)&K.tok_pos, 4 * nls));
      CK0(CA((void**)&K.o_present, nls));
      CK0(CA((void**)&K.o_number, nls));
      CK0(CA((void**)&K.o_num, 8 * nlk));
      CK0(CA((void**)&K.o_tok_off, 8 * nlk));
      CK0(CA((void**)&K.o_tok, (size_t)L));   // tokens are disjoint pieces of the chunk's text
      K.tok_base = n_tok;
    }
    CK0(cudaEventRecord(k2, ex));
    ev_start_scatter_kernel<<<nblk(L, EV_THREADS), EV_THREADS, 0, ex>>>(d_flag, d_lid, L, nl, starts);
    const unsigned gl = nblk(nl, EV_THREADS);
    if (use_smem && ka)
      ev_parse_smem_kernel<true><<<gl, EV_THREADS, EV_SMEM_BYTES, ex>>>(t, starts, nl, df, d_scratch, Ls, K);
    else if (use_smem)
      ev_parse_smem_kernel<false><<<gl, EV_THREADS, EV_SMEM_BYTES, ex>>>(t, starts, nl, df, d_scratch, Ls, K);
    else if (ka)
      ev_parse_kernel<true><<<gl, EV_THREADS, 0, ex>>>(t, starts, nl, df, d_scratch, Ls, K);
    else
      ev_parse_kernel<false><<<gl, EV_THREADS, 0, ex>>>(t, starts, nl, df, d_scratch, Ls, K);
    CK0(cudaGetLastError());
    CK0(scan_exclusive_u32(Ls.is_match, Ls.match_pos, nls, ex, nullptr));
    CK0(scan_exclusive_u32(Ls.is_fb, Ls.fb_pos, nls, ex, nullptr));
    CK0(scan_exclusive_u32(Ls.eid_len, Ls.eid_pos, nls, ex, nullptr));
    CK0(scan_exclusive_u32(Ls.tid_len, Ls.tid_pos, nls, ex, nullptr));
    if (ka) CK0(scan_exclusive_u32(K.tok_len, K.tok_pos, nls, ex, nullptr));
    EvBase cb_{here.line, here.byte, base.eid, base.tid};
    if (ka)
      ev_compact_kernel<true><<<gl, EV_THREADS, 0, ex>>>(t, starts, nl, cb_, d_scratch, Ls, o, K);
    else
      ev_compact_kernel<false><<<gl, EV_THREADS, 0, ex>>>(t, starts, nl, cb_, d_scratch, Ls, o, K);
    ev_totals_kernel<<<1, 1, 0, ex>>>(Ls, nl, d_tot);
    CK0(cudaGetLastError());
    CK0(cudaEventRecord(k3, ex));
    CK0(cudaMemcpyAsync(h_tot, d_tot, 4 * sizeof(uint32_t), cudaMemcpyDeviceToHost, ex));
    if (ka) {   // token bytes of the chunk: last exclusive position + last length
      CK0(cudaMemcpyAsync(h_tot + 6, K.tok_pos + nl - 1, 4, cudaMemcpyDeviceToHost, ex));
      CK0(cudaMemcpyAsync(h_tot + 7, K.tok_len + nl - 1, 4, cudaMemcpyDeviceToHost, ex));
    }
    // find and stage the next chunk while this one is parsed (oversized lines before it belong after this chunk's
    // lines, so their line numbers are assigned only now that this chunk's line count is known)
    int64_t nb, ne;
    next_chunk(ce, &nb, &ne);
    if (nb < ne && prefetch(slot ^ 1, nb, ne) != PIO_ALS_OK) return PIO_ALS_ERR_CUDA;
    CK0(cudaStreamSynchronize(ex));
    const int64_t nm = h_tot[0], nf = h_tot[1], eb = h_tot[2], tb = h_tot[3];
    if (n_ev + nm > capacity) return fail(nullptr, PIO_ALS_ERR_ARG, "more matched events than capacity");
    CK0(cudaEventRecord(d0, ex));
    CK0(cudaMemcpyAsync(out_line + n_ev, o.line, 8 * nm, cudaMemcpyDeviceToHost, ex));
    CK0(cudaMemcpyAsync(out_code + n_ev, o.code, 4 * nm, cudaMemcpyDeviceToHost, ex));
    CK0(cudaMemcpyAsync(out_value + n_ev, o.value, 8 * nm, cudaMemcpyDeviceToHost, ex));
    CK0(cudaMemcpyAsync(out_flags + n_ev, o.flags, nm, cudaMemcpyDeviceToHost, ex));
    CK0(cudaMemcpyAsync(out_time_us + n_ev, o.time_us, 8 * nm, cudaMemcpyDeviceToHost, ex));
    CK0(cudaMemcpyAsync(out_eid_off + n_ev, o.eid_off, 8 * nm, cudaMemcpyDeviceToHost, ex));
    CK0(cudaMemcpyAsync(out_tid_off + n_ev, o.tid_off, 8 * nm, cudaMemcpyDeviceToHost, ex));
    CK0(cudaMemcpyAsync(out_eid_bytes + base.eid, o.eid_bytes, eb, cudaMemcpyDeviceToHost, ex));
    CK0(cudaMemcpyAsync(out_tid_bytes + base.tid, o.tid_bytes, tb, cudaMemcpyDeviceToHost, ex));
    int64_t tk = 0;
    if (ka) {
      tk = (int64_t)h_tot[6] + h_tot[7];
      CK0(cudaMemcpyAsync(ka->out_present + n_ev, K.o_present, nm, cudaMemcpyDeviceToHost, ex));
      CK0(cudaMemcpyAsync(ka->out_number + n_ev, K.o_number, nm, cudaMemcpyDeviceToHost, ex));
      CK0(cudaMemcpyAsync(ka->out_num + n_ev * nk, K.o_num, 8 * nm * nk, cudaMemcpyDeviceToHost, ex));
      CK0(cudaMemcpyAsync(ka->out_tok_off + n_ev * nk, K.o_tok_off, 8 * nm * nk, cudaMemcpyDeviceToHost, ex));
      CK0(cudaMemcpyAsync(ka->out_tok_bytes + n_tok, K.o_tok, tk, cudaMemcpyDeviceToHost, ex));
    }
    const int64_t room = fb_capacity - n_fb, nfc = nf < room ? nf : (room > 0 ? room : 0);
    if (nfc > 0) {
      CK0(cudaMemcpyAsync(out_fb_line + n_fb, o.fb_line, 8 * nfc, cudaMemcpyDeviceToHost, ex));
      CK0(cudaMemcpyAsync(out_fb_begin + n_fb, o.fb_begin, 8 * nfc, cudaMemcpyDeviceToHost, ex));
      CK0(cudaMemcpyAsync(out_fb_end + n_fb, o.fb_end, 8 * nfc, cudaMemcpyDeviceToHost, ex));
    }
    CK0(cudaEventRecord(d1, ex));
    CK0(cudaStreamSynchronize(ex));
    tm.h2d_ms += ms(h2d_begin[slot], copied[slot]);
    tm.kernel_ms += ms(k0, k1) + ms(k2, k3);
    tm.d2h_ms += ms(d0, d1);
    ++tm.chunks;
    n_ev += nm;
    n_fb += nf;
    base.eid += eb;
    base.tid += tb;
    n_tok += tk;
    flush_oversized();
    cb = nb, ce = ne;
  }
  out_eid_off[n_ev] = base.eid;
  out_tid_off[n_ev] = base.tid;
  if (ka) ka->out_tok_off[n_ev * nk] = n_tok;
  *out_n_events = n_ev;
  *out_n_fallback = n_fb;
  *out_n_lines = base.line;
  return PIO_ALS_OK;
}

int pio_events_scan(int device, const uint8_t* text, int64_t n_bytes, const pio_events_filter* f, int64_t capacity,
                    int64_t* out_line, int32_t* out_code, double* out_value, uint8_t* out_flags, int64_t* out_time_us,
                    uint8_t* out_eid_bytes, int64_t* out_eid_off, uint8_t* out_tid_bytes, int64_t* out_tid_off,
                    int64_t* out_n_events, int64_t fb_capacity, int64_t* out_fb_line, int64_t* out_fb_begin,
                    int64_t* out_fb_end, int64_t* out_n_fallback, int64_t* out_n_lines) {
  return events_scan_impl(device, text, n_bytes, f, capacity, out_line, out_code, out_value, out_flags, out_time_us,
                          out_eid_bytes, out_eid_off, out_tid_bytes, out_tid_off, out_n_events, fb_capacity, out_fb_line,
                          out_fb_begin, out_fb_end, out_n_fallback, out_n_lines, nullptr);
}

int pio_events_scan_keys(int device, const uint8_t* text, int64_t n_bytes, const pio_events_filter* f,
                         const char* const* keys, int n_keys, int64_t capacity, int64_t* out_line, int32_t* out_code,
                         double* out_value, uint8_t* out_flags, int64_t* out_time_us, uint8_t* out_eid_bytes,
                         int64_t* out_eid_off, uint8_t* out_tid_bytes, int64_t* out_tid_off, uint8_t* out_present,
                         uint8_t* out_number, double* out_num, uint8_t* out_tok_bytes, int64_t* out_tok_off,
                         int64_t* out_n_events, int64_t fb_capacity, int64_t* out_fb_line, int64_t* out_fb_begin,
                         int64_t* out_fb_end, int64_t* out_n_fallback, int64_t* out_n_lines) {
  if (n_keys < 1 || n_keys > ev::MAX_KEYS || !keys || !out_present || !out_number || !out_num || !out_tok_bytes ||
      !out_tok_off)
    return fail(nullptr, PIO_ALS_ERR_ARG, "bad pio_events_scan_keys arguments (n_keys must be 1..%d)", ev::MAX_KEYS);
  if (!f || f->property)
    return fail(nullptr, PIO_ALS_ERR_ARG, "pio_events_scan_keys: filter->property must be NULL");
  for (int q = 0; q < n_keys; ++q) {
    if (!keys[q] || !keys[q][0]) return fail(nullptr, PIO_ALS_ERR_ARG, "key %d is NULL or empty", q);
    for (int p = 0; p < q; ++p)
      if (!strcmp(keys[p], keys[q])) return fail(nullptr, PIO_ALS_ERR_ARG, "key %d repeats key %d", q, p);
  }
  const EvKeyArgs ka{keys, n_keys, out_present, out_number, out_num, out_tok_bytes, out_tok_off};
  return events_scan_impl(device, text, n_bytes, f, capacity, out_line, out_code, out_value, out_flags, out_time_us,
                          out_eid_bytes, out_eid_off, out_tid_bytes, out_tid_off, out_n_events, fb_capacity, out_fb_line,
                          out_fb_begin, out_fb_end, out_n_fallback, out_n_lines, &ka);
}

// ---- $set / $unset / $delete fold (PEventStore.aggregatePropertyColumns; events_fold.cuh) -----------------------------
int pio_events_fold(int device, const uint8_t* eid_bytes, const int64_t* eid_off, const int32_t* code,
                    const int64_t* time_us, const uint8_t* present, int64_t n, int n_keys, int64_t* out_first_event,
                    uint8_t* out_exists, int64_t* out_first_us, int64_t* out_last_us, int64_t* out_winner,
                    int64_t* out_n_entities) {
  if (n < 0 || n_keys < 0 || n_keys > ev::MAX_KEYS || !eid_off || !out_n_entities || (n > 0 && (!code || !time_us ||
      !out_first_event || !out_exists || !out_first_us || !out_last_us || (n_keys > 0 && (!present || !out_winner)) ||
      (!eid_bytes && eid_off[n] > eid_off[0]))))
    return fail(nullptr, PIO_ALS_ERR_ARG, "bad pio_events_fold arguments (n_keys must be 0..%d)", ev::MAX_KEYS);
  *out_n_entities = 0;
  if (n == 0) return PIO_ALS_OK;
  if (n >= (1ll << 31)) return fail(nullptr, PIO_ALS_ERR_ARG, "n must be < 2^31");
  if (eid_off[0] != 0) return fail(nullptr, PIO_ALS_ERR_ARG, "eid_off[0] must be 0");
  for (int64_t e = 0; e < n; ++e)
    if (code[e] < FOLD_SET || code[e] > FOLD_DELETE)
      return fail(nullptr, PIO_ALS_ERR_ARG, "code[%lld] = %d is not 0 ($set), 1 ($unset) or 2 ($delete)", (long long)e,
                  code[e]);
  CK0(cudaSetDevice(device));
  const size_t nb = (size_t)eid_off[n], nn = (size_t)n, nk = (size_t)n_keys;
  std::vector<void*> owned;
  auto A = [&](void** p, size_t bytes_) -> cudaError_t {
    cudaError_t e = cudaMalloc(p, bytes_ ? bytes_ : 1);
    if (e == cudaSuccess) owned.push_back(*p);
    return e;
  };
  struct Guard { std::vector<void*>& v; ~Guard() { for (void* q : v) cudaFree(q); } } guard{owned};
  uint8_t *d_bytes = nullptr, *d_present = nullptr, *d_exists = nullptr;
  long long *d_off = nullptr, *d_time = nullptr, *d_first = nullptr, *d_fus = nullptr, *d_lus = nullptr, *d_win = nullptr;
  int32_t* d_code = nullptr;
  int *d_ent = nullptr, *seg_first = nullptr, *seg_last = nullptr, *last_set = nullptr, *last_del = nullptr, *win = nullptr;
  uint64_t *ka = nullptr, *kb = nullptr;
  uint32_t *va = nullptr, *vb = nullptr;
  CK0(A((void**)&d_bytes, nb));
  CK0(A((void**)&d_off, 8 * (nn + 1)));
  CK0(A((void**)&d_code, 4 * nn));
  CK0(A((void**)&d_time, 8 * nn));
  CK0(A((void**)&d_present, nn));
  CK0(A((void**)&d_ent, 4 * nn));
  CK0(A((void**)&d_first, 8 * nn));
  CK0(A((void**)&ka, 8 * nn)); CK0(A((void**)&kb, 8 * nn));
  CK0(A((void**)&va, 4 * nn)); CK0(A((void**)&vb, 4 * nn));
  cudaStream_t st = 0;
  CK0(cudaMemcpyAsync(d_bytes, eid_bytes, nb, cudaMemcpyHostToDevice, st));
  CK0(cudaMemcpyAsync(d_off, eid_off, 8 * (nn + 1), cudaMemcpyHostToDevice, st));
  CK0(cudaMemcpyAsync(d_code, code, 4 * nn, cudaMemcpyHostToDevice, st));
  CK0(cudaMemcpyAsync(d_time, time_us, 8 * nn, cudaMemcpyHostToDevice, st));
  if (n_keys) CK0(cudaMemcpyAsync(d_present, present, nn, cudaMemcpyHostToDevice, st));
  int64_t n_ent = 0;
  const int rc = ids_encode_device(d_bytes, d_off, n, st, d_ent, d_first, &n_ent);
  if (rc != PIO_ALS_OK) return rc;
  const size_t ne = (size_t)n_ent;
  CK0(A((void**)&seg_first, 4 * ne)); CK0(A((void**)&seg_last, 4 * ne));
  CK0(A((void**)&last_set, 4 * ne)); CK0(A((void**)&last_del, 4 * ne));
  CK0(A((void**)&win, 4 * ne * nk));
  CK0(A((void**)&d_exists, ne));
  CK0(A((void**)&d_fus, 8 * ne)); CK0(A((void**)&d_lus, 8 * ne));
  CK0(A((void**)&d_win, 8 * ne * nk));
  CK0(cudaMemsetAsync(last_set, 0xFF, 4 * ne, st));   // -1: none
  CK0(cudaMemsetAsync(last_del, 0xFF, 4 * ne, st));
  if (nk) CK0(cudaMemsetAsync(win, 0xFF, 4 * ne * nk, st));
  // (entity, time, line): stable by time, then stable by entity
  fold_time_key_kernel<<<nblk(n, 256), 256, 0, st>>>(d_time, n, ka, va);
  bool in_b = false;
  CK0(radix_sort_pairs(ka, va, kb, vb, nn, 64, st, &in_b, nullptr));
  uint64_t* k1 = in_b ? kb : ka;   // sorted by time; the other pair is free
  uint32_t* v1 = in_b ? vb : va;
  uint64_t* k2 = in_b ? ka : kb;
  uint32_t* v2 = in_b ? va : vb;
  fold_entity_key_kernel<<<nblk(n, 256), 256, 0, st>>>(v1, d_ent, n, k1);
  CK0(radix_sort_pairs(k1, v1, k2, v2, nn, ceil_log2((uint64_t)n_ent), st, &in_b, nullptr));
  const uint64_t* ks = in_b ? k2 : k1;
  const uint32_t* vs = in_b ? v2 : v1;
  fold_reduce_kernel<<<nblk(n, 256), 256, 0, st>>>(ks, vs, d_code, d_present, n_keys, n, seg_first, seg_last, last_set,
                                                   last_del, win);
  fold_finish_kernel<<<nblk(n_ent, 256), 256, 0, st>>>(vs, d_code, d_time, seg_first, seg_last, last_set, last_del, win,
                                                       n_keys, n_ent, d_exists, d_fus, d_lus, d_win);
  CK0(cudaGetLastError());
  CK0(cudaMemcpyAsync(out_first_event, d_first, 8 * ne, cudaMemcpyDeviceToHost, st));
  CK0(cudaMemcpyAsync(out_exists, d_exists, ne, cudaMemcpyDeviceToHost, st));
  CK0(cudaMemcpyAsync(out_first_us, d_fus, 8 * ne, cudaMemcpyDeviceToHost, st));
  CK0(cudaMemcpyAsync(out_last_us, d_lus, 8 * ne, cudaMemcpyDeviceToHost, st));
  if (nk) CK0(cudaMemcpyAsync(out_winner, d_win, 8 * ne * nk, cudaMemcpyDeviceToHost, st));
  CK0(cudaStreamSynchronize(st));
  *out_n_entities = n_ent;
  return PIO_ALS_OK;
}

/* debug only (not in pio_als.h): out[0] host-to-device copy, out[1] kernels, out[2] device-to-host copy (device ms),
 * out[3] host copy into pinned staging (wall ms), out[4] device chunks -- of the last pio_events_scan on this thread.
 * Used by tools/events_bench.py. */
__attribute__((visibility("default"))) int pio_events_debug_timing(double out[5]) {
  if (!out) return PIO_ALS_ERR_ARG;
  const EvTiming& t = g_ev_timing;
  out[0] = t.h2d_ms, out[1] = t.kernel_ms, out[2] = t.d2h_ms, out[3] = t.stage_ms, out[4] = (double)t.chunks;
  return PIO_ALS_OK;
}

// ---- item co-occurrence (similarproduct CooccurrenceAlgorithm) ------------------------------------------------------------
int pio_cooc_train(int device, const int32_t* user, const int32_t* item, int64_t n, int32_t n_users, int32_t n_items,
                   int topn, int32_t* out_item, int32_t* out_count, int32_t* out_n) {
  if (!user || !item || !out_item || !out_count || !out_n || n < 1 || n_users < 1 || n_items < 1 || topn < 1)
    return fail(nullptr, PIO_ALS_ERR_ARG, "bad pio_cooc_train arguments");
  if (n >= (1ll << 32)) return fail(nullptr, PIO_ALS_ERR_ARG, "n must be < 2^32");
  for (int64_t e = 0; e < n; ++e)
    if (user[e] < 0 || user[e] >= n_users || item[e] < 0 || item[e] >= n_items)
      return fail(nullptr, PIO_ALS_ERR_ARG, "event %lld has a user/item index out of range", (long long)e);
  CK0(cudaSetDevice(device));
  const int bits_u = ceil_log2((uint64_t)n_users), bits_i = ceil_log2((uint64_t)n_items);
  if (2 * bits_i > 40) return fail(nullptr, PIO_ALS_ERR_ARG, "n_items too large for the pair keys (max 2^20 items)");
  const int bits_c = 64 - 2 * bits_i > 32 ? 32 : 64 - 2 * bits_i;
  std::vector<void*> owned;
  auto A = [&](void** p, size_t bytes_) -> cudaError_t {
    cudaError_t e = cudaMalloc(p, bytes_ ? bytes_ : 1);
    if (e == cudaSuccess) owned.push_back(*p);
    return e;
  };
  struct Guard { std::vector<void*>& v; ~Guard() { for (void* q : v) cudaFree(q); } } guard{owned};
  cudaStream_t st = 0;
  int *du = nullptr, *di = nullptr;
  uint64_t *ka = nullptr, *kb = nullptr, *dk = nullptr;
  uint32_t *va = nullptr, *vb = nullptr, *flag = nullptr, *rank = nullptr;
  CK0(A((void**)&du, 4 * (size_t)n)); CK0(A((void**)&di, 4 * (size_t)n));
  CK0(A((void**)&ka, 8 * (size_t)n)); CK0(A((void**)&kb, 8 * (size_t)n));
  CK0(A((void**)&va, 4 * (size_t)n)); CK0(A((void**)&vb, 4 * (size_t)n));
  CK0(A((void**)&flag, 4 * (size_t)n)); CK0(A((void**)&dk, 8 * (size_t)n)); CK0(A((void**)&rank, 4 * (size_t)n));
  CK0(cudaMemcpyAsync(du, user, 4 * (size_t)n, cudaMemcpyHostToDevice, st));
  CK0(cudaMemcpyAsync(di, item, 4 * (size_t)n, cudaMemcpyHostToDevice, st));
  // 1. distinct (user, item), sorted by user then item
  cooc_keys_kernel<<<nblk(n, 256), 256, 0, st>>>(du, di, n, bits_i, ka, va);
  bool in_b = false;
  CK0(radix_sort_pairs(ka, va, kb, vb, (size_t)n, bits_u + bits_i, st, &in_b, nullptr));
  const uint64_t* ks = in_b ? kb : ka;
  cooc_head_kernel<<<nblk(n, 256), 256, 0, st>>>(ks, n, flag);
  uint32_t lf = 0, lp = 0;
  CK0(cudaMemcpyAsync(&lf, flag + n - 1, 4, cudaMemcpyDeviceToHost, st));
  uint32_t* pos = in_b ? va : vb;   // the payload buffer that is free now
  CK0(scan_exclusive_u32(flag, pos, (size_t)n, st, nullptr));
  CK0(cudaMemcpyAsync(&lp, pos + n - 1, 4, cudaMemcpyDeviceToHost, st));
  CK0(cudaStreamSynchronize(st));
  const long long m = (long long)lp + lf;
  cooc_compact_kernel<<<nblk(n, 256), 256, 0, st>>>(ks, flag, pos, n, dk);
  // 2. pairs (item1 < item2) per user
  cooc_rank_kernel<<<nblk(m, 256), 256, 0, st>>>(dk, m, bits_i, rank);
  uint32_t* off = flag;
  CK0(scan_exclusive_u32(rank, off, (size_t)m, st, nullptr));
  uint32_t lr = 0, lo = 0;
  CK0(cudaMemcpyAsync(&lr, rank + m - 1, 4, cudaMemcpyDeviceToHost, st));
  CK0(cudaMemcpyAsync(&lo, off + m - 1, 4, cudaMemcpyDeviceToHost, st));
  CK0(cudaStreamSynchronize(st));
  const long long np = (long long)lo + lr;
  if (np >= (1ll << 31)) return fail(nullptr, PIO_ALS_ERR_ARG, "more than 2^31-1 co-occurrence pairs (%lld)", np);
  std::vector<int> h_item((size_t)n_items * topn, -1), h_cnt((size_t)n_items * topn, 0), h_n((size_t)n_items, 0);
  if (np > 0) {
    uint64_t *pk = nullptr, *pk2 = nullptr, *rk = nullptr, *rk2 = nullptr;
    uint32_t *pp = nullptr, *pp2 = nullptr, *pf = nullptr, *ppos = nullptr, *rp = nullptr, *rp2 = nullptr;
    CK0(A((void**)&pk, 8 * (size_t)np)); CK0(A((void**)&pk2, 8 * (size_t)np));
    CK0(A((void**)&pp, 4 * (size_t)np)); CK0(A((void**)&pp2, 4 * (size_t)np));
    CK0(A((void**)&pf, 4 * (size_t)np)); CK0(A((void**)&ppos, 4 * (size_t)np));
    cooc_pairs_kernel<<<nblk(m, 256), 256, 0, st>>>(dk, rank, off, m, bits_i, pk, pp);
    bool pb_ = false;
    CK0(radix_sort_pairs(pk, pp, pk2, pp2, (size_t)np, 2 * bits_i, st, &pb_, nullptr));
    const uint64_t* pks = pb_ ? pk2 : pk;
    cooc_head_kernel<<<nblk(np, 256), 256, 0, st>>>(pks, np, pf);
    uint32_t cf = 0, cp = 0;
    CK0(cudaMemcpyAsync(&cf, pf + np - 1, 4, cudaMemcpyDeviceToHost, st));
    CK0(scan_exclusive_u32(pf, ppos, (size_t)np, st, nullptr));
    CK0(cudaMemcpyAsync(&cp, ppos + np - 1, 4, cudaMemcpyDeviceToHost, st));
    CK0(cudaStreamSynchronize(st));
    const long long C = (long long)cp + cf, n2 = 2 * C;
    // 3. both directions, ranked per item by (count desc, other item asc)
    CK0(A((void**)&rk, 8 * (size_t)n2)); CK0(A((void**)&rk2, 8 * (size_t)n2));
    CK0(A((void**)&rp, 4 * (size_t)n2)); CK0(A((void**)&rp2, 4 * (size_t)n2));
    cooc_runs_kernel<<<nblk(np, 256), 256, 0, st>>>(pks, pf, ppos, np, bits_i, bits_c, rk, rp);
    bool rb = false;
    CK0(radix_sort_pairs(rk, rp, rk2, rp2, (size_t)n2, 2 * bits_i + bits_c, st, &rb, nullptr));
    int *d_oi = nullptr, *d_oc = nullptr, *d_on = nullptr;
    CK0(A((void**)&d_oi, 4 * (size_t)n_items * topn)); CK0(A((void**)&d_oc, 4 * (size_t)n_items * topn));
    CK0(A((void**)&d_on, 4 * (size_t)n_items));
    CK0(cudaMemsetAsync(d_oi, 0xff, 4 * (size_t)n_items * topn, st));
    CK0(cudaMemsetAsync(d_oc, 0, 4 * (size_t)n_items * topn, st));
    CK0(cudaMemsetAsync(d_on, 0, 4 * (size_t)n_items, st));
    cooc_take_kernel<<<nblk(n2, 256), 256, 0, st>>>(rb ? rk2 : rk, rb ? rp2 : rp, n2, bits_i, bits_c, topn, d_oi, d_oc, d_on);
    CK0(cudaMemcpyAsync(h_item.data(), d_oi, 4 * h_item.size(), cudaMemcpyDeviceToHost, st));
    CK0(cudaMemcpyAsync(h_cnt.data(), d_oc, 4 * h_cnt.size(), cudaMemcpyDeviceToHost, st));
    CK0(cudaMemcpyAsync(h_n.data(), d_on, 4 * h_n.size(), cudaMemcpyDeviceToHost, st));
    CK0(cudaStreamSynchronize(st));
  }
  memcpy(out_item, h_item.data(), 4 * h_item.size());
  memcpy(out_count, h_cnt.data(), 4 * h_cnt.size());
  memcpy(out_n, h_n.data(), 4 * h_n.size());
  return PIO_ALS_OK;
}

// ---- NaiveBayes ---------------------------------------------------------------------------------
int pio_nb_train(int device, const int32_t* label, const float* x, int64_t n, int n_feat, int n_class, double lambda,
                 double* pi, double* theta) {
  if (!label || !x || !pi || !theta || n <= 0 || n_feat < 1 || n_class < 1)
    return fail(nullptr, PIO_ALS_ERR_ARG, "bad NaiveBayes arguments");
  const int width = n_class * (n_feat + 1);
  if ((size_t)width * 8 * sizeof(double) > 200 * 1024) return fail(nullptr, PIO_ALS_ERR_ARG, "n_class*(n_feat+1) too large");
  CK0(cudaSetDevice(device));
  for (int64_t r = 0; r < n; ++r)
    if (label[r] < 0 || label[r] >= n_class) return fail(nullptr, PIO_ALS_ERR_ARG, "label out of range at row %lld", (long long)r);
  int* dl = nullptr;
  float* dx = nullptr;
  double *dp = nullptr, *dout = nullptr;
  const int nb = 296;
  CK0(cudaMalloc((void**)&dl, sizeof(int) * n));
  CK0(cudaMalloc((void**)&dx, sizeof(float) * n * n_feat));
  CK0(cudaMalloc((void**)&dp, sizeof(double) * (size_t)nb * width));
  CK0(cudaMalloc((void**)&dout, sizeof(double) * width));
  CK0(cudaMemcpy(dl, label, sizeof(int) * n, cudaMemcpyHostToDevice));
  CK0(cudaMemcpy(dx, x, sizeof(float) * n * n_feat, cudaMemcpyHostToDevice));
  const size_t smem = sizeof(double) * 8 * width;
  CK0(cudaFuncSetAttribute(nb_partial_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  nb_partial_kernel<<<nb, 256, smem>>>(dl, dx, n, n_feat, n_class, dp);
  nb_reduce_kernel<<<nblk(width, 128), 128>>>(dp, nb, width, dout);
  std::vector<double> acc(width);
  CK0(cudaMemcpy(acc.data(), dout, sizeof(double) * width, cudaMemcpyDeviceToHost));
  cudaFree(dl); cudaFree(dx); cudaFree(dp); cudaFree(dout);
  // MLlib multinomial: pi_c = log(n_c + l) - log(N + C l); theta_cj = log(s_cj + l) - log(sum_j s_cj + F l)
  const double logden = log((double)n + n_class * lambda);
  for (int c = 0; c < n_class; ++c) {
    pi[c] = log(acc[c * (n_feat + 1) + n_feat] + lambda) - logden;
    double tot = 0;
    for (int j = 0; j < n_feat; ++j) tot += acc[c * (n_feat + 1) + j];
    const double lt = log(tot + n_feat * lambda);
    for (int j = 0; j < n_feat; ++j) theta[c * n_feat + j] = log(acc[c * (n_feat + 1) + j] + lambda) - lt;
  }
  return PIO_ALS_OK;
}

int pio_nb_predict(int device, const float* x, int64_t n, int n_feat, int n_class, const double* pi, const double* theta,
                   int32_t* out_label) {
  if (!x || !pi || !theta || !out_label || n <= 0) return fail(nullptr, PIO_ALS_ERR_ARG, "bad NaiveBayes arguments");
  CK0(cudaSetDevice(device));
  float* dx = nullptr;
  double *dpi = nullptr, *dth = nullptr;
  int* dout = nullptr;
  CK0(cudaMalloc((void**)&dx, sizeof(float) * n * n_feat));
  CK0(cudaMalloc((void**)&dpi, sizeof(double) * n_class));
  CK0(cudaMalloc((void**)&dth, sizeof(double) * n_class * n_feat));
  CK0(cudaMalloc((void**)&dout, sizeof(int) * n));
  CK0(cudaMemcpy(dx, x, sizeof(float) * n * n_feat, cudaMemcpyHostToDevice));
  CK0(cudaMemcpy(dpi, pi, sizeof(double) * n_class, cudaMemcpyHostToDevice));
  CK0(cudaMemcpy(dth, theta, sizeof(double) * n_class * n_feat, cudaMemcpyHostToDevice));
  nb_predict_kernel<<<nblk(n, 256), 256>>>(dx, n, n_feat, n_class, dpi, dth, dout);
  CK0(cudaMemcpy(out_label, dout, sizeof(int) * n, cudaMemcpyDeviceToHost));
  cudaFree(dx); cudaFree(dpi); cudaFree(dth); cudaFree(dout);
  return PIO_ALS_OK;
}

}  // extern "C"
