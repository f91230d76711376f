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
#include <array>
#include <deque>
#include <exception>
#include <map>
#include <memory>
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
#include "events_index.cuh"
#include "cooc.cuh"
#include "cooc_predict.cuh"
#include "popular.cuh"
#include "serve_merge.cuh"
#include "forest.cuh"
#include "sessions.cuh"
#include "eval_folds.cuh"
#include "cls_folds.cuh"
#include "assoc.cuh"
#include "rank_lists.cuh"
#include "assoc_predict.cuh"
#include "text_nb.cuh"
#include "text_plan.h"
#include "dense_pca.cuh"
#include "logreg.cuh"

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
// one thread per run head: fold the run in event order (sum: reduceByKey(_ + _), so a run of one keeps its rating's
// bits, -0.0 included) or pick the latest event (keep-last)
__global__ void dedup_compact_kernel(const uint64_t* keys, const uint32_t* pay, const uint32_t* pos,
                                     long long n, int bits_i, const float* rating, const long long* ts,
                                     int mode, int* ou, int* oi, float* orr) {
  const long long e = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (e >= n) return;
  const uint64_t key = keys[e];
  if (e > 0 && keys[e - 1] == key) return;
  float acc;
  if (mode == PIO_ALS_DEDUP_SUM) {
    acc = rating[pay[e]];
    for (long long t = e + 1; t < n && keys[t] == key; ++t) acc += rating[pay[t]];
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

static int vfail(std::string& sink, int code, const char* fmt, va_list ap) {
  char buf[512];
  vsnprintf(buf, sizeof buf, fmt, ap);
  sink = buf;
  return code;
}
// the message goes to the handle, or (h == nullptr) to the thread's last error
static int fail(pio_als_handle* h, int code, const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  const int rc = vfail(h ? h->err : g_create_error, code, fmt, ap);
  va_end(ap);
  return rc;
}
static int fail_to(std::string* sink, int code, const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  const int rc = vfail(*sink, code, fmt, ap);
  va_end(ap);
  return rc;
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

// Device temporaries of one API call, or of one chunk of an event scan, on stream s: released (stream-ordered) on every
// exit path, including the early error returns of CK() and CK0().
struct Scratch {
  cudaStream_t s;
  std::vector<void*> ptrs;
  explicit Scratch(cudaStream_t s_) : s(s_) {}
  Scratch(const Scratch&) = delete;
  Scratch& operator=(const Scratch&) = delete;
  template <class T>
  cudaError_t alloc(T** p, size_t n) {
    const cudaError_t e = cudaMallocAsync((void**)p, (n ? n : 1) * sizeof(T), s);
    if (e == cudaSuccess) ptrs.push_back((void*)*p);
    return e;
  }
  ~Scratch() {
    for (void* q : ptrs) cudaFreeAsync(q, s);
  }
};

// Everything a synchronous call without a handle holds until it returns: device memory (cudaMalloc), pinned host memory
// (cudaHostAlloc), and the streams and events it creates.  On every exit path, including the early error returns of
// CK0(), the stream it was given and the streams it created are drained first, so that nothing is freed under a
// running kernel or copy; then everything is released.
struct CallMem {
  std::vector<cudaStream_t> drain, streams;
  std::vector<cudaEvent_t> events;
  std::vector<void*> dev, pinned;
  CallMem() = default;
  explicit CallMem(cudaStream_t st) : drain{st} {}
  CallMem(const CallMem&) = delete;
  CallMem& operator=(const CallMem&) = delete;
  template <class T>
  cudaError_t device(T** p, size_t n) {
    const size_t bytes = n * sizeof(T);
    const cudaError_t e = cudaMalloc((void**)p, bytes ? bytes : 1);
    if (e == cudaSuccess) dev.push_back((void*)*p);
    return e;
  }
  template <class T>
  cudaError_t host(T** p, size_t n) {
    const size_t bytes = n * sizeof(T);
    const cudaError_t e = cudaHostAlloc((void**)p, bytes ? bytes : 1, cudaHostAllocDefault);
    if (e == cudaSuccess) pinned.push_back((void*)*p);
    return e;
  }
  cudaError_t stream(cudaStream_t* s) {
    const cudaError_t e = cudaStreamCreateWithFlags(s, cudaStreamNonBlocking);
    if (e == cudaSuccess) drain.push_back(*s), streams.push_back(*s);
    return e;
  }
  cudaError_t event(cudaEvent_t* ev) {
    const cudaError_t e = cudaEventCreate(ev);
    if (e == cudaSuccess) events.push_back(*ev);
    return e;
  }
  ~CallMem() {
    for (cudaStream_t s : drain) cudaStreamSynchronize(s);
    for (void* q : dev) cudaFree(q);
    for (void* q : pinned) cudaFreeHost(q);
    for (cudaStream_t s : streams) cudaStreamDestroy(s);
    for (cudaEvent_t e : events) cudaEventDestroy(e);
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
  Scratch tmp(h->stream);
  SortBufs sb;
  for (int i : {0, 1}) {
    CK(h, tmp.alloc(&sb.k[i], (size_t)nnz));
    CK(h, tmp.alloc(&sb.v[i], (size_t)nnz));
  }
  if (nnz > 0) {
    make_keys_int_kernel<<<nblk(nnz, 256), 256, 0, st>>>(rowext, colext, nnz, row.perm, col.rpos, col.bits, sb.keys(),
                                                         sb.vals());
    LAUNCHED(h);
    CK(h, radix_sort_pairs(sb, (size_t)nnz, row.bits + col.bits, st, &h->st.kernel_launches));
  }
  tmark(h, "  side: keys + radix sort");
  const uint64_t* ks = sb.keys();
  const uint32_t* vs = sb.vals();
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
  Scratch tmp(h->stream);
  SortBufs sb;
  for (int i : {0, 1}) {
    CK(h, tmp.alloc(&sb.k[i], (size_t)s.n));
    CK(h, tmp.alloc(&sb.v[i], (size_t)s.n));
  }
  degree_keys_kernel<<<nblk(s.n, 256), 256, 0, st>>>(s.deg, s.n, sb.keys(), sb.vals());
  LAUNCHED(h);
  CK(h, radix_sort_pairs(sb, (size_t)s.n, 32, st, &h->st.kernel_launches));
  fill_int_kernel<<<nblk(s.n_internal, 256), 256, 0, st>>>(s.inv, s.n_internal, -1);
  LAUNCHED(h);
  assign_internal_kernel<<<nblk(s.n, 256), 256, 0, st>>>(sb.vals(), s.n, h->cfg.world_size, s.R, s.perm, s.inv,
                                                         s.rpos, s.p2i);
  LAUNCHED(h);
  return PIO_ALS_OK;
}

// ---- sharded ingest: all-to-all exchange of event arrays ------------------------------------------------------------
// The n events on this rank go to the ranks named by the sort keys (destination rank, payload = event index; built by the
// caller in sb's live half).  Events keep their order per destination and arrive concatenated in source-rank order, so a
// global event order (rank r's slice precedes rank r + 1's) survives.  The received arrays are allocated in `keep`.
struct XArr {
  const void* in;
  void** out;
  size_t elem;
};
static int exchange_events(pio_als_handle* h, Scratch& keep, SortBufs& sb, long long n, XArr* arrs, int na,
                           long long* n_out) {
  cudaStream_t st = h->stream;
  NcclApi& nc = nccl_api();
  const int W = h->cfg.world_size, me = h->cfg.world_rank;
  Scratch tmp(h->stream);
  if (n > 0) CK(h, radix_sort_pairs(sb, (size_t)n, ceil_log2((uint64_t)W), st, &h->st.kernel_launches));
  const uint64_t* ks = sb.keys();
  const uint32_t* vs = sb.vals();
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
  Scratch tmp(h->stream);   // everything temporary: released on every exit path, including the CK() early returns
  // 0. sharded + dedup: first bring all events of a user to one rank (user mod W), keeping the event order
  const int* su = d_user;
  const int* si = d_item;
  const float* sr = d_rating;
  const long long* sts = d_ts;
  long long ns = nnz;
  if (sharded && dedup != PIO_ALS_DEDUP_NONE) {
    Scratch xs(h->stream);
    SortBufs sb;
    for (int i : {0, 1}) {
      CK(h, xs.alloc(&sb.k[i], (size_t)nnz));
      CK(h, xs.alloc(&sb.v[i], (size_t)nnz));
    }
    if (nnz > 0) {
      dest_mod_kernel<<<nblk(nnz, 256), 256, 0, st>>>(d_user, nnz, W, sb.keys(), sb.vals());
      LAUNCHED(h);
    }
    void *xu = nullptr, *xi = nullptr, *xr = nullptr, *xt = nullptr;
    XArr arrs[4] = {{d_user, &xu, 4}, {d_item, &xi, 4}, {d_rating, &xr, 4},
                    {dedup == PIO_ALS_DEDUP_KEEP_LAST ? (const void*)d_ts : nullptr, &xt, 8}};
    int rc = exchange_events(h, tmp, sb, nnz, arrs, 4, &ns);
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
    Scratch ds(h->stream);
    SortBufs sb;
    for (int i : {0, 1}) {
      CK(h, ds.alloc(&sb.k[i], (size_t)ns));
      CK(h, ds.alloc(&sb.v[i], (size_t)ns));
    }
    const int bu = ceil_log2((uint64_t)U.n), bi = ceil_log2((uint64_t)I.n);
    make_keys_ext_kernel<<<nblk(ns, 256), 256, 0, st>>>(su, si, ns, bi, sb.keys(), sb.vals());
    LAUNCHED(h);
    CK(h, radix_sort_pairs(sb, (size_t)ns, bu + bi, st, &h->st.kernel_launches));
    const uint64_t* ks = sb.keys();
    const uint32_t* vs = sb.vals();
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
      Scratch xs(h->stream), recv(h->stream);
      SortBufs sb;
      for (int i : {0, 1}) {
        CK(h, xs.alloc(&sb.k[i], (size_t)n2));
        CK(h, xs.alloc(&sb.v[i], (size_t)n2));
      }
      if (n2 > 0) {
        dest_owner_kernel<<<nblk(n2, 256), 256, 0, st>>>(j.rowext, n2, j.row->perm, j.row->R, sb.keys(), sb.vals());
        LAUNCHED(h);
      }
      void *xrow = nullptr, *xcol = nullptr, *xr = nullptr;
      XArr arrs[3] = {{j.rowext, &xrow, 4}, {j.colext, &xcol, 4}, {cr, &xr, 4}};
      long long ne = 0;
      rc = exchange_events(h, recv, sb, n2, arrs, 3, &ne);
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
  // before anything is staged: a host copy of nnz events would read past arrays the call is about to refuse
  if (nnz >= (1ll << 32)) return fail(h, PIO_ALS_ERR_ARG, "nnz must be < 2^32 per call");
  if (dedup_mode < 0 || dedup_mode > 2) return fail(h, PIO_ALS_ERR_ARG, "bad dedup_mode %d", dedup_mode);
  std::lock_guard<std::mutex> lk(h->mu);
  CK(h, cudaSetDevice(h->cfg.device));
  cudaStream_t st = h->stream;
  cudaEvent_t a, b;
  cudaEventCreate(&a);
  cudaEventCreate(&b);
  cudaEventRecord(a, st);
  int rc;
  {
    Scratch tmp(h->stream);
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

/* debug only (not in pio_als.h): what the last set_ratings built on one side (0 = users, 1 = items) of this rank.
 * scalars[11]: n, R, n_internal, bits, nnz_local, n_active, n_heavy, n_parts, nnz after dedup over all ranks, heavy_t,
 * part_len.  Arrays (HOST; each may be null, sizes from scalars): deg / npos / perm / rpos [n], inv [n_internal], the
 * local ptr [R + 1], idx / val [nnz_local], nreg [R], part_beg / part_end [n_parts], row_part_ptr [n_heavy + 1].  Only
 * copies out; changes nothing.  Used by tests/test_gpu_ingest.py. */
__attribute__((visibility("default"))) int pio_als_debug_side(pio_als_handle* h, int side, int64_t scalars[11],
                                                              uint32_t* deg, uint32_t* npos, int32_t* perm, int32_t* inv,
                                                              int32_t* rpos, int64_t* ptr, int32_t* idx, float* val,
                                                              float* nreg, int64_t* part_beg, int64_t* part_end,
                                                              int32_t* row_part_ptr) {
  if (!h || !scalars || (side != 0 && side != 1)) return PIO_ALS_ERR_ARG;
  std::lock_guard<std::mutex> lk(h->mu);
  if (!h->have_ratings) return fail(h, PIO_ALS_ERR_STATE, "pio_als_debug_side before set_ratings");
  CK(h, cudaSetDevice(h->cfg.device));
  const Side& s = side == 0 ? h->U : h->I;
  const int64_t v[11] = {s.n, s.R, s.n_internal, s.bits, s.nnz_local, s.n_active, s.n_heavy, s.n_parts, h->st.nnz,
                         s.plan.heavy_t, s.plan.part_len};
  std::copy(v, v + 11, scalars);
  const cudaStream_t st = h->stream;
  const struct { void* to; const void* from; size_t bytes; } jobs[] = {
      {deg, s.deg, sizeof(uint32_t) * (size_t)s.n},          {npos, s.npos, sizeof(uint32_t) * (size_t)s.n},
      {perm, s.perm, sizeof(int32_t) * (size_t)s.n},         {inv, s.inv, sizeof(int32_t) * (size_t)s.n_internal},
      {rpos, s.rpos, sizeof(int32_t) * (size_t)s.n},         {ptr, s.ptr, sizeof(int64_t) * ((size_t)s.R + 1)},
      {idx, s.idx, sizeof(int32_t) * (size_t)s.nnz_local},   {val, s.val, sizeof(float) * (size_t)s.nnz_local},
      {nreg, s.nreg, sizeof(float) * (size_t)s.R},           {part_beg, s.part_beg, sizeof(int64_t) * (size_t)s.n_parts},
      {part_end, s.part_end, sizeof(int64_t) * (size_t)s.n_parts}};
  for (const auto& j : jobs)
    if (j.to && j.bytes) CK(h, cudaMemcpyAsync(j.to, j.from, j.bytes, cudaMemcpyDeviceToHost, st));
  if (row_part_ptr && s.n_heavy > 0) std::copy(s.h_row_part_ptr.begin(), s.h_row_part_ptr.end(), row_part_ptr);
  CK(h, cudaStreamSynchronize(st));
  return PIO_ALS_OK;
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

// f(std::true_type / std::false_type): the filtered or the plain instantiation of a batch kernel
template <class F>
static int with_filt(bool filtered, F&& f) {
  return filtered ? f(std::true_type()) : f(std::false_type());
}
// the per-query filter of chunk c: the call's filter, numbered from the chunk's first query
static QueryFilterDev chunk_filter(const QueryFilterDev* qf, const Chunk& c) {
  QueryFilterDev q;
  if (qf) q = *qf;
  q.qbase = c.q0;
  return q;
}
// the recommend kernel of the plan for the users of chunk c (xq / valid: the gathered user vectors)
static int launch_dot(pio_als_handle* h, const ScorePlan& p, const Chunk& c, const float* d_xq, const uint8_t* d_valid,
                      const DevFilter& f, const QueryFilterDev* qf = nullptr) {
  const float* xq = d_xq + (size_t)c.q0 * h->KP;
  const QueryFilterDev q = chunk_filter(qf, c);
  return with_filt(p.filtered, [&](auto filt) {
    constexpr bool FILT = decltype(filt)::value;
    if (p.kernel == PIO_ALS_PATH_DOT_BLOCKED)
      return with_kp(h->KP, [&](auto kp) {
        return score_launch(h, score_dot_blocked_kernel<decltype(kp)::value, FILT>, c.grid, dim3(p.threads), p.smem,
                            p.launch_bits(), h->I.F, h->I.n_internal, xq, d_valid + c.q0, c.nq, h->I.cand_ext, f.mask, f.weight,
                            c.pk, c.cand, q);
      });
    return score_launch(h, score_dot_topk_batched_kernel<FILT>, c.grid, dim3(p.threads), p.smem, p.launch_bits(), h->I.F,
                        h->I.n_internal, h->KP, xq, d_valid + c.q0, c.nq, h->I.cand_ext, f.mask, f.weight, c.bound, c.pk, c.cand,
                        q);
  });
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
static int launch_cos(pio_als_handle* h, const ScorePlan& p, const Chunk& c, const CosQueries& q, const DevFilter& f,
                      const QueryFilterDev* qf = nullptr) {
  const QueryFilterDev qd = chunk_filter(qf, c);   // bins carry the call's query numbers: their chunks start at query 0
  return with_filt(p.filtered, [&](auto filt) {
    constexpr bool FILT = decltype(filt)::value;
    if (p.kernel == PIO_ALS_PATH_COS_BLOCKED)
      return with_kp(h->KP, [&](auto kp) {
        return score_launch(h, score_cos_blocked_kernel<decltype(kp)::value, FILT>, c.grid, dim3(p.threads), p.smem,
                            p.launch_bits(), h->I.F, h->I.n_internal, h->cfg.rank, q.qf, q.q0 + (size_t)c.g0 * DB_WPR,
                            q.v0 + (size_t)c.g0 * DB_WPR, q.n_bins - c.g0 * DB_WPR, q.vq, q.qptr, q.qid, h->I.cand_ext, f.mask,
                            f.weight, q.keep, c.pk, c.cand, qd);
      });
    return score_launch(h, score_cos_topk_multi_kernel<FILT>, c.grid, dim3(p.threads), p.smem, p.launch_bits(), h->I.F,
                        h->I.n_internal, h->KP, h->cfg.rank, q.qf, q.v0 + c.g0, q.vq, q.qptr + c.q0, q.qid, c.nq, h->I.cand_ext,
                        f.mask, f.weight, c.bound, q.keep, c.pk, c.cand, qd);
  });
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
                          float* out_scores, int32_t* out_count, const QueryFilterDev* qf = nullptr) {
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
  rc = run_passes(h, p, n_queries, topk, d_cand, o, [&](const Chunk& c) { return launch_cos(h, p, c, q, f, qf); });
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
  Scratch tmp(h->stream);
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

// ---- filtered batch calls (pio_als_query_filter) -------------------------------------------------------------------------
// one key per list entry: (query of the entry << 32) | item id; thread t finds its query in ptr (the last j with ptr[j] <= t)
__global__ void qf_keys_kernel(const int* __restrict__ items, const long long* __restrict__ ptr, int nq, long long total,
                               unsigned long long* __restrict__ keys) {
  const long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= total) return;
  int lo = 0, hi = nq;
  while (hi - lo > 1) {
    const int mid = (lo + hi) >> 1;
    if (ptr[mid] <= t) lo = mid;
    else hi = mid;
  }
  keys[t] = ((unsigned long long)(unsigned)lo << 32) | (unsigned)items[t];
}
// item_sets rows (one byte per item) -> one bit per item, `words` 32-bit words per row
__global__ void qf_pack_sets_kernel(const uint8_t* __restrict__ sets, int n_items, int words, long long n_words,
                                    unsigned* __restrict__ bits) {
  const long long w = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (w >= n_words) return;
  const uint8_t* row = sets + (size_t)(w / words) * n_items;
  const int i0 = (int)(w % words) * 32;
  unsigned v = 0;
  for (int b = 0; b < 32 && i0 + b < n_items; ++b)
    if (row[i0 + b]) v |= 1u << b;
  bits[w] = v;
}

// the argument rules of a filter for n queries (pio_als.h); nullptr = fine, else what is wrong
static const char* query_filter_error(const pio_als_query_filter* f, int n) {
  if (f->n_sets < 0) return "query filter: n_sets < 0";
  const struct { const int64_t* ptr; const int32_t* items; const char* order; const char* missing; } lists[2] = {
      {f->ex_ptr, f->ex_items, "query filter: ex_ptr must be non-negative and non-decreasing", "query filter: ex_ptr names entries but ex_items is NULL"},
      {f->wl_ptr, f->wl_items, "query filter: wl_ptr must be non-negative and non-decreasing", "query filter: wl_ptr names entries but wl_items is NULL"}};
  for (const auto& l : lists) {
    if (!l.ptr) continue;
    if (l.ptr[0] < 0) return l.order;
    for (int j = 0; j < n; ++j)
      if (l.ptr[j + 1] < l.ptr[j]) return l.order;
    if (l.ptr[n] > l.ptr[0] && !l.items) return l.missing;
  }
  if (f->set_ix)
    for (int j = 0; j < n; ++j) {
      if (f->set_ix[j] < -1 || f->set_ix[j] >= f->n_sets) return "query filter: set_ix must be -1 or a row of item_sets";
      if (f->set_ix[j] >= 0 && !f->item_sets) return "query filter: set_ix names a row but item_sets is NULL";
    }
  return nullptr;
}

// What the per-query filter uploads need from their caller: the stream they run on, the item count of the set rows, the
// launch counter they add to and where a failure's message goes.  The ALS scoring calls pass their handle's
// (filter_env); the co-occurrence model passes its own.
struct FilterEnv {
  cudaStream_t st;
  int n_items;
  int64_t* launches;
  std::string* err;
};
static FilterEnv filter_env(pio_als_handle* h) { return FilterEnv{h->stream, h->I.n, &h->st.kernel_launches, &h->err}; }
#define CKF(env, call)                                                                                        \
  do {                                                                                                        \
    cudaError_t e_ = (call);                                                                                  \
    if (e_ != cudaSuccess)                                                                                    \
      return fail_to((env).err, PIO_ALS_ERR_CUDA, "%s failed: %s (%s:%d)", #call, cudaGetErrorString(e_), \
                     __FILE__, __LINE__);                                                                     \
  } while (0)
// one launch of n_threads threads in blocks of 256 on env's stream, counted, failing on a launch error
template <typename... KArgs, typename... Args>
static int env_launch(const FilterEnv& env, void (*kernel)(KArgs...), long long n_threads, Args... args) {
  kernel<<<nblk(n_threads, 256), 256, 0, env.st>>>(args...);
  ++*env.launches;
  CKF(env, cudaGetLastError());
  return PIO_ALS_OK;
}

// the lists ptr / items of the queries idx on the device, as sorted keys; the queries are renumbered 0 .. idx.size() - 1
struct DevLists {
  const unsigned long long* keys = nullptr;
  long long* ptr = nullptr;
};
static int upload_lists(const FilterEnv& env, const int64_t* ptr, const int32_t* items, const std::vector<int>& idx,
                        Scratch& tmp, DevLists* out) {
  cudaStream_t st = env.st;
  const int n = (int)idx.size();
  std::vector<long long> rel((size_t)n + 1, 0);
  for (int i = 0; i < n; ++i) rel[i + 1] = rel[i] + (ptr ? ptr[idx[i] + 1] - ptr[idx[i]] : 0);
  const long long total = rel[n];
  CKF(env, tmp.alloc(&out->ptr, rel.size()));
  CKF(env, cudaMemcpyAsync(out->ptr, rel.data(), sizeof(long long) * rel.size(), cudaMemcpyHostToDevice, st));
  if (total == 0) return PIO_ALS_OK;
  std::vector<int> flat((size_t)total);
  for (int i = 0; i < n; ++i)
    if (rel[i + 1] > rel[i]) memcpy(flat.data() + rel[i], items + ptr[idx[i]], sizeof(int) * (size_t)(rel[i + 1] - rel[i]));
  int* d_items = nullptr;
  SortBufs sb;
  CKF(env, tmp.alloc(&d_items, (size_t)total));
  for (int b = 0; b < 2; ++b) {
    CKF(env, tmp.alloc(&sb.k[b], (size_t)total));
    CKF(env, tmp.alloc(&sb.v[b], (size_t)total));
  }
  CKF(env, cudaMemcpyAsync(d_items, flat.data(), sizeof(int) * (size_t)total, cudaMemcpyHostToDevice, st));
  const int rc = env_launch(env, qf_keys_kernel, total, (const int*)d_items, (const long long*)out->ptr, n, total,
                               (unsigned long long*)sb.k[0]);
  if (rc) return rc;
  CKF(env, cudaMemsetAsync(sb.v[0], 0, sizeof(uint32_t) * (size_t)total, st));   // the sort carries a payload; none is needed
  CKF(env, radix_sort_pairs(sb, (size_t)total, 32 + ceil_log2((uint64_t)n), st, env.launches));
  out->keys = (const unsigned long long*)sb.keys();
  return PIO_ALS_OK;
}

// what every part of a filtered call shares on the device: the dense mask / weights and the set rows as bits
struct CallFilter {
  DevFilter dense;
  unsigned* set_bits = nullptr;
  int set_words = 0;
};
// the set rows of f (n_items bytes each) as bits, into out->set_bits / set_words
static int upload_set_rows(const FilterEnv& env, const pio_als_query_filter* f, Scratch& tmp, CallFilter* out) {
  if (!f->set_ix || f->n_sets == 0 || !f->item_sets) return PIO_ALS_OK;
  const int n_items = env.n_items;
  out->set_words = (n_items + 31) / 32;
  const long long n_words = (long long)f->n_sets * out->set_words;
  uint8_t* d_sets = nullptr;
  CKF(env, tmp.alloc(&d_sets, (size_t)f->n_sets * n_items));
  CKF(env, tmp.alloc(&out->set_bits, (size_t)n_words));
  CKF(env, cudaMemcpyAsync(d_sets, f->item_sets, (size_t)f->n_sets * n_items, cudaMemcpyHostToDevice, env.st));
  return env_launch(env, qf_pack_sets_kernel, n_words, (const uint8_t*)d_sets, n_items, out->set_words, n_words,
                       out->set_bits);
}
static int upload_call_filter(pio_als_handle* h, const uint8_t* item_mask, const double* item_weight,
                              const pio_als_query_filter* f, Scratch& tmp, CallFilter* out) {
  const int rc = upload_filter(h, item_mask, item_weight, &tmp, 0, &out->dense);
  if (rc) return rc;
  return upload_set_rows(filter_env(h), f, tmp, out);
}
// the exclusion lists and set rows of the queries idx (renumbered 0 .. idx.size() - 1)
static int upload_part_filter(const FilterEnv& env, const pio_als_query_filter* f, const CallFilter& cf,
                              const std::vector<int>& idx, Scratch& tmp, QueryFilterDev* out) {
  if (f->ex_ptr) {
    DevLists ex;
    const int rc = upload_lists(env, f->ex_ptr, f->ex_items, idx, tmp, &ex);
    if (rc) return rc;
    out->ex = ex.keys;
    out->ex_ptr = ex.ptr;
  }
  if (cf.set_bits) {
    std::vector<int> six(idx.size());
    for (size_t i = 0; i < idx.size(); ++i) six[i] = f->set_ix[idx[i]];
    int* d_six = nullptr;
    CKF(env, tmp.alloc(&d_six, six.size()));
    CKF(env, cudaMemcpyAsync(d_six, six.data(), sizeof(int) * six.size(), cudaMemcpyHostToDevice, env.st));
    out->set_ix = d_six;
    out->set_bits = cf.set_bits;
    out->set_words = cf.set_words;
  }
  return PIO_ALS_OK;
}

// host rows of a part's results, and their way back to the rows idx of the caller's arrays
struct PartOut {
  std::vector<int32_t> items, count;
  std::vector<float> scores;
  PartOut(size_t n, int topk) : items(n * topk), count(n), scores(n * topk) {}
  void scatter(const std::vector<int>& idx, int topk, int32_t* out_items, float* out_scores, int32_t* out_count) const {
    for (size_t i = 0; i < idx.size(); ++i) {
      memcpy(out_items + (size_t)idx[i] * topk, items.data() + i * topk, sizeof(int32_t) * topk);
      memcpy(out_scores + (size_t)idx[i] * topk, scores.data() + i * topk, sizeof(float) * topk);
      if (out_count) out_count[idx[i]] = count[i];
    }
  }
};

// the users idx of a filtered recommend call: scanned by R3 / R4 with the filter test, or (listed) scored over their
// white lists
static int recommend_part(pio_als_handle* h, const int32_t* users, const std::vector<int>& idx, bool listed, int topk,
                          const pio_als_query_filter* f, const CallFilter& cf, int32_t* out_items, float* out_scores,
                          int32_t* out_count) {
  const int n = (int)idx.size();
  if (n == 0) return PIO_ALS_OK;
  cudaStream_t st = h->stream;
  const int KP = h->KP;
  Scratch tmp(st);
  std::vector<int> sub((size_t)n);
  for (int i = 0; i < n; ++i) sub[i] = users[idx[i]];
  const ScorePlan p = listed ? plan_listed(n, topk) : plan_recommend_filtered(score_env(h), n, topk);
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
  CK(h, cudaMemcpyAsync(d_users, sub.data(), sizeof(int) * n, cudaMemcpyHostToDevice, st));
  rc = score_launch(h, gather_rows_kernel, dim3(n), dim3(64), 0, 0, h->U.F, KP, (const int*)d_users, n, h->U.perm, h->U.deg,
                    h->U.n, d_xq, d_valid);
  if (rc) return rc;
  QueryFilterDev qf;
  rc = upload_part_filter(filter_env(h), f, cf, idx, tmp, &qf);
  if (rc) return rc;
  if (listed) {
    DevLists wl;
    rc = upload_lists(filter_env(h), f->wl_ptr, f->wl_items, idx, tmp, &wl);
    if (rc) return rc;
    rc = run_passes(h, p, n, topk, d_cand, o, [&](const Chunk& c) {
      return score_launch(h, score_listed_kernel<false>, c.grid, dim3(p.threads), p.smem, p.launch_bits(), h->I.F, KP, h->I.perm,
                          h->I.deg, h->I.n, (const float*)d_xq, (const uint8_t*)d_valid, (const long long*)nullptr,
                          (const int*)nullptr, wl.keys, (const long long*)wl.ptr, cf.dense.mask, cf.dense.weight, c.bound, 0, c.pk,
                          c.cand, chunk_filter(&qf, c));
    });
  } else {
    rc = run_passes(h, p, n, topk, d_cand, o,
                    [&](const Chunk& c) { return launch_dot(h, p, c, d_xq, d_valid, cf.dense, &qf); });
  }
  if (rc) return rc;
  PartOut po((size_t)n, topk);
  rc = deliver(h, o, n, topk, po.items.data(), po.scores.data(), po.count.data());
  if (rc) return rc;
  po.scatter(idx, topk, out_items, out_scores, out_count);
  return PIO_ALS_OK;
}

// the queries idx of a filtered similar call.  sp / flat: their id lists, renumbered and concatenated.
static int similar_part(pio_als_handle* h, const std::vector<int64_t>& sp, const std::vector<int32_t>& flat,
                        const std::vector<int>& idx, bool listed, int topk, const uint8_t* item_mask,
                        const pio_als_query_filter* f, const CallFilter& cf, int flags, int32_t* out_items, float* out_scores,
                        int32_t* out_count) {
  const int n = (int)idx.size();
  if (n == 0) return PIO_ALS_OK;
  cudaStream_t st = h->stream;
  const ScoreEnv env = score_env(h);
  const long long total = sp[n];
  Scratch tmp(st);
  PartOut po((size_t)n, topk);
  QueryFilterDev qf;
  int rc = PIO_ALS_OK;
  const ScorePlan first = listed ? plan_listed(n, topk) : plan_similar_filtered(n, total, topk);
  bool done = false;
  if (listed || first.route == ROUTE_BATCH) {
    if (total >= (1ll << 31)) return fail(h, PIO_ALS_ERR_ARG, "white-listed queries with 2^31 or more query items in all");
    rc = upload_part_filter(filter_env(h), f, cf, idx, tmp, &qf);
    if (rc) return rc;
    // all query item vectors in one gather (zeros for an id without a factor)
    int* d_qid = nullptr;
    float* d_qf_all = nullptr;
    uint8_t* d_valid = nullptr;
    CK(h, tmp.alloc(&d_qid, (size_t)total));
    CK(h, tmp.alloc(&d_qf_all, (size_t)total * h->KP));
    CK(h, tmp.alloc(&d_valid, (size_t)total));
    if (total > 0) {
      CK(h, cudaMemcpyAsync(d_qid, flat.data(), sizeof(int) * total, cudaMemcpyHostToDevice, st));
      rc = score_launch(h, gather_rows_kernel, dim3((unsigned)total), dim3(64), 0, 0, h->I.F, h->KP, (const int*)d_qid,
                        (int)total, h->I.perm, h->I.deg, h->I.n, d_qf_all, d_valid);
      if (rc) return rc;
    }
    if (listed) {
      DevLists wl;
      rc = upload_lists(filter_env(h), f->wl_ptr, f->wl_items, idx, tmp, &wl);
      if (rc) return rc;
      std::vector<long long> rel(sp.begin(), sp.end());
      long long* d_qptr = nullptr;
      ScoreIdx* d_cand = nullptr;
      CK(h, tmp.alloc(&d_qptr, rel.size()));
      CK(h, cudaMemcpyAsync(d_qptr, rel.data(), sizeof(long long) * rel.size(), cudaMemcpyHostToDevice, st));
      CK(h, tmp.alloc(&d_cand, (size_t)n * first.lists * first.pass_k));
      MergeOut o;
      rc = alloc_results(h, tmp, n, topk, first.passes > 1, &o);
      if (rc) return rc;
      const int keep = (flags & PIO_ALS_SIM_KEEP_QUERY_ITEMS) ? 1 : 0;
      rc = run_passes(h, first, n, topk, d_cand, o, [&](const Chunk& c) {
        return score_launch(h, score_listed_kernel<true>, c.grid, dim3(first.threads), first.smem, first.launch_bits(), h->I.F,
                            h->KP, h->I.perm, h->I.deg, h->I.n, (const float*)d_qf_all, (const uint8_t*)nullptr,
                            (const long long*)d_qptr, (const int*)d_qid, wl.keys, (const long long*)wl.ptr, cf.dense.mask,
                            cf.dense.weight, c.bound, keep, c.pk, c.cand, chunk_filter(&qf, c));
      });
      if (rc) return rc;
      rc = deliver(h, o, n, topk, po.items.data(), po.scores.data(), po.count.data());
      if (rc) return rc;
      done = true;
    } else {
      std::vector<uint8_t> valid((size_t)total);
      CK(h, cudaMemcpyAsync(valid.data(), d_valid, (size_t)total, cudaMemcpyDeviceToHost, st));
      CK(h, cudaStreamSynchronize(st));
      std::vector<int> nvalid((size_t)n, 0), q0;
      for (int j = 0; j < n; ++j)
        for (long long t = sp[j]; t < sp[j + 1]; ++t) nvalid[j] += valid[(size_t)t] ? 1 : 0;
      ScorePlan b = plan_similar_batch(env, nvalid, topk, &q0);
      if (b.route == ROUTE_BATCH) {
        b.filtered = true;
        rc = similar_groups(h, b, q0, sp.data(), n, topk, valid, d_qf_all, d_qid, cf.dense, flags, tmp, po.items.data(),
                            po.scores.data(), po.count.data(), &qf);
        if (rc) return rc;
        done = true;
      }
    }
  }
  if (!done) {
    // S5, one query at a time: the kernels of long single queries take a dense mask, so the query's filter becomes one
    const size_t ni = (size_t)h->I.n;
    std::vector<uint8_t> m(ni);
    uint8_t* d_m = nullptr;
    CK(h, tmp.alloc(&d_m, ni));
    for (int j = 0; j < n; ++j) {
      const int qj = idx[j];
      if (item_mask) memcpy(m.data(), item_mask, ni);
      else memset(m.data(), 0, ni);
      if (f->set_ix && f->set_ix[qj] >= 0) {
        const uint8_t* row = f->item_sets + (size_t)f->set_ix[qj] * ni;
        for (size_t i = 0; i < ni; ++i) m[i] |= row[i] ? 1 : 0;
      }
      if (f->ex_ptr)
        for (int64_t t = f->ex_ptr[qj]; t < f->ex_ptr[qj + 1]; ++t)
          if (f->ex_items[t] >= 0 && (size_t)f->ex_items[t] < ni) m[f->ex_items[t]] = 1;
      CK(h, cudaMemcpyAsync(d_m, m.data(), ni, cudaMemcpyHostToDevice, st));
      DevFilter fj;
      fj.mask = d_m;
      fj.weight = cf.dense.weight;
      rc = similar_one(h, flat.data() + sp[j], (int)(sp[j + 1] - sp[j]), topk, fj, flags, po.items.data() + (size_t)j * topk,
                       po.scores.data() + (size_t)j * topk, &po.count[j]);
      if (rc) return rc;
      CK(h, cudaStreamSynchronize(st));   // m is rewritten for the next query
    }
  }
  po.scatter(idx, topk, out_items, out_scores, out_count);
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
  Scratch tmp(h->stream);
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
  Scratch tmp(h->stream);
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

// Filtered batch calls: the white-listed queries are scored over their lists, the others scanned with the per-query test
// at the pool insertion (score_plan.h); both parts write the caller's rows.
static bool no_query_filter(const pio_als_query_filter* f) { return !f || (!f->ex_ptr && !f->has_wl && !f->set_ix); }

int pio_als_recommend_filtered(pio_als_handle* h, const int32_t* users, int n, int topk, const uint8_t* item_mask,
                               const double* item_weight, const pio_als_query_filter* f, int32_t* out_items,
                               float* out_scores, int32_t* out_count) {
  if (!h) return PIO_ALS_ERR_ARG;
  if (no_query_filter(f)) return pio_als_recommend(h, users, n, topk, item_mask, item_weight, out_items, out_scores, out_count);
  std::lock_guard<std::mutex> lk(h->mu);
  h->st.last_score_path = 0;
  if (n < 0 || topk < 1) return fail(h, PIO_ALS_ERR_ARG, "topk must be >= 1 and n >= 0");
  if (n == 0) return PIO_ALS_OK;
  if (!users || !out_items || !out_scores) return fail(h, PIO_ALS_ERR_ARG, "null argument");
  if (const char* what = query_filter_error(f, n)) return fail(h, PIO_ALS_ERR_ARG, "%s", what);
  if (!h->U.F || !h->I.F || !h->I.cand_ext) return fail(h, PIO_ALS_ERR_STATE, "no model");
  CK(h, cudaSetDevice(h->cfg.device));
  std::vector<int> listed, scanned;
  split_listed(f->has_wl, n, &listed, &scanned);
  Scratch tmp(h->stream);
  CallFilter cf;
  int rc = upload_call_filter(h, item_mask, item_weight, f, tmp, &cf);
  if (rc) return rc;
  rc = recommend_part(h, users, scanned, false, topk, f, cf, out_items, out_scores, out_count);
  if (rc) return rc;
  return recommend_part(h, users, listed, true, topk, f, cf, out_items, out_scores, out_count);
}

int pio_als_similar_batch_filtered(pio_als_handle* h, const int64_t* q_ptr, const int32_t* q_items, int n_queries, int topk,
                                   const uint8_t* item_mask, const double* item_weight, int flags,
                                   const pio_als_query_filter* f, int32_t* out_items, float* out_scores, int32_t* out_count) {
  if (!h) return PIO_ALS_ERR_ARG;
  if (no_query_filter(f))
    return pio_als_similar_batch(h, q_ptr, q_items, n_queries, topk, item_mask, item_weight, flags, out_items, out_scores,
                                 out_count);
  std::lock_guard<std::mutex> lk(h->mu);
  h->st.last_score_path = 0;
  if (n_queries < 0 || topk < 1) return fail(h, PIO_ALS_ERR_ARG, "topk must be >= 1 and n_queries >= 0");
  if (n_queries == 0) return PIO_ALS_OK;
  if (!q_ptr || !out_items || !out_scores) return fail(h, PIO_ALS_ERR_ARG, "null argument");
  for (int j = 0; j < n_queries; ++j)
    if (q_ptr[j + 1] < q_ptr[j] || (q_ptr[j + 1] > q_ptr[j] && !q_items))
      return fail(h, PIO_ALS_ERR_ARG, "q_ptr must be non-decreasing offsets into q_items");
  if (const char* what = query_filter_error(f, n_queries)) return fail(h, PIO_ALS_ERR_ARG, "%s", what);
  if (!h->I.F || !h->I.cand_ext) return fail(h, PIO_ALS_ERR_STATE, "no model");
  CK(h, cudaSetDevice(h->cfg.device));
  std::vector<int> listed, scanned;
  split_listed(f->has_wl, n_queries, &listed, &scanned);
  Scratch tmp(h->stream);
  CallFilter cf;
  int rc = upload_call_filter(h, item_mask, item_weight, f, tmp, &cf);
  if (rc) return rc;
  const std::vector<int>* parts[2] = {&scanned, &listed};
  for (int part = 0; part < 2; ++part) {
    const std::vector<int>& idx = *parts[part];
    std::vector<int64_t> sp(idx.size() + 1, 0);
    for (size_t i = 0; i < idx.size(); ++i) sp[i + 1] = sp[i] + (q_ptr[idx[i] + 1] - q_ptr[idx[i]]);
    std::vector<int32_t> flat((size_t)sp[idx.size()]);
    for (size_t i = 0; i < idx.size(); ++i)
      if (sp[i + 1] > sp[i]) memcpy(flat.data() + sp[i], q_items + q_ptr[idx[i]], sizeof(int32_t) * (size_t)(sp[i + 1] - sp[i]));
    rc = similar_part(h, sp, flat, idx, part == 1, topk, item_mask, f, cf, flags, out_items, out_scores, out_count);
    if (rc) return rc;
  }
  return PIO_ALS_OK;
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
      Scratch tmp(h->stream);
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

// a status-returning call: return its status unless it is PIO_ALS_OK
#define EVF(call)                          \
  do {                                     \
    const int rc_ = (call);                \
    if (rc_ != PIO_ALS_OK) return rc_;     \
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
      chol_lockstep<N>(sm + grp * LL::STRIDE, bvec + grp * (N > 64 ? N : 80), ridge, N, colbuf + grp * 80,
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
  CallMem tmp(0);
  float *dA = nullptr, *db = nullptr, *dx = nullptr;
  int* dfail = nullptr;
  CK0(tmp.device(&dA, (size_t)n * N * N));
  CK0(tmp.device(&db, (size_t)n * N));
  CK0(tmp.device(&dx, (size_t)n * N));
  CK0(tmp.device(&dfail, 1));
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
  CK0(tmp.event(&e0));
  CK0(tmp.event(&e1));
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
  CK0(cudaGetLastError());
  CK0(cudaDeviceSynchronize());
  float ms = 0.f;
  cudaEventElapsedTime(&ms, e0, e1);
  if (ms_out) *ms_out = ms;
  CK0(cudaMemcpy(x, dx, sizeof(float) * (size_t)n * N, cudaMemcpyDeviceToHost));
  if (fail_out) CK0(cudaMemcpy(fail_out, dfail, sizeof(int), cudaMemcpyDeviceToHost));
  return PIO_ALS_OK;
}

/* debug only (not in pio_als.h): the stable radix sort of sort_scan.cuh on n (key, payload) pairs (HOST buffers, sorted
 * in place) by key bits [0, nbits), read back from whichever half of the ping-pong holds the result.  Used by
 * tests/test_gpu_sort_scan.py. */
__attribute__((visibility("default"))) int pio_debug_radix_sort(int device, uint64_t* keys, uint32_t* vals, int64_t n,
                                                                int nbits) {
  if (!keys || !vals || n < 1 || n >= (1ll << 32) || nbits < 1 || nbits > 64) return PIO_ALS_ERR_ARG;
  CK0(cudaSetDevice(device));
  CallMem tmp(0);
  SortBufs sb;
  for (int i : {0, 1}) {
    CK0(tmp.device(&sb.k[i], (size_t)n));
    CK0(tmp.device(&sb.v[i], (size_t)n));
  }
  CK0(cudaMemcpy(sb.keys(), keys, sizeof(uint64_t) * (size_t)n, cudaMemcpyHostToDevice));
  CK0(cudaMemcpy(sb.vals(), vals, sizeof(uint32_t) * (size_t)n, cudaMemcpyHostToDevice));
  CK0(radix_sort_pairs(sb, (size_t)n, nbits, 0, nullptr));
  CK0(cudaDeviceSynchronize());
  CK0(cudaMemcpy(keys, sb.keys(), sizeof(uint64_t) * (size_t)n, cudaMemcpyDeviceToHost));
  CK0(cudaMemcpy(vals, sb.vals(), sizeof(uint32_t) * (size_t)n, cudaMemcpyDeviceToHost));
  return PIO_ALS_OK;
}

/* debug only (not in pio_als.h): the exclusive uint32 scan of sort_scan.cuh (sums mod 2^32) on n values (HOST buffers),
 * out of place, or in place on one device buffer when in_place != 0.  Used by tests/test_gpu_sort_scan.py. */
__attribute__((visibility("default"))) int pio_debug_scan_u32(int device, const uint32_t* in, uint32_t* out, int64_t n,
                                                              int in_place) {
  if (!in || !out || n < 1) return PIO_ALS_ERR_ARG;
  CK0(cudaSetDevice(device));
  CallMem tmp(0);
  uint32_t *din = nullptr, *dout = nullptr;
  CK0(tmp.device(&din, (size_t)n));
  if (in_place) dout = din;
  else CK0(tmp.device(&dout, (size_t)n));
  CK0(cudaMemcpy(din, in, sizeof(uint32_t) * (size_t)n, cudaMemcpyHostToDevice));
  CK0(scan_exclusive_u32(din, dout, (size_t)n, 0, nullptr));
  CK0(cudaDeviceSynchronize());
  CK0(cudaMemcpy(out, dout, sizeof(uint32_t) * (size_t)n, cudaMemcpyDeviceToHost));
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
  SortBufs sb;
  uint32_t *f1 = nullptr, *f2 = nullptr, *run_start = nullptr, *head = nullptr, *ishead = nullptr, *firstpos = nullptr,
           *isfirst = nullptr;
  CallMem tmp(st);
  for (uint64_t** p : {&sb.k[0], &sb.k[1]}) CK0(tmp.device(p, (size_t)n));
  for (uint32_t** p : {&sb.v[0], &sb.v[1], &f1, &f2, &run_start, &head, &ishead, &firstpos, &isfirst})
    CK0(tmp.device(p, (size_t)n));
  ids_hash_kernel<<<nblk(n, 256), 256, 0, st>>>(d_bytes, d_off, n, sb.keys(), sb.vals(), ids_hash_mask());
  CK0(radix_sort_pairs(sb, (size_t)n, 64, st, nullptr));
  const uint64_t* ks = sb.keys();
  const uint32_t* vs = sb.vals();
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

// ids_encode_device over the host string column (bytes, offsets[0..n]), uploaded on st: *d_index and, when d_first is
// not null, *d_first (n entries each) are allocated in tmp.  0 < n < 2^32, offsets[0] == 0.
static int ids_encode_host(CallMem& tmp, cudaStream_t st, const uint8_t* bytes, const int64_t* offsets, int64_t n,
                           int** d_index, long long** d_first, int64_t* n_unique) {
  const size_t nb = (size_t)offsets[n];
  uint8_t* d_bytes = nullptr;
  long long* d_off = nullptr;
  CK0(tmp.device(&d_bytes, nb));
  CK0(tmp.device(&d_off, (size_t)n + 1));
  CK0(tmp.device(d_index, (size_t)n));
  if (d_first) CK0(tmp.device(d_first, (size_t)n));
  CK0(cudaMemcpyAsync(d_bytes, bytes, nb, cudaMemcpyHostToDevice, st));
  CK0(cudaMemcpyAsync(d_off, offsets, sizeof(long long) * ((size_t)n + 1), cudaMemcpyHostToDevice, st));
  return ids_encode_device(d_bytes, d_off, n, st, *d_index, d_first ? *d_first : nullptr, n_unique);
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
  long long* d_first = nullptr;
  int* d_out = nullptr;
  cudaStream_t st = 0;
  CallMem tmp(st);
  int64_t nuniq = 0;
  const int rc = ids_encode_host(tmp, st, bytes, offsets, n, &d_out, out_first ? &d_first : nullptr, &nuniq);
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

// where pio_events_scan and pio_events_scan_keys put the matched events: host columns of `capacity` events, n taken
struct EvHostCols {
  int64_t capacity;
  int64_t* line;
  int32_t* code;
  double* value;
  uint8_t* flags;
  int64_t* time_us;
  uint8_t* eid_bytes;
  int64_t* eid_off;
  uint8_t* tid_bytes;
  int64_t* tid_off;
  int64_t n;
};

// the lines a scan leaves to the host, in line order: line number (line may be NULL) and byte range without the
// terminator, for the first `capacity`; n counts every one
struct EvFallback {
  int64_t capacity;
  int64_t* line;
  int64_t* begin;
  int64_t* end;
  int64_t n;
};

// where pio_events_scan_props puts the UTC offsets and records of the matched events (host buffers; capacities are
// rec_capacity records and byte_capacity key / token bytes), and the records and bytes taken so far
struct EvPropArgs {
  int16_t* out_utc_off;     // per event
  int64_t* out_prop_off;    // per event, and the closing entry
  int64_t rec_capacity, byte_capacity;
  uint8_t* out_key_bytes;
  int64_t* out_key_off;     // per record, and the closing entry
  uint8_t* out_tok_bytes;
  int64_t* out_tok_off;
  int64_t n_rec, n_key, n_tok;
};

// one parsed chunk: matched events, fallback lines, entityId, targetEntityId and token bytes, records
struct EvTotals {
  int64_t nm, nf, eb, tb, tk, nr;
};

// the checks of a scan's filter or an index view, made before any CUDA call
static int ev_check_filter(const pio_events_filter* f) {
  if (f->n_event_names < 0 || (f->n_event_names > 0 && !f->event_names))
    return fail(nullptr, PIO_ALS_ERR_ARG, "bad event name list");
  for (int k = 0; k < f->n_event_names; ++k)
    if (!f->event_names[k]) return fail(nullptr, PIO_ALS_ERR_ARG, "event name %d is NULL", k);
  if (f->target_entity_type_mode < PIO_EVENTS_TARGET_ANY || f->target_entity_type_mode > PIO_EVENTS_TARGET_EQUALS ||
      (f->target_entity_type_mode == PIO_EVENTS_TARGET_EQUALS && !f->target_entity_type))
    return fail(nullptr, PIO_ALS_ERR_ARG, "bad target_entity_type_mode / target_entity_type");
  return PIO_ALS_OK;
}

// the filter's strings and the nk tracked keys on the device, in tmp: the parse kernels' filter and key list
static int ev_upload_filter(const pio_events_filter* f, const char* const* keys, int nk, CallMem& tmp, ev::Filter* df,
                            ev::KeyList* dk) {
  // packed: entity type | target entity type | property | names... | keys...
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
  std::vector<int> koff(1, (int)fbytes.size());
  for (int q = 0; q < nk; ++q) {
    put(keys[q]);
    koff.push_back((int)fbytes.size());
  }
  uint8_t* d_fbytes = nullptr;
  int *d_noff = nullptr, *d_koff = nullptr;
  CK0(tmp.device(&d_fbytes, fbytes.size()));
  CK0(tmp.device(&d_noff, noff.size()));
  CK0(tmp.device(&d_koff, koff.size()));
  if (!fbytes.empty()) CK0(cudaMemcpy(d_fbytes, fbytes.data(), fbytes.size(), cudaMemcpyHostToDevice));
  CK0(cudaMemcpy(d_noff, noff.data(), sizeof(int) * noff.size(), cudaMemcpyHostToDevice));
  CK0(cudaMemcpy(d_koff, koff.data(), sizeof(int) * koff.size(), cudaMemcpyHostToDevice));
  df->entity_type = d_fbytes + at_et;
  df->entity_type_len = len_et;
  df->names = d_fbytes;
  df->name_off = d_noff;
  df->n_names = f->event_names ? f->n_event_names : -1;   // NULL: any name; an empty list: none
  df->target_mode = f->target_entity_type_mode;
  df->target = d_fbytes + at_tt;
  df->target_len = len_tt;
  df->prop = d_fbytes + at_pr;
  df->prop_len = len_pr;
  df->has_start = f->has_start != 0;
  df->has_until = f->has_until != 0;
  df->start_us = f->start_us;
  df->until_us = f->until_us;
  dk->names = d_fbytes;
  dk->off = d_koff;
  dk->n = nk;
  return PIO_ALS_OK;
}

// the parse and compaction kernels of a scan with (keys) or without tracked keys; smem: the parse that stages its lines
// in shared memory
struct EvKernels {
  decltype(&ev_parse_kernel<false>) parse;
  decltype(&ev_compact_kernel<false>) compact;
};
static EvKernels ev_kernels(bool keys, bool all, bool smem) {
  if (keys) return {smem ? ev_parse_smem_kernel<true> : ev_parse_kernel<true>, ev_compact_kernel<true>};
  if (all)
    return {smem ? ev_parse_smem_kernel<false, true> : ev_parse_kernel<false, true>, ev_compact_kernel<false, true>};
  return {smem ? ev_parse_smem_kernel<false> : ev_parse_kernel<false>, ev_compact_kernel<false>};
}

// Delivery into host columns: a parsed chunk's matched events, and with ka their key columns, after those of the chunks
// before it (here: its id bytes; K.tok_base: its token bytes).  The offset columns are closed after each chunk; the
// next chunk's first event overwrites the closing entries with the same values.
static int ev_take_host(EvHostCols& c, const EvKeyArgs* ka, const EvOut& o, const EvKeys& K, const EvBase& here,
                        const EvTotals& tot, cudaStream_t st) {
  const int64_t n = c.n, nm = tot.nm;
  if (n + nm > c.capacity) return fail(nullptr, PIO_ALS_ERR_ARG, "more matched events than capacity");
  CK0(cudaMemcpyAsync(c.line + n, o.line, 8 * nm, cudaMemcpyDeviceToHost, st));
  CK0(cudaMemcpyAsync(c.code + n, o.code, 4 * nm, cudaMemcpyDeviceToHost, st));
  CK0(cudaMemcpyAsync(c.value + n, o.value, 8 * nm, cudaMemcpyDeviceToHost, st));
  CK0(cudaMemcpyAsync(c.flags + n, o.flags, nm, cudaMemcpyDeviceToHost, st));
  CK0(cudaMemcpyAsync(c.time_us + n, o.time_us, 8 * nm, cudaMemcpyDeviceToHost, st));
  CK0(cudaMemcpyAsync(c.eid_off + n, o.eid_off, 8 * nm, cudaMemcpyDeviceToHost, st));
  CK0(cudaMemcpyAsync(c.tid_off + n, o.tid_off, 8 * nm, cudaMemcpyDeviceToHost, st));
  CK0(cudaMemcpyAsync(c.eid_bytes + here.eid, o.eid_bytes, tot.eb, cudaMemcpyDeviceToHost, st));
  CK0(cudaMemcpyAsync(c.tid_bytes + here.tid, o.tid_bytes, tot.tb, cudaMemcpyDeviceToHost, st));
  c.n += nm;
  c.eid_off[c.n] = here.eid + tot.eb, c.tid_off[c.n] = here.tid + tot.tb;
  if (ka) {
    const int nk = ka->n;
    CK0(cudaMemcpyAsync(ka->out_present + n, K.o_present, nm, cudaMemcpyDeviceToHost, st));
    CK0(cudaMemcpyAsync(ka->out_number + n, K.o_number, nm, cudaMemcpyDeviceToHost, st));
    CK0(cudaMemcpyAsync(ka->out_num + n * nk, K.o_num, 8 * nm * nk, cudaMemcpyDeviceToHost, st));
    CK0(cudaMemcpyAsync(ka->out_tok_off + n * nk, K.o_tok_off, 8 * nm * nk, cudaMemcpyDeviceToHost, st));
    CK0(cudaMemcpyAsync(ka->out_tok_bytes + K.tok_base, K.o_tok, tot.tk, cudaMemcpyDeviceToHost, st));
    ka->out_tok_off[c.n * nk] = K.tok_base + tot.tk;
  }
  return PIO_ALS_OK;
}

// Delivery of the whole-map scan: ev_take_host's columns, each event's UTC offset and first record, and the chunk's
// tot.nr records (per line: P.n_rec at P.rec_pos), walked out of the text t, their decoded keys and raw value tokens
// placed by two scans and copied to the host after the records of the chunks before it.
static int ev_take_props(EvHostCols& c, EvPropArgs* pa, const EvOut& o, const EvKeys& K, const EvProps& P,
                         const uint8_t* t, const uint32_t* starts, long long nl, const EvBase& here, const EvTotals& tot,
                         cudaStream_t st) {
  const int64_t n = c.n, nm = tot.nm, nr = tot.nr;
  if (pa->n_rec + nr > pa->rec_capacity) return fail(nullptr, PIO_ALS_ERR_ARG, "more records than rec_capacity");
  const int rc = ev_take_host(c, nullptr, o, K, here, tot, st);
  if (rc != PIO_ALS_OK) return rc;
  CK0(cudaMemcpyAsync(pa->out_utc_off + n, P.o_utc_off, 2 * nm, cudaMemcpyDeviceToHost, st));
  CK0(cudaMemcpyAsync(pa->out_prop_off + n, P.o_prop_off, 8 * nm, cudaMemcpyDeviceToHost, st));
  pa->out_prop_off[c.n] = pa->n_rec + nr;
  if (nr == 0) return PIO_ALS_OK;
  Scratch sc(st);
  EvRecs R;
  for (uint32_t** p : {&R.kb, &R.ke, &R.vb, &R.k_len, &R.v_len, &R.k_pos, &R.v_pos}) CK0(sc.alloc(p, (size_t)nr));
  uint32_t* d_tot = nullptr;
  CK0(sc.alloc(&d_tot, 2));
  ev_props_emit_kernel<<<nblk(nl, EV_THREADS), EV_THREADS, 0, st>>>(t, starts, nl, P, R);
  CK0(cudaGetLastError());
  CK0(scan_exclusive_u32(R.k_len, R.k_pos, (size_t)nr, st, nullptr));
  CK0(scan_exclusive_u32(R.v_len, R.v_pos, (size_t)nr, st, nullptr));
  ev_props_totals_kernel<<<1, 1, 0, st>>>(R, nr, d_tot);
  uint32_t h_tot[2];
  CK0(cudaMemcpyAsync(h_tot, d_tot, sizeof h_tot, cudaMemcpyDeviceToHost, st));
  CK0(cudaStreamSynchronize(st));
  const int64_t kb = h_tot[0], vb = h_tot[1];
  if (pa->n_key + kb > pa->byte_capacity || pa->n_tok + vb > pa->byte_capacity)
    return fail(nullptr, PIO_ALS_ERR_ARG, "more key or token bytes than n_bytes");
  uint8_t *o_key = nullptr, *o_tok = nullptr;
  long long *o_key_off = nullptr, *o_tok_off = nullptr;
  CK0(sc.alloc(&o_key, (size_t)kb));
  CK0(sc.alloc(&o_tok, (size_t)vb));
  CK0(sc.alloc(&o_key_off, (size_t)nr));
  CK0(sc.alloc(&o_tok_off, (size_t)nr));
  ev_props_copy_kernel<<<nblk(nr, EV_THREADS), EV_THREADS, 0, st>>>(t, nr, R, pa->n_key, pa->n_tok, o_key_off, o_key,
                                                                    o_tok_off, o_tok);
  CK0(cudaGetLastError());
  CK0(cudaMemcpyAsync(pa->out_key_off + pa->n_rec, o_key_off, 8 * nr, cudaMemcpyDeviceToHost, st));
  CK0(cudaMemcpyAsync(pa->out_tok_off + pa->n_rec, o_tok_off, 8 * nr, cudaMemcpyDeviceToHost, st));
  CK0(cudaMemcpyAsync(pa->out_key_bytes + pa->n_key, o_key, (size_t)kb, cudaMemcpyDeviceToHost, st));
  CK0(cudaMemcpyAsync(pa->out_tok_bytes + pa->n_tok, o_tok, (size_t)vb, cudaMemcpyDeviceToHost, st));
  pa->n_rec += nr, pa->n_key += kb, pa->n_tok += vb;
  pa->out_key_off[pa->n_rec] = pa->n_key, pa->out_tok_off[pa->n_rec] = pa->n_tok;
  return PIO_ALS_OK;
}

// ---- event index (pio_events_index_*; events_index.cuh) --------------------------------------------------------------
// the entry columns of a run, n entries each, and their entry sizes (the arena, of arena_bytes, is apart)
struct EixCol {
  void** p;
  size_t size;
};
static std::array<EixCol, 6> eix_cols(EixRun& r) {
  return {{{(void**)&r.hash, sizeof *r.hash}, {(void**)&r.time_us, sizeof *r.time_us}, {(void**)&r.off, sizeof *r.off},
           {(void**)&r.len, sizeof *r.len}, {(void**)&r.id_off, sizeof *r.id_off}, {(void**)&r.id_len, sizeof *r.id_len}}};
}

static void eix_free(EixRun& r) {
  for (const EixCol& c : eix_cols(r)) cudaFree(*c.p);
  cudaFree(r.arena);
  r = EixRun{};
}

// device arrays of a run for n entries and `bytes` arena bytes (bytes < 0: no arena); nothing is copied
static cudaError_t eix_alloc(EixRun& r, long long n, long long bytes) {
  const size_t m = n > 0 ? (size_t)n : 1;
  for (const EixCol& c : eix_cols(r)) {
    const cudaError_t e = cudaMalloc(c.p, c.size * m);
    if (e != cudaSuccess) return e;
  }
  return bytes < 0 ? cudaSuccess : cudaMalloc((void**)&r.arena, bytes > 0 ? (size_t)bytes : 1);
}

// The entries of one append in file order, grown chunk by chunk: ev_scan puts a chunk's matched events here instead of
// copying them to the host.  The arena is the scan's entityId column.  The batch owns its run.
struct EixBatch {
  EixRun r;
  long long cap_n = 0, cap_bytes = 0;
  long long file_base = 0;   // file offset of the scanned text's first byte
  uint64_t mask = ~0ull;
  EixBatch() = default;
  EixBatch(const EixBatch&) = delete;
  EixBatch& operator=(const EixBatch&) = delete;
  ~EixBatch() { eix_free(r); }
};

static int eix_reserve(EixBatch* b, long long n, long long bytes, cudaStream_t st) {
  if (n <= b->cap_n && bytes <= b->cap_bytes) return PIO_ALS_OK;
  const long long cn = n > 2 * b->cap_n ? n : 2 * b->cap_n, cb = bytes > 2 * b->cap_bytes ? bytes : 2 * b->cap_bytes;
  EixRun g;
  cudaError_t e = eix_alloc(g, cn, cb);
  const auto to = eix_cols(g), from = eix_cols(b->r);
  for (size_t k = 0; k < to.size() && e == cudaSuccess; ++k)
    e = cudaMemcpyAsync(*to[k].p, *from[k].p, to[k].size * (size_t)b->r.n, cudaMemcpyDeviceToDevice, st);
  if (e == cudaSuccess) e = cudaMemcpyAsync(g.arena, b->r.arena, (size_t)b->r.arena_bytes, cudaMemcpyDeviceToDevice, st);
  if (e == cudaSuccess) e = cudaStreamSynchronize(st);
  if (e != cudaSuccess) {
    eix_free(g);
    return fail(nullptr, PIO_ALS_ERR_CUDA, "event index: %s", cudaGetErrorString(e));
  }
  g.n = b->r.n;
  g.arena_bytes = b->r.arena_bytes;
  eix_free(b->r);
  b->r = g;
  b->cap_n = cn, b->cap_bytes = cb;
  return PIO_ALS_OK;
}

// Delivery into an index batch: one chunk's nm matched events (o, line order) and their eb id bytes, which start at
// eid_base in the call's id column
static int eix_take_chunk(EixBatch* b, const EvOut& o, const uint8_t* t, const uint32_t* starts, const EvBase& here,
                          long long eid_base, int64_t nm, int64_t eb, cudaStream_t st) {
  if (nm == 0) return PIO_ALS_OK;
  const int rc = eix_reserve(b, b->r.n + nm, eid_base + eb, st);
  if (rc != PIO_ALS_OK) return rc;
  CK0(cudaMemcpyAsync(b->r.arena + eid_base, o.eid_bytes, (size_t)eb, cudaMemcpyDeviceToDevice, st));
  eix_take_kernel<<<nblk(nm, 256), 256, 0, st>>>(o, t, starts, nm, here.line, b->file_base + here.byte, eid_base + eb,
                                                 b->mask, b->r, b->r.n);
  CK0(cudaGetLastError());
  b->r.n += nm;
  b->r.arena_bytes = eid_base + eb;
  return PIO_ALS_OK;
}

// The chunk loop of every event scan, over text[0, n_bytes) (n_bytes > 0, f checked): cuts the text into device chunks,
// stages each through pinned memory on a copy stream, and parses, scans and compacts it on the scan stream.  Each
// chunk's matched events are delivered to the host columns `cols` (with ka: and their key columns) or, when batch is
// set, into that index batch; with pa, the host columns and every key of `properties` as records (ka is then NULL).
// Lines longer than a chunk and the lines the device leaves to the host go to *fb.
static int ev_scan(int device, const uint8_t* text, int64_t n_bytes, const pio_events_filter* f, const EvKeyArgs* ka,
                   EvPropArgs* pa, EvHostCols* cols, EixBatch* batch, EvFallback* fb, int64_t* n_lines) {
  CK0(cudaSetDevice(device));
  int64_t cap = 64ll << 20;   // device chunk; PIO_EVENTS_DEVICE_CHUNK (bytes) lets tests straddle its boundaries
  if (const char* c = getenv("PIO_EVENTS_DEVICE_CHUNK")) {
    const long long v = atoll(c);
    if (v >= 1 && v <= (1ll << 30)) cap = v;
  }
  if (cap > n_bytes) cap = n_bytes;

  CallMem tmp;
  cudaStream_t ex = nullptr, cp = nullptr;   // scan, host-to-device copies
  // copy begin / end per staging slot, then on the scan stream: kernels before and after the line count, and the
  // device-to-host copies (pio_events_debug_timing)
  cudaEvent_t evs[10] = {};
  cudaEvent_t *h2d_begin = evs, *copied = evs + 2, &k0 = evs[4], &k1 = evs[5], &k2 = evs[6], &k3 = evs[7],
              &d0 = evs[8], &d1 = evs[9];
  CK0(tmp.stream(&ex));
  CK0(tmp.stream(&cp));
  for (cudaEvent_t& e : evs) CK0(tmp.event(&e));
  EvTiming& tm = g_ev_timing;
  tm = EvTiming{};
  bool use_smem = true;   // PIO_EVENTS_SMEM=0: the parse reads its lines from global memory (A/B measurements)
  if (const char* c = getenv("PIO_EVENTS_SMEM")) use_smem = atoi(c) != 0;
  const EvKernels kn = ev_kernels(ka != nullptr, pa != nullptr, use_smem);
  if (use_smem) CK0(cudaFuncSetAttribute(kn.parse, cudaFuncAttributeMaxDynamicSharedMemorySize, EV_SMEM_BYTES));
  uint8_t *d_text[2] = {nullptr, nullptr}, *stage[2] = {nullptr, nullptr}, *d_scratch = nullptr;
  uint32_t *d_flag = nullptr, *d_lid = nullptr, *d_tot = nullptr, *h_tot = nullptr;
  for (int k = 0; k < 2; ++k) {
    CK0(tmp.device(&d_text[k], (size_t)cap));
    CK0(tmp.host(&stage[k], (size_t)cap));
  }
  CK0(tmp.device(&d_scratch, (size_t)cap));
  CK0(tmp.device(&d_flag, (size_t)cap));
  CK0(tmp.device(&d_lid, (size_t)cap));
  CK0(tmp.device(&d_tot, 4));
  CK0(tmp.host(&h_tot, 8));
  ev::Filter df;
  EvKeys K{};
  EvProps P{};
  const int nk = ka ? ka->n : 0;
  const int urc = ev_upload_filter(f, ka ? ka->keys : nullptr, nk, tmp, &df, &K.list);
  if (urc != PIO_ALS_OK) return urc;

  EvBase base{0, 0, 0, 0};
  int64_t n_tok = 0;   // token bytes so far
  // lines longer than a chunk, found while cutting the next chunk: written after the current chunk's fallback lines so
  // that the fallback list stays in line order
  std::vector<int64_t> oversized;
  auto flush_oversized = [&]() {
    for (size_t k = 0; k < oversized.size(); k += 3) {
      if (fb->n < fb->capacity) {
        if (fb->line) fb->line[fb->n] = oversized[k];
        fb->begin[fb->n] = oversized[k + 1], fb->end[fb->n] = oversized[k + 2];
      }
      ++fb->n;
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
    const EvBase here = base;   // lines and text bytes before this chunk, and the call's id bytes
    base.line += nl;

    Scratch chunk(ex);
    uint32_t* starts = nullptr;
    EvLines Ls;
    EvOut o;
    const size_t nls = (size_t)nl;
    CK0(chunk.alloc(&starts, nls + 1));
    for (uint32_t** p : {&Ls.is_match, &Ls.is_fb, &Ls.eid_len, &Ls.tid_len, &Ls.match_pos, &Ls.fb_pos, &Ls.eid_pos,
                         &Ls.tid_pos})
      CK0(chunk.alloc(p, nls));
    CK0(chunk.alloc(&Ls.code, nls));
    CK0(chunk.alloc(&Ls.value, nls));
    CK0(chunk.alloc(&Ls.time_us, nls));
    CK0(chunk.alloc(&Ls.flags, nls));
    CK0(chunk.alloc(&o.line, nls));
    CK0(chunk.alloc(&o.code, nls));
    CK0(chunk.alloc(&o.value, nls));
    CK0(chunk.alloc(&o.flags, nls));
    CK0(chunk.alloc(&o.time_us, nls));
    CK0(chunk.alloc(&o.eid_off, nls));
    CK0(chunk.alloc(&o.tid_off, nls));
    CK0(chunk.alloc(&o.fb_line, nls));
    CK0(chunk.alloc(&o.fb_begin, nls));
    CK0(chunk.alloc(&o.fb_end, nls));
    CK0(chunk.alloc(&o.eid_bytes, (size_t)L));
    CK0(chunk.alloc(&o.tid_bytes, (size_t)L));
    if (ka) {
      const size_t nlk = nls * (size_t)nk;
      CK0(chunk.alloc(&K.present, nls));
      CK0(chunk.alloc(&K.number, nls));
      CK0(chunk.alloc(&K.num, nlk));
      CK0(chunk.alloc(&K.tok_b, nlk));
      CK0(chunk.alloc(&K.tok_e, nlk));
      CK0(chunk.alloc(&K.tok_len, nls));
      CK0(chunk.alloc(&K.tok_pos, nls));
      CK0(chunk.alloc(&K.o_present, nls));
      CK0(chunk.alloc(&K.o_number, nls));
      CK0(chunk.alloc(&K.o_num, nlk));
      CK0(chunk.alloc(&K.o_tok_off, nlk));
      CK0(chunk.alloc(&K.o_tok, (size_t)L));   // tokens are disjoint pieces of the chunk's text
      K.tok_base = n_tok;
    }
    if (pa) {
      for (uint32_t** p : {&P.n_rec, &P.rec_pos, &P.obj_b, &P.obj_e}) CK0(chunk.alloc(p, nls));
      CK0(chunk.alloc(&P.utc_off, nls));
      CK0(chunk.alloc(&P.o_utc_off, nls));
      CK0(chunk.alloc(&P.o_prop_off, nls));
      P.rec_base = pa->n_rec;
    }
    CK0(cudaEventRecord(k2, ex));
    ev_start_scatter_kernel<<<nblk(L, EV_THREADS), EV_THREADS, 0, ex>>>(d_flag, d_lid, L, nl, starts);
    const unsigned gl = nblk(nl, EV_THREADS);
    kn.parse<<<gl, EV_THREADS, use_smem ? EV_SMEM_BYTES : 0, ex>>>(t, starts, nl, df, d_scratch, Ls, K, P);
    CK0(cudaGetLastError());
    CK0(scan_exclusive_u32(Ls.is_match, Ls.match_pos, nls, ex, nullptr));
    CK0(scan_exclusive_u32(Ls.is_fb, Ls.fb_pos, nls, ex, nullptr));
    CK0(scan_exclusive_u32(Ls.eid_len, Ls.eid_pos, nls, ex, nullptr));
    CK0(scan_exclusive_u32(Ls.tid_len, Ls.tid_pos, nls, ex, nullptr));
    if (ka) CK0(scan_exclusive_u32(K.tok_len, K.tok_pos, nls, ex, nullptr));
    if (pa) CK0(scan_exclusive_u32(P.n_rec, P.rec_pos, nls, ex, nullptr));
    kn.compact<<<gl, EV_THREADS, 0, ex>>>(t, starts, nl, here, d_scratch, Ls, o, K, P);
    ev_totals_kernel<<<1, 1, 0, ex>>>(Ls, nl, d_tot);
    CK0(cudaGetLastError());
    CK0(cudaEventRecord(k3, ex));
    CK0(cudaMemcpyAsync(h_tot, d_tot, 4 * sizeof(uint32_t), cudaMemcpyDeviceToHost, ex));
    if (ka) {   // token bytes of the chunk: last exclusive position + last length
      CK0(cudaMemcpyAsync(h_tot + 6, K.tok_pos + nl - 1, 4, cudaMemcpyDeviceToHost, ex));
      CK0(cudaMemcpyAsync(h_tot + 7, K.tok_len + nl - 1, 4, cudaMemcpyDeviceToHost, ex));
    }
    if (pa) {   // records of the chunk, the same way
      CK0(cudaMemcpyAsync(h_tot + 6, P.rec_pos + nl - 1, 4, cudaMemcpyDeviceToHost, ex));
      CK0(cudaMemcpyAsync(h_tot + 7, P.n_rec + nl - 1, 4, cudaMemcpyDeviceToHost, ex));
    }
    // find and stage the next chunk while this one is parsed (oversized lines before it belong after this chunk's
    // lines, so their line numbers are assigned only now that this chunk's line count is known)
    int64_t nb, ne;
    next_chunk(ce, &nb, &ne);
    if (nb < ne && prefetch(slot ^ 1, nb, ne) != PIO_ALS_OK) return PIO_ALS_ERR_CUDA;
    CK0(cudaStreamSynchronize(ex));
    const int64_t last = (int64_t)h_tot[6] + h_tot[7];
    const EvTotals tot{h_tot[0], h_tot[1], h_tot[2], h_tot[3], ka ? last : 0, pa ? last : 0};
    CK0(cudaEventRecord(d0, ex));
    const int rc = batch ? eix_take_chunk(batch, o, t, starts, here, here.eid, tot.nm, tot.eb, ex)
                   : pa  ? ev_take_props(*cols, pa, o, K, P, t, starts, nl, here, tot, ex)
                         : ev_take_host(*cols, ka, o, K, here, tot, ex);
    if (rc != PIO_ALS_OK) return rc;
    const int64_t room = fb->capacity - fb->n, nfc = tot.nf < room ? tot.nf : (room > 0 ? room : 0);
    if (nfc > 0) {
      if (fb->line) CK0(cudaMemcpyAsync(fb->line + fb->n, o.fb_line, 8 * nfc, cudaMemcpyDeviceToHost, ex));
      CK0(cudaMemcpyAsync(fb->begin + fb->n, o.fb_begin, 8 * nfc, cudaMemcpyDeviceToHost, ex));
      CK0(cudaMemcpyAsync(fb->end + fb->n, o.fb_end, 8 * nfc, cudaMemcpyDeviceToHost, ex));
    }
    CK0(cudaEventRecord(d1, ex));
    CK0(cudaStreamSynchronize(ex));
    tm.h2d_ms += ms(h2d_begin[slot], copied[slot]);
    tm.kernel_ms += ms(k0, k1) + ms(k2, k3);
    tm.d2h_ms += ms(d0, d1);
    ++tm.chunks;
    fb->n += tot.nf;
    base.eid += tot.eb;
    base.tid += tot.tb;
    n_tok += tot.tk;
    flush_oversized();
    cb = nb, ce = ne;
  }
  if (n_lines) *n_lines = base.line;
  return PIO_ALS_OK;
}

// pio_events_scan (ka, pa == nullptr), pio_events_scan_keys (ka) and pio_events_scan_props (pa): the checks they share,
// then the chunk loop into host columns
static int ev_scan_host(int device, const uint8_t* text, int64_t n_bytes, const pio_events_filter* f,
                        const EvKeyArgs* ka, EvPropArgs* pa, EvHostCols cols, int64_t* out_n_events, EvFallback fb,
                        int64_t* out_n_fallback, int64_t* out_n_lines) {
  if (n_bytes < 0 || (n_bytes > 0 && !text) || !f || fb.capacity < 0 || cols.capacity < n_bytes /
      PIO_EVENTS_MIN_EVENT_BYTES + 1 || !cols.line || !cols.code || !cols.value || !cols.flags || !cols.time_us ||
      !cols.eid_bytes || !cols.eid_off || !cols.tid_bytes || !cols.tid_off || !out_n_events || (fb.capacity > 0 &&
      (!fb.line || !fb.begin || !fb.end)) || !out_n_fallback || !out_n_lines)
    return fail(nullptr, PIO_ALS_ERR_ARG, "bad pio_events_scan arguments");
  int rc = ev_check_filter(f);
  if (rc != PIO_ALS_OK) return rc;
  *out_n_fallback = *out_n_lines = *out_n_events = 0;
  cols.eid_off[0] = cols.tid_off[0] = 0;
  if (ka) ka->out_tok_off[0] = 0;
  if (pa) pa->out_prop_off[0] = pa->out_key_off[0] = pa->out_tok_off[0] = 0;
  if (n_bytes == 0) return PIO_ALS_OK;
  rc = ev_scan(device, text, n_bytes, f, ka, pa, &cols, nullptr, &fb, out_n_lines);
  if (rc != PIO_ALS_OK) return rc;
  *out_n_events = cols.n;
  *out_n_fallback = fb.n;
  return PIO_ALS_OK;
}

int pio_events_scan(int device, const uint8_t* text, int64_t n_bytes, const pio_events_filter* f, int64_t capacity,
                    int64_t* out_line, int32_t* out_code, double* out_value, uint8_t* out_flags, int64_t* out_time_us,
                    uint8_t* out_eid_bytes, int64_t* out_eid_off, uint8_t* out_tid_bytes, int64_t* out_tid_off,
                    int64_t* out_n_events, int64_t fb_capacity, int64_t* out_fb_line, int64_t* out_fb_begin,
                    int64_t* out_fb_end, int64_t* out_n_fallback, int64_t* out_n_lines) {
  const EvHostCols cols{capacity,      out_line,    out_code,      out_value,   out_flags, out_time_us,
                        out_eid_bytes, out_eid_off, out_tid_bytes, out_tid_off, 0};
  return ev_scan_host(device, text, n_bytes, f, nullptr, nullptr, cols, out_n_events,
                      EvFallback{fb_capacity, out_fb_line, out_fb_begin, out_fb_end, 0}, out_n_fallback, out_n_lines);
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
  const EvHostCols cols{capacity,      out_line,    out_code,      out_value,   out_flags, out_time_us,
                        out_eid_bytes, out_eid_off, out_tid_bytes, out_tid_off, 0};
  return ev_scan_host(device, text, n_bytes, f, &ka, nullptr, cols, out_n_events,
                      EvFallback{fb_capacity, out_fb_line, out_fb_begin, out_fb_end, 0}, out_n_fallback, out_n_lines);
}

int pio_events_scan_props(int device, const uint8_t* text, int64_t n_bytes, const pio_events_filter* f,
                          int64_t capacity, int64_t* out_line, int32_t* out_code, double* out_value, uint8_t* out_flags,
                          int64_t* out_time_us, uint8_t* out_eid_bytes, int64_t* out_eid_off, uint8_t* out_tid_bytes,
                          int64_t* out_tid_off, int16_t* out_utc_offset, int64_t* out_prop_off, int64_t rec_capacity,
                          uint8_t* out_key_bytes, int64_t* out_key_off, uint8_t* out_tok_bytes, int64_t* out_tok_off,
                          int64_t* out_n_events, int64_t* out_n_records, int64_t fb_capacity, int64_t* out_fb_line,
                          int64_t* out_fb_begin, int64_t* out_fb_end, int64_t* out_n_fallback, int64_t* out_n_lines) {
  if (n_bytes < 0 || !out_utc_offset || !out_prop_off || rec_capacity < n_bytes / PIO_EVENTS_MIN_RECORD_BYTES + 1 ||
      !out_key_bytes || !out_key_off || !out_tok_bytes || !out_tok_off || !out_n_records)
    return fail(nullptr, PIO_ALS_ERR_ARG, "bad pio_events_scan_props arguments");
  if (!f || f->property) return fail(nullptr, PIO_ALS_ERR_ARG, "pio_events_scan_props: filter->property must be NULL");
  *out_n_records = 0;
  EvPropArgs pa{out_utc_offset, out_prop_off, rec_capacity, n_bytes, out_key_bytes, out_key_off, out_tok_bytes,
                out_tok_off, 0, 0, 0};
  const EvHostCols cols{capacity,      out_line,    out_code,      out_value,   out_flags, out_time_us,
                        out_eid_bytes, out_eid_off, out_tid_bytes, out_tid_off, 0};
  const int rc = ev_scan_host(device, text, n_bytes, f, nullptr, &pa, cols, out_n_events,
                              EvFallback{fb_capacity, out_fb_line, out_fb_begin, out_fb_end, 0}, out_n_fallback,
                              out_n_lines);
  if (rc == PIO_ALS_OK) *out_n_records = pa.n_rec;
  return rc;
}

// ---- $set / $unset / $delete fold (PEventStore.aggregatePropertyColumns; events_fold.cuh) -----------------------------
// PIO_ALS_OK, or the error both folds report for code[e] outside $set / $unset / $delete
static int fold_check_code(const int32_t* code, int64_t e) {
  if (code[e] >= FOLD_SET && code[e] <= FOLD_DELETE) return PIO_ALS_OK;
  return fail(nullptr, PIO_ALS_ERR_ARG, "code[%lld] = %d is not 0 ($set), 1 ($unset) or 2 ($delete)", (long long)e,
              code[e]);
}

// What both folds do before they diverge, for n > 0 checked events: upload them, number their entities, order them by
// (entity, time, line) and reduce that order per entity (fold_reduce_kernel). Device arrays are owned by the caller's
// CallMem.
struct FoldOrder {
  int32_t* code = nullptr;      // [n]
  long long* time = nullptr;    // [n] eventTime, us
  int* ent = nullptr;           // [n] entity of each event, numbered in order of first occurrence
  long long* first = nullptr;   // [n_ent] first event of each entity
  int64_t n_ent = 0;
  SortBufs sorted;              // live half: entity keys and event indices in (entity, time, line) order
  int *seg_first = nullptr, *seg_last = nullptr, *last_set = nullptr, *last_del = nullptr;   // [n_ent], see the kernel
  int* win = nullptr;           // [n_ent x n_keys] last toucher of each tracked key; null when n_keys == 0
};

static int fold_order(CallMem& tmp, cudaStream_t st, const uint8_t* eid_bytes, const int64_t* eid_off,
                      const int32_t* code, const int64_t* time_us, const uint8_t* present, int64_t n, int n_keys,
                      FoldOrder* o) {
  const size_t nn = (size_t)n, nk = (size_t)n_keys;
  uint8_t* d_present = nullptr;
  CK0(tmp.device(&o->code, nn));
  CK0(tmp.device(&o->time, nn));
  for (int i : {0, 1}) {
    CK0(tmp.device(&o->sorted.k[i], nn));
    CK0(tmp.device(&o->sorted.v[i], nn));
  }
  CK0(cudaMemcpyAsync(o->code, code, 4 * nn, cudaMemcpyHostToDevice, st));
  CK0(cudaMemcpyAsync(o->time, time_us, 8 * nn, cudaMemcpyHostToDevice, st));
  if (nk) {
    CK0(tmp.device(&d_present, nn));
    CK0(cudaMemcpyAsync(d_present, present, nn, cudaMemcpyHostToDevice, st));
  }
  const int rc = ids_encode_host(tmp, st, eid_bytes, eid_off, n, &o->ent, &o->first, &o->n_ent);
  if (rc != PIO_ALS_OK) return rc;
  const size_t ne = (size_t)o->n_ent;
  for (int** p : {&o->seg_first, &o->seg_last, &o->last_set, &o->last_del}) CK0(tmp.device(p, ne));
  CK0(cudaMemsetAsync(o->last_set, 0xFF, 4 * ne, st));   // -1: none
  CK0(cudaMemsetAsync(o->last_del, 0xFF, 4 * ne, st));
  if (nk) {
    CK0(tmp.device(&o->win, ne * nk));
    CK0(cudaMemsetAsync(o->win, 0xFF, 4 * ne * nk, st));
  }
  // stable by time, then stable by entity
  SortBufs& s = o->sorted;
  fold_time_key_kernel<<<nblk(n, 256), 256, 0, st>>>(o->time, n, s.keys(), s.vals());
  CK0(radix_sort_pairs(s, nn, 64, st, nullptr));
  fold_entity_key_kernel<<<nblk(n, 256), 256, 0, st>>>(s.vals(), o->ent, n, s.keys());
  CK0(radix_sort_pairs(s, nn, ceil_log2((uint64_t)o->n_ent), st, nullptr));
  fold_reduce_kernel<<<nblk(n, 256), 256, 0, st>>>(s.keys(), s.vals(), o->code, d_present, n_keys, n, o->seg_first,
                                                   o->seg_last, o->last_set, o->last_del, o->win);
  return PIO_ALS_OK;
}

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
    if (const int rc = fold_check_code(code, e)) return rc;
  CK0(cudaSetDevice(device));
  cudaStream_t st = 0;
  CallMem tmp(st);
  FoldOrder o;
  const int rc = fold_order(tmp, st, eid_bytes, eid_off, code, time_us, present, n, n_keys, &o);
  if (rc != PIO_ALS_OK) return rc;
  const size_t ne = (size_t)o.n_ent, nk = (size_t)n_keys;
  uint8_t* d_exists = nullptr;
  long long *d_fus = nullptr, *d_lus = nullptr, *d_win = nullptr;
  CK0(tmp.device(&d_exists, ne));
  CK0(tmp.device(&d_fus, ne)); CK0(tmp.device(&d_lus, ne));
  CK0(tmp.device(&d_win, ne * nk));
  fold_finish_kernel<<<nblk(o.n_ent, 256), 256, 0, st>>>(o.sorted.vals(), o.code, o.time, o.seg_first, o.seg_last,
                                                         o.last_set, o.last_del, o.win, n_keys, o.n_ent, d_exists,
                                                         d_fus, d_lus, d_win);
  CK0(cudaGetLastError());
  CK0(cudaMemcpyAsync(out_first_event, o.first, 8 * ne, cudaMemcpyDeviceToHost, st));
  CK0(cudaMemcpyAsync(out_exists, d_exists, ne, cudaMemcpyDeviceToHost, st));
  CK0(cudaMemcpyAsync(out_first_us, d_fus, 8 * ne, cudaMemcpyDeviceToHost, st));
  CK0(cudaMemcpyAsync(out_last_us, d_lus, 8 * ne, cudaMemcpyDeviceToHost, st));
  if (nk) CK0(cudaMemcpyAsync(out_winner, d_win, 8 * ne * nk, cudaMemcpyDeviceToHost, st));
  CK0(cudaStreamSynchronize(st));
  *out_n_entities = o.n_ent;
  return PIO_ALS_OK;
}

// ---- the fold of every key (PEventStore.aggregatePropertyMaps; events_fold.cuh) ----------------------------------------
int pio_events_fold_props(int device, const uint8_t* eid_bytes, const int64_t* eid_off, const int32_t* code,
                          const int64_t* time_us, const int64_t* prop_off, int64_t n, const uint8_t* key_bytes,
                          const int64_t* key_off, int64_t* out_first_event, uint8_t* out_exists,
                          int64_t* out_first_time_event, int64_t* out_last_time_event, int64_t* out_win_off,
                          int64_t* out_win_rec, int32_t* out_win_key, int64_t* out_key_first, int64_t* out_n_entities,
                          int64_t* out_n_keys) {
  if (n < 0 || !eid_off || !prop_off || !out_n_entities || !out_n_keys ||
      (n > 0 && (!code || !time_us || !out_first_event || !out_exists || !out_first_time_event ||
                 !out_last_time_event || !out_win_off || (!eid_bytes && eid_off[n] > eid_off[0]))))
    return fail(nullptr, PIO_ALS_ERR_ARG, "bad pio_events_fold_props arguments");
  *out_n_entities = *out_n_keys = 0;
  if (n == 0) return PIO_ALS_OK;
  if (n >= (1ll << 31)) return fail(nullptr, PIO_ALS_ERR_ARG, "n must be < 2^31");
  if (eid_off[0] != 0 || prop_off[0] != 0) return fail(nullptr, PIO_ALS_ERR_ARG, "eid_off[0] and prop_off[0] must be 0");
  int64_t max_keys = 0;   // records of the largest event: the bits of an index in one object
  for (int64_t e = 0; e < n; ++e) {
    if (const int rc = fold_check_code(code, e)) return rc;
    if (prop_off[e + 1] < prop_off[e]) return fail(nullptr, PIO_ALS_ERR_ARG, "prop_off must not decrease");
    max_keys = std::max(max_keys, prop_off[e + 1] - prop_off[e]);
  }
  const int64_t nr = prop_off[n];
  if (nr >= (1ll << 31)) return fail(nullptr, PIO_ALS_ERR_ARG, "prop_off[n] must be < 2^31");
  if (nr > 0 && (!key_off || !out_win_rec || !out_win_key || !out_key_first || key_off[0] != 0 ||
                 (!key_bytes && key_off[nr] > 0)))
    return fail(nullptr, PIO_ALS_ERR_ARG, "bad pio_events_fold_props record arguments");
  CK0(cudaSetDevice(device));
  const size_t nn = (size_t)n;
  cudaStream_t st = 0;
  CallMem tmp(st);
  uint8_t* d_exists = nullptr;
  long long *d_fev = nullptr, *d_lev = nullptr, *d_woff = nullptr, *d_prop = nullptr;
  int* last_time = nullptr;
  uint32_t* rank = nullptr;
  CK0(tmp.device(&d_prop, nn + 1));
  CK0(tmp.device(&rank, nn));
  CK0(cudaMemcpyAsync(d_prop, prop_off, 8 * (nn + 1), cudaMemcpyHostToDevice, st));
  FoldOrder o;
  int rc = fold_order(tmp, st, eid_bytes, eid_off, code, time_us, nullptr, n, 0, &o);
  if (rc != PIO_ALS_OK) return rc;
  const int64_t n_ent = o.n_ent;
  const size_t ne = (size_t)n_ent;
  CK0(tmp.device(&last_time, ne));
  CK0(tmp.device(&d_exists, ne));
  CK0(tmp.device(&d_fev, ne)); CK0(tmp.device(&d_lev, ne));
  CK0(tmp.device(&d_woff, ne + 1));
  const uint32_t* vs = o.sorted.vals();
  fold_last_time_kernel<<<nblk(n, 256), 256, 0, st>>>(o.sorted.keys(), vs, o.time, o.seg_last, n, last_time);
  fold_rank_kernel<<<nblk(n, 256), 256, 0, st>>>(vs, n, rank);
  CK0(cudaGetLastError());

  uint32_t* count = nullptr;   // winners per entity, then their exclusive scan: the CSR
  CK0(tmp.device(&count, ne + 1));
  CK0(cudaMemsetAsync(count, 0, 4 * (ne + 1), st));
  int64_t n_kc = 0, nw = 0;
  if (nr > 0) {
    const size_t nrs = (size_t)nr;
    long long *d_kfirst = nullptr, *d_wrec = nullptr;
    int *kcode = nullptr, *seg_unset = nullptr, *seg_set = nullptr, *seg_place = nullptr, *d_wkey = nullptr;
    uint32_t *rec_ev = nullptr, *head = nullptr, *seg_id = nullptr;
    SortBufs r;
    CK0(tmp.device(&rec_ev, nrs));
    CK0(tmp.device(&head, nrs)); CK0(tmp.device(&seg_id, nrs));
    for (int i : {0, 1}) {
      CK0(tmp.device(&r.k[i], nrs));
      CK0(tmp.device(&r.v[i], nrs));
    }
    rc = ids_encode_host(tmp, st, key_bytes, key_off, nr, &kcode, &d_kfirst, &n_kc);   // key codes
    if (rc != PIO_ALS_OK) return rc;
    const int kbits = ceil_log2((uint64_t)n_kc), ebits = ceil_log2((uint64_t)n_ent);
    fold_rec_event_kernel<<<nblk(n, 256), 256, 0, st>>>(d_prop, n, rec_ev);
    // (entity, key, time, line, index in the object): stable by sorted event position, then by (entity, key)
    fold_rec_rank_key_kernel<<<nblk(nr, 256), 256, 0, st>>>(rec_ev, rank, nr, r.keys(), r.vals());
    CK0(radix_sort_pairs(r, nrs, ceil_log2((uint64_t)n), st, nullptr));
    fold_rec_key_kernel<<<nblk(nr, 256), 256, 0, st>>>(r.vals(), rec_ev, o.ent, kcode, kbits, nr, r.keys());
    CK0(radix_sort_pairs(r, nrs, ebits + kbits, st, nullptr));
    const uint64_t* rk = r.keys();
    const uint32_t* rp = r.vals();
    fold_seg_flag_kernel<<<nblk(nr, 256), 256, 0, st>>>(rk, nr, head);
    CK0(scan_exclusive_u32(head, seg_id, nrs, st, nullptr));
    uint32_t last[2] = {0, 0};
    CK0(cudaMemcpyAsync(last, seg_id + nr - 1, 4, cudaMemcpyDeviceToHost, st));
    CK0(cudaMemcpyAsync(last + 1, head + nr - 1, 4, cudaMemcpyDeviceToHost, st));
    CK0(cudaStreamSynchronize(st));
    const int64_t n_seg = (int64_t)last[0] + last[1];
    const size_t nsg = (size_t)n_seg;
    uint32_t *present = nullptr, *w_pos = nullptr;
    CK0(tmp.device(&seg_unset, nsg)); CK0(tmp.device(&seg_set, nsg)); CK0(tmp.device(&seg_place, nsg));
    CK0(tmp.device(&present, nsg)); CK0(tmp.device(&w_pos, nsg));
    CK0(cudaMemsetAsync(seg_unset, 0xFF, 4 * nsg, st));
    CK0(cudaMemsetAsync(seg_set, 0xFF, 4 * nsg, st));
    CK0(cudaMemsetAsync(seg_place, 0x7F, 4 * nsg, st));   // 0x7F7F7F7F: above every position
    fold_props_last_kernel<<<nblk(nr, 256), 256, 0, st>>>(rp, rec_ev, rank, o.code, head, seg_id, nr, seg_unset,
                                                          seg_set);
    fold_props_place_kernel<<<nblk(nr, 256), 256, 0, st>>>(rp, rec_ev, rank, o.code, o.ent, o.last_del, head, seg_id,
                                                           seg_unset, nr, seg_place);
    fold_props_present_kernel<<<nblk(n_seg, 256), 256, 0, st>>>(rp, rec_ev, rank, o.ent, o.last_del, seg_unset,
                                                                seg_set, n_seg, present);
    CK0(cudaGetLastError());
    CK0(scan_exclusive_u32(present, w_pos, nsg, st, nullptr));
    CK0(cudaMemcpyAsync(last, w_pos + n_seg - 1, 4, cudaMemcpyDeviceToHost, st));
    CK0(cudaMemcpyAsync(last + 1, present + n_seg - 1, 4, cudaMemcpyDeviceToHost, st));
    CK0(cudaStreamSynchronize(st));
    nw = (int64_t)last[0] + last[1];
    if (nw > 0) {
      // the winners in dict order, keyed into the spare record half; then they are the data to sort, and the sorted
      // records (rk / rp) are no longer read
      const int ibits = ceil_log2((uint64_t)max_keys);
      fold_props_winner_kernel<<<nblk(n_seg, 256), 256, 0, st>>>(rp, rec_ev, rank, d_prop, present, w_pos, seg_set,
                                                                 seg_place, ibits, n_seg, r.spare_keys(),
                                                                 r.spare_vals());
      r.flip();
      CK0(radix_sort_pairs(r, (size_t)nw, ceil_log2((uint64_t)n) + ibits, st, nullptr));
      CK0(tmp.device(&d_wrec, (size_t)nw));
      CK0(tmp.device(&d_wkey, (size_t)nw));
      fold_props_out_kernel<<<nblk(nw, 256), 256, 0, st>>>(r.vals(), rec_ev, o.ent, kcode, nw, count, d_wrec, d_wkey);
      CK0(cudaGetLastError());
      CK0(cudaMemcpyAsync(out_win_rec, d_wrec, 8 * (size_t)nw, cudaMemcpyDeviceToHost, st));
      CK0(cudaMemcpyAsync(out_win_key, d_wkey, 4 * (size_t)nw, cudaMemcpyDeviceToHost, st));
    }
    CK0(cudaMemcpyAsync(out_key_first, d_kfirst, 8 * (size_t)n_kc, cudaMemcpyDeviceToHost, st));
    CK0(cudaStreamSynchronize(st));
  }
  uint32_t* w_off = nullptr;
  CK0(tmp.device(&w_off, ne + 1));
  CK0(scan_exclusive_u32(count, w_off, ne + 1, st, nullptr));
  fold_props_finish_kernel<<<nblk(n_ent + 1, 256), 256, 0, st>>>(vs, o.seg_first, last_time, o.last_set, o.last_del,
                                                                 w_off, n_ent, d_exists, d_fev, d_lev, d_woff);
  CK0(cudaGetLastError());
  CK0(cudaMemcpyAsync(out_first_event, o.first, 8 * ne, cudaMemcpyDeviceToHost, st));
  CK0(cudaMemcpyAsync(out_exists, d_exists, ne, cudaMemcpyDeviceToHost, st));
  CK0(cudaMemcpyAsync(out_first_time_event, d_fev, 8 * ne, cudaMemcpyDeviceToHost, st));
  CK0(cudaMemcpyAsync(out_last_time_event, d_lev, 8 * ne, cudaMemcpyDeviceToHost, st));
  CK0(cudaMemcpyAsync(out_win_off, d_woff, 8 * (ne + 1), cudaMemcpyDeviceToHost, st));
  CK0(cudaStreamSynchronize(st));
  *out_n_entities = n_ent;
  *out_n_keys = n_kc;
  return PIO_ALS_OK;
}

}  // extern "C"

// ---- event index (LEventStore.findByEntity for one view; events_index.cuh) ---------------------------------------------
struct pio_events_index {
  int device = 0;
  uint64_t mask = ~0ull;                 // ids_hash_mask() when the index was created: build and lookup hash alike
  cudaStream_t st = nullptr;
  std::string entity_type, target;       // the view's strings, owned
  std::vector<std::string> names;
  std::vector<const char*> name_ptrs;
  pio_events_filter view{};
  pio::EixRun main, delta;
  pio_events_index_stats stats{};
  // lookup scratch, grown as needed: query ids, counts, positions, results
  uint8_t* q_bytes = nullptr;
  long long* q_off = nullptr;
  uint32_t *count = nullptr, *pos = nullptr;
  long long* r_off = nullptr;
  int32_t* r_len = nullptr;
  size_t cap_qb = 0, cap_qo = 0, cap_count = 0, cap_pos = 0, cap_roff = 0, cap_rlen = 0;
};

namespace pio {
using Clock = std::chrono::steady_clock;
static double ms_since(Clock::time_point t0) {
  return std::chrono::duration<double, std::milli>(Clock::now() - t0).count();
}

// batch b (entries in file order) -> a run in (hash, time descending, offset ascending) order; b's arena moves into it
static int eix_sort(pio_events_index* ix, EixBatch& b, EixRun* out) {
  const long long n = b.r.n;
  const cudaStream_t st = ix->st;
  CallMem tmp(st);
  SortBufs sb;
  for (int i : {0, 1}) {
    CK0(tmp.device(&sb.k[i], (size_t)n));
    CK0(tmp.device(&sb.v[i], (size_t)n));
  }
  eix_time_key_kernel<<<nblk(n, 256), 256, 0, st>>>(b.r.time_us, n, sb.keys(), sb.vals());
  CK0(radix_sort_pairs(sb, (size_t)n, 64, st, nullptr));
  eix_hash_key_kernel<<<nblk(n, 256), 256, 0, st>>>(sb.vals(), b.r.hash, n, sb.keys());
  CK0(radix_sort_pairs(sb, (size_t)n, 64 - __builtin_clzll(ix->mask), st, nullptr));
  EixRun r;
  const cudaError_t e = eix_alloc(r, n, -1);
  if (e != cudaSuccess) {
    eix_free(r);
    return fail(nullptr, PIO_ALS_ERR_CUDA, "event index: %s", cudaGetErrorString(e));
  }
  r.n = n;
  eix_gather_kernel<<<nblk(n, 256), 256, 0, st>>>(b.r, sb.vals(), r);
  r.arena = b.r.arena, r.arena_bytes = b.r.arena_bytes;
  b.r.arena = nullptr;
  cudaError_t e2 = cudaStreamSynchronize(st);
  if (e2 == cudaSuccess) e2 = cudaGetLastError();
  eix_free(b.r);
  if (e2 != cudaSuccess) {
    eix_free(r);
    return fail(nullptr, PIO_ALS_ERR_CUDA, "event index sort: %s", cudaGetErrorString(e2));
  }
  *out = r;
  return PIO_ALS_OK;
}

// *a = merge(*a, *b); both are consumed
static int eix_merge(pio_events_index* ix, EixRun* a, EixRun* b) {
  if (b->n == 0 || a->n == 0) {
    EixRun& keep = a->n == 0 ? *b : *a;
    EixRun& drop = a->n == 0 ? *a : *b;
    eix_free(drop);
    *a = keep;
    if (&keep == b) *b = EixRun{};
    return PIO_ALS_OK;
  }
  EixRun r;
  const long long n = a->n + b->n;
  const cudaError_t e = eix_alloc(r, n, a->arena_bytes + b->arena_bytes);
  if (e != cudaSuccess) {
    eix_free(r);
    return fail(nullptr, PIO_ALS_ERR_CUDA, "event index merge: %s", cudaGetErrorString(e));
  }
  r.n = n;
  r.arena_bytes = a->arena_bytes + b->arena_bytes;
  CK0(cudaMemcpyAsync(r.arena, a->arena, (size_t)a->arena_bytes, cudaMemcpyDeviceToDevice, ix->st));
  CK0(cudaMemcpyAsync(r.arena + a->arena_bytes, b->arena, (size_t)b->arena_bytes, cudaMemcpyDeviceToDevice, ix->st));
  eix_merge_kernel<<<nblk(n, EIX_MERGE_SPAN), EIX_MERGE_THREADS, 0, ix->st>>>(*a, *b, r);
  CK0(cudaGetLastError());
  CK0(cudaStreamSynchronize(ix->st));
  eix_free(*a);
  eix_free(*b);
  *a = r;
  return PIO_ALS_OK;
}

// sorts a batch into delta, and merges delta into main once it is past 1 / PIO_EVENTS_INDEX_MERGE_DIVISOR of main
static int eix_add_batch(pio_events_index* ix, EixBatch& b) {
  if (b.r.n == 0) return PIO_ALS_OK;
  const auto t0 = Clock::now();
  EixRun r;
  int rc = eix_sort(ix, b, &r);
  if (rc == PIO_ALS_OK) rc = eix_merge(ix, &ix->delta, &r);
  ix->stats.sort_ms = ms_since(t0);
  if (rc != PIO_ALS_OK) return rc;
  if (ix->delta.n * PIO_EVENTS_INDEX_MERGE_DIVISOR > ix->main.n) {
    const auto t1 = Clock::now();
    rc = eix_merge(ix, &ix->main, &ix->delta);
    ix->stats.merge_ms = ms_since(t1);
    ++ix->stats.n_merges;
  }
  ix->stats.n_main = ix->main.n;
  ix->stats.n_delta = ix->delta.n;
  return rc;
}

// a lookup buffer of at least n elements (contents are not kept)
template <typename T>
static cudaError_t eix_grow(T** p, size_t* cap, size_t n) {
  if (n <= *cap) return cudaSuccess;
  const size_t c = n > 2 * *cap ? n : 2 * *cap;
  cudaFree(*p);
  *p = nullptr;
  *cap = 0;
  const cudaError_t e = cudaMalloc((void**)p, c * sizeof(T));
  if (e == cudaSuccess) *cap = c;
  return e;
}
}  // namespace pio

extern "C" {

int pio_events_index_create(int device, const pio_events_filter* view, pio_events_index** out) {
  if (!view || !out) return fail(nullptr, PIO_ALS_ERR_ARG, "bad pio_events_index_create arguments");
  *out = nullptr;
  if (view->property || view->has_start || view->has_until)
    return fail(nullptr, PIO_ALS_ERR_ARG, "an event index view has no property and no time bounds");
  const int rc = ev_check_filter(view);
  if (rc != PIO_ALS_OK) return rc;
  CK0(cudaSetDevice(device));
  auto* ix = new pio_events_index;
  ix->device = device;
  ix->mask = ids_hash_mask();
  if (view->entity_type) ix->entity_type = view->entity_type;
  if (view->target_entity_type_mode == PIO_EVENTS_TARGET_EQUALS) ix->target = view->target_entity_type;
  for (int k = 0; k < view->n_event_names; ++k) ix->names.emplace_back(view->event_names[k]);
  for (const std::string& nm : ix->names) ix->name_ptrs.push_back(nm.c_str());
  ix->view.entity_type = view->entity_type ? ix->entity_type.c_str() : nullptr;
  ix->view.event_names = view->event_names ? (ix->name_ptrs.empty() ? &ix->view.entity_type : ix->name_ptrs.data())
                                           : nullptr;   // an empty list stays non-NULL: no event matches
  ix->view.n_event_names = view->n_event_names;
  ix->view.target_entity_type_mode = view->target_entity_type_mode;
  ix->view.target_entity_type = view->target_entity_type_mode == PIO_EVENTS_TARGET_EQUALS ? ix->target.c_str() : nullptr;
  const cudaError_t e = cudaStreamCreateWithFlags(&ix->st, cudaStreamNonBlocking);
  if (e != cudaSuccess) {
    delete ix;
    return fail(nullptr, PIO_ALS_ERR_CUDA, "cudaStreamCreate: %s", cudaGetErrorString(e));
  }
  *out = ix;
  return PIO_ALS_OK;
}

int pio_events_index_append(pio_events_index* ix, const uint8_t* text, int64_t n_bytes, int64_t base_offset,
                            int64_t fb_capacity, int64_t* out_fb_begin, int64_t* out_fb_end, int64_t* out_n_fallback) {
  if (!ix || n_bytes < 0 || (n_bytes > 0 && !text) || base_offset < 0 || fb_capacity < 0 || !out_n_fallback ||
      (fb_capacity > 0 && (!out_fb_begin || !out_fb_end)))
    return fail(nullptr, PIO_ALS_ERR_ARG, "bad pio_events_index_append arguments");
  *out_n_fallback = 0;
  ix->stats.scan_ms = ix->stats.sort_ms = ix->stats.merge_ms = 0;
  if (n_bytes == 0) return PIO_ALS_OK;
  EixBatch b;
  b.file_base = base_offset;
  b.mask = ix->mask;
  EvFallback fb{fb_capacity, nullptr, out_fb_begin, out_fb_end, 0};
  const auto t0 = Clock::now();
  const int rc = ev_scan(ix->device, text, n_bytes, &ix->view, nullptr, nullptr, nullptr, &b, &fb, nullptr);
  ix->stats.scan_ms = ms_since(t0);
  if (rc != PIO_ALS_OK) return rc;
  *out_n_fallback = fb.n;
  if (fb.n > fb_capacity) return PIO_ALS_OK;   // nothing added; the caller asks again with more room
  return eix_add_batch(ix, b);
}

int pio_events_index_add_host(pio_events_index* ix, const uint8_t* id_bytes, const int64_t* id_off,
                              const int64_t* time_us, const int64_t* offset, const int32_t* length, int64_t n) {
  if (!ix || n < 0 || (n > 0 && (!id_off || !time_us || !offset || !length || id_off[0] != 0 ||
                                 (!id_bytes && id_off[n] > 0))))
    return fail(nullptr, PIO_ALS_ERR_ARG, "bad pio_events_index_add_host arguments");
  if (n >= (1ll << 32)) return fail(nullptr, PIO_ALS_ERR_ARG, "n must be < 2^32");
  for (int64_t k = 0; k < n; ++k)
    if (id_off[k + 1] < id_off[k] || length[k] < 0 || (k > 0 && offset[k] <= offset[k - 1]))
      return fail(nullptr, PIO_ALS_ERR_ARG, "event %lld: id offsets must not decrease and line offsets must increase",
                  (long long)k);
  ix->stats.scan_ms = ix->stats.sort_ms = ix->stats.merge_ms = 0;
  if (n == 0) return PIO_ALS_OK;
  CK0(cudaSetDevice(ix->device));
  EixBatch b;
  const cudaError_t e = eix_alloc(b.r, n, id_off[n]);
  if (e != cudaSuccess) return fail(nullptr, PIO_ALS_ERR_CUDA, "event index: %s", cudaGetErrorString(e));
  b.r.n = n;
  b.r.arena_bytes = id_off[n];
  std::vector<int32_t> id_len((size_t)n);
  for (int64_t k = 0; k < n; ++k) id_len[k] = (int32_t)(id_off[k + 1] - id_off[k]);
  CK0(cudaMemcpyAsync(b.r.arena, id_bytes, (size_t)id_off[n], cudaMemcpyHostToDevice, ix->st));
  const void* from[6] = {nullptr, time_us, offset, length, id_off, id_len.data()};   // in eix_cols order; hashed below
  const auto to = eix_cols(b.r);
  for (size_t k = 1; k < to.size(); ++k)
    CK0(cudaMemcpyAsync(*to[k].p, from[k], to[k].size * (size_t)n, cudaMemcpyHostToDevice, ix->st));
  eix_hash_kernel<<<nblk(n, 256), 256, 0, ix->st>>>(b.r, ix->mask);
  CK0(cudaGetLastError());
  return eix_add_batch(ix, b);
}

int pio_events_index_lookup(pio_events_index* ix, const uint8_t* id_bytes, const int64_t* id_off, int32_t n,
                            int64_t limit, int64_t capacity, int64_t* out_count, int64_t* out_total,
                            int64_t* out_offset, int32_t* out_len) {
  if (!ix || n < 0 || capacity < 0 || !out_total || (n > 0 && (!id_off || !out_count || id_off[0] != 0 ||
      (!id_bytes && id_off[n] > 0))) || (capacity > 0 && (!out_offset || !out_len)))
    return fail(nullptr, PIO_ALS_ERR_ARG, "bad pio_events_index_lookup arguments");
  *out_total = 0;
  if (n == 0) return PIO_ALS_OK;
  CK0(cudaSetDevice(ix->device));
  const cudaStream_t st = ix->st;
  const size_t nb = (size_t)id_off[n], nq = (size_t)n;
  CK0(eix_grow(&ix->q_bytes, &ix->cap_qb, nb ? nb : 1));
  CK0(eix_grow(&ix->q_off, &ix->cap_qo, nq + 1));
  CK0(eix_grow(&ix->count, &ix->cap_count, nq));
  CK0(eix_grow(&ix->pos, &ix->cap_pos, nq));
  CK0(cudaMemcpyAsync(ix->q_bytes, id_bytes, nb, cudaMemcpyHostToDevice, st));
  CK0(cudaMemcpyAsync(ix->q_off, id_off, 8 * (nq + 1), cudaMemcpyHostToDevice, st));
  const unsigned grid = nblk(n, EIX_LOOKUP_WARPS);
  eix_count_kernel<<<grid, 32 * EIX_LOOKUP_WARPS, 0, st>>>(ix->main, ix->delta, ix->q_bytes, ix->q_off, n, ix->mask,
                                                            limit, ix->count);
  CK0(cudaGetLastError());
  CK0(scan_exclusive_u32(ix->count, ix->pos, nq, st, nullptr));
  std::vector<uint32_t> cnt(nq);
  CK0(cudaMemcpyAsync(cnt.data(), ix->count, 4 * nq, cudaMemcpyDeviceToHost, st));
  CK0(cudaStreamSynchronize(st));
  int64_t total = 0;
  for (size_t k = 0; k < nq; ++k) total += out_count[k] = cnt[k];
  *out_total = total;
  if (total == 0 || total > capacity) return PIO_ALS_OK;
  if (total >= (1ll << 32)) return fail(nullptr, PIO_ALS_ERR_ARG, "more than 2^32-1 events in one lookup");
  CK0(eix_grow(&ix->r_off, &ix->cap_roff, (size_t)total));
  CK0(eix_grow(&ix->r_len, &ix->cap_rlen, (size_t)total));
  eix_write_kernel<<<grid, 32 * EIX_LOOKUP_WARPS, 0, st>>>(ix->main, ix->delta, ix->q_bytes, ix->q_off, n, ix->mask,
                                                            ix->count, ix->pos, ix->r_off, ix->r_len);
  CK0(cudaGetLastError());
  CK0(cudaMemcpyAsync(out_offset, ix->r_off, 8 * (size_t)total, cudaMemcpyDeviceToHost, st));
  CK0(cudaMemcpyAsync(out_len, ix->r_len, 4 * (size_t)total, cudaMemcpyDeviceToHost, st));
  CK0(cudaStreamSynchronize(st));
  return PIO_ALS_OK;
}

int pio_events_index_get_stats(const pio_events_index* ix, pio_events_index_stats* out) {
  if (!ix || !out) return fail(nullptr, PIO_ALS_ERR_ARG, "bad pio_events_index_get_stats arguments");
  *out = ix->stats;
  return PIO_ALS_OK;
}

int pio_events_index_destroy(pio_events_index* ix) {
  if (!ix) return PIO_ALS_OK;
  cudaSetDevice(ix->device);
  if (ix->st) cudaStreamSynchronize(ix->st);
  eix_free(ix->main);
  eix_free(ix->delta);
  void* ps[6] = {ix->q_bytes, ix->q_off, ix->count, ix->pos, ix->r_off, ix->r_len};
  for (void* q : ps) cudaFree(q);
  if (ix->st) cudaStreamDestroy(ix->st);
  delete ix;
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
  cudaStream_t st = 0;
  CallMem tmp(st);
  int *du = nullptr, *di = nullptr;
  uint64_t* dk = nullptr;
  uint32_t *flag = nullptr, *rank = nullptr;
  SortBufs sb;
  CK0(tmp.device(&du, (size_t)n)); CK0(tmp.device(&di, (size_t)n));
  for (int i : {0, 1}) {
    CK0(tmp.device(&sb.k[i], (size_t)n));
    CK0(tmp.device(&sb.v[i], (size_t)n));
  }
  CK0(tmp.device(&flag, (size_t)n)); CK0(tmp.device(&dk, (size_t)n)); CK0(tmp.device(&rank, (size_t)n));
  CK0(cudaMemcpyAsync(du, user, 4 * (size_t)n, cudaMemcpyHostToDevice, st));
  CK0(cudaMemcpyAsync(di, item, 4 * (size_t)n, cudaMemcpyHostToDevice, st));
  // 1. distinct (user, item), sorted by user then item
  cooc_keys_kernel<<<nblk(n, 256), 256, 0, st>>>(du, di, n, bits_i, sb.keys(), sb.vals());
  CK0(radix_sort_pairs(sb, (size_t)n, bits_u + bits_i, st, nullptr));
  const uint64_t* ks = sb.keys();
  cooc_head_kernel<<<nblk(n, 256), 256, 0, st>>>(ks, n, flag);
  uint32_t lf = 0, lp = 0;
  CK0(cudaMemcpyAsync(&lf, flag + n - 1, 4, cudaMemcpyDeviceToHost, st));
  uint32_t* pos = sb.spare_vals();
  CK0(scan_exclusive_u32(flag, pos, (size_t)n, st, nullptr));
  CK0(cudaMemcpyAsync(&lp, pos + n - 1, 4, cudaMemcpyDeviceToHost, st));
  CK0(cudaStreamSynchronize(st));
  const long long m = (long long)lp + lf;
  cooc_compact_kernel<<<nblk(n, 256), 256, 0, st>>>(ks, flag, pos, n, dk);
  // 2. pairs (item1 < item2) per user; their total is counted in 64 bits and checked before the uint32 scan of the
  // ranks is used as an index
  unsigned long long* dtot = nullptr;
  CK0(tmp.device(&dtot, 1));
  CK0(cudaMemsetAsync(dtot, 0, sizeof(unsigned long long), st));
  cooc_rank_kernel<<<nblk(m, 256), 256, 0, st>>>(dk, m, bits_i, rank, dtot);
  unsigned long long tot = 0;
  CK0(cudaMemcpyAsync(&tot, dtot, sizeof(tot), cudaMemcpyDeviceToHost, st));
  CK0(cudaStreamSynchronize(st));
  if (tot >= (1ull << 31)) return fail(nullptr, PIO_ALS_ERR_ARG, "more than 2^31-1 co-occurrence pairs (%llu)", tot);
  const long long np = (long long)tot;
  uint32_t* off = flag;
  CK0(scan_exclusive_u32(rank, off, (size_t)m, st, nullptr));
  std::vector<int> h_item((size_t)n_items * topn, -1), h_cnt((size_t)n_items * topn, 0), h_n((size_t)n_items, 0);
  if (np > 0) {
    SortBufs ps, rs;
    uint32_t *pf = nullptr, *ppos = nullptr;
    for (int i : {0, 1}) {
      CK0(tmp.device(&ps.k[i], (size_t)np));
      CK0(tmp.device(&ps.v[i], (size_t)np));
    }
    CK0(tmp.device(&pf, (size_t)np)); CK0(tmp.device(&ppos, (size_t)np));
    cooc_pairs_kernel<<<nblk(m, 256), 256, 0, st>>>(dk, rank, off, m, bits_i, ps.keys(), ps.vals());
    CK0(radix_sort_pairs(ps, (size_t)np, 2 * bits_i, st, nullptr));
    const uint64_t* pks = ps.keys();
    cooc_head_kernel<<<nblk(np, 256), 256, 0, st>>>(pks, np, pf);
    uint32_t cf = 0, cp = 0;
    CK0(cudaMemcpyAsync(&cf, pf + np - 1, 4, cudaMemcpyDeviceToHost, st));
    CK0(scan_exclusive_u32(pf, ppos, (size_t)np, st, nullptr));
    CK0(cudaMemcpyAsync(&cp, ppos + np - 1, 4, cudaMemcpyDeviceToHost, st));
    CK0(cudaStreamSynchronize(st));
    const long long C = (long long)cp + cf, n2 = 2 * C;
    // 3. both directions, ranked per item by (count desc, other item asc)
    for (int i : {0, 1}) {
      CK0(tmp.device(&rs.k[i], (size_t)n2));
      CK0(tmp.device(&rs.v[i], (size_t)n2));
    }
    cooc_runs_kernel<<<nblk(np, 256), 256, 0, st>>>(pks, pf, ppos, np, bits_i, bits_c, rs.keys(), rs.vals());
    CK0(radix_sort_pairs(rs, (size_t)n2, 2 * bits_i + bits_c, st, nullptr));
    int *d_oi = nullptr, *d_oc = nullptr, *d_on = nullptr;
    CK0(tmp.device(&d_oi, (size_t)n_items * topn)); CK0(tmp.device(&d_oc, (size_t)n_items * topn));
    CK0(tmp.device(&d_on, (size_t)n_items));
    CK0(cudaMemsetAsync(d_oi, 0xff, 4 * (size_t)n_items * topn, st));
    CK0(cudaMemsetAsync(d_oc, 0, 4 * (size_t)n_items * topn, st));
    CK0(cudaMemsetAsync(d_on, 0, 4 * (size_t)n_items, st));
    cooc_take_kernel<<<nblk(n2, 256), 256, 0, st>>>(rs.keys(), rs.vals(), n2, bits_i, bits_c, topn, d_oi, d_oc, d_on);
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

}  // extern "C"

// ---- co-occurrence batch scoring (similarproduct CooccurrenceAlgorithm.predict) --------------------------------------------
struct pio_cooc_model {
  int device = 0, n_items = 0, topn = 0;
  std::vector<int32_t> top_n;           // sizes a call's parts before any device work
  std::vector<int64_t> row_sum;         // per item, the sum of its counts: a query's scores are at most the sum over its ids
  std::vector<int32_t> items, counts;   // host copies until the first call uploads them
  cudaStream_t st = nullptr;
  int *d_items = nullptr, *d_counts = nullptr, *d_n = nullptr;   // set together, once every copy has landed
  mutable std::mutex mu;                // serialises the calls, and guards stats
  pio_cooc_stats stats{};
};

namespace pio {

// A call's parts: consecutive queries [first[p], first[p + 1]).  A part closes before the query that would take its
// listed expansion over the budget or its listed ids past 2^31 - 1; each part holds at least one query.
struct CoocPlan {
  std::vector<int> first;
  std::vector<uint64_t> bound;   // per part, the largest score bound of its queries
};
static int cooc_plan(const pio_cooc_model* m, const int64_t* q_ptr, const int32_t* q_items, int n, long long budget,
                     CoocPlan* p) {
  long long acc = 0, acc_ids = 0;
  for (int j = 0; j < n; ++j) {
    unsigned long long ex = 0, bound = 0;
    for (int64_t t = q_ptr[j]; t < q_ptr[j + 1]; ++t) {
      const int32_t it = q_items[t];
      if (it < 0 || it >= m->n_items) continue;
      ex += (unsigned)m->top_n[it];
      bound += (unsigned long long)m->row_sum[it];
    }
    const long long ids = q_ptr[j + 1] - q_ptr[j];
    if (ex >= (1ull << 32))
      return fail(nullptr, PIO_ALS_ERR_ARG, "query %d expands to %llu entries: at most 2^32 - 1 fit one part", j, ex);
    if (ids >= (1ll << 31)) return fail(nullptr, PIO_ALS_ERR_ARG, "query %d lists 2^31 or more ids", j);
    if (j == 0 || acc + (long long)ex > budget || acc_ids + ids >= (1ll << 31)) {
      p->first.push_back(j);
      p->bound.push_back(0);
      acc = acc_ids = 0;
    }
    acc += (long long)ex;
    acc_ids += ids;
    p->bound.back() = std::max<uint64_t>(p->bound.back(), bound);
  }
  p->first.push_back(n);
  return PIO_ALS_OK;
}

// The model's device copy, made on its own stream by the first call.  The device pointers are published only after the
// copies have completed, so a failed upload leaves nothing half made: its allocations are freed and the next call
// starts over.
static int cooc_upload(pio_cooc_model* m, const FilterEnv& env) {
  if (m->d_items) return PIO_ALS_OK;
  if (!m->st) CKF(env, cudaStreamCreateWithFlags(&m->st, cudaStreamNonBlocking));
  const size_t cells = (size_t)m->n_items * m->topn;
  const size_t len[3] = {cells, cells, (size_t)m->n_items};
  const int32_t* src[3] = {m->items.data(), m->counts.data(), m->top_n.data()};
  int* d[3] = {nullptr, nullptr, nullptr};
  cudaError_t e = cudaSuccess;
  for (int k = 0; k < 3 && e == cudaSuccess; ++k) e = cudaMalloc((void**)&d[k], sizeof(int) * len[k]);
  for (int k = 0; k < 3 && e == cudaSuccess; ++k)
    e = cudaMemcpyAsync(d[k], src[k], sizeof(int) * len[k], cudaMemcpyHostToDevice, m->st);
  if (e == cudaSuccess) e = cudaStreamSynchronize(m->st);   // the host copies are read until here
  if (e != cudaSuccess) {
    cudaStreamSynchronize(m->st);
    for (int* p : d)
      if (p) cudaFree(p);
    return fail_to(env.err, PIO_ALS_ERR_CUDA, "uploading the co-occurrence model: %s", cudaGetErrorString(e));
  }
  m->d_items = d[0], m->d_counts = d[1], m->d_n = d[2];
  std::vector<int32_t>().swap(m->items);
  std::vector<int32_t>().swap(m->counts);
  return PIO_ALS_OK;
}

// the queries [j0, j1) of a call: rows j0 .. j1 - 1 of the caller's outputs
static int cooc_part(pio_cooc_model* m, const FilterEnv& env, const int64_t* q_ptr, const int32_t* q_items, int j0, int j1,
                     int topk, uint64_t bound, const pio_als_query_filter* f, const CallFilter& cf, int32_t* out_items,
                     int64_t* out_scores, int32_t* out_count) {
  const int n = j1 - j0;
  cudaStream_t st = m->st;
  Scratch tmp(st);
  std::vector<int> idx((size_t)n);
  for (int i = 0; i < n; ++i) idx[i] = j0 + i;
  DevLists ql;
  int rc = upload_lists(env, q_ptr, q_items, idx, tmp, &ql);
  if (rc) return rc;
  CoocLists L;
  L.q = ql.keys;
  L.q_ptr = ql.ptr;
  QueryFilterDev qf;
  if (f) {
    rc = upload_part_filter(env, f, cf, idx, tmp, &qf);
    if (rc) return rc;
    if (f->has_wl && std::any_of(f->has_wl + j0, f->has_wl + j1, [](uint8_t x) { return x != 0; })) {
      DevLists wl;
      rc = upload_lists(env, f->wl_ptr, f->wl_items, idx, tmp, &wl);
      if (rc) return rc;
      uint8_t* d_has = nullptr;
      CKF(env, tmp.alloc(&d_has, (size_t)n));
      CKF(env, cudaMemcpyAsync(d_has, f->has_wl + j0, (size_t)n, cudaMemcpyHostToDevice, st));
      L.has_wl = d_has;
      L.wl = wl.keys;
      L.wl_ptr = wl.ptr;
    }
  }
  // sizes and offsets of the expansion
  const long long T = q_ptr[j1] - q_ptr[j0];
  uint32_t *size = nullptr, *off = nullptr;
  long long E = 0;
  if (T > 0) {
    CKF(env, tmp.alloc(&size, (size_t)T));
    CKF(env, tmp.alloc(&off, (size_t)T));
    rc = env_launch(env, cp_size_kernel, T, ql.keys, T, m->n_items, (const int*)m->d_n, size);
    if (rc) return rc;
    CKF(env, scan_exclusive_u32(size, off, (size_t)T, st, env.launches));
    uint32_t last[2] = {0, 0};
    CKF(env, cudaMemcpyAsync(&last[0], off + T - 1, 4, cudaMemcpyDeviceToHost, st));
    CKF(env, cudaMemcpyAsync(&last[1], size + T - 1, 4, cudaMemcpyDeviceToHost, st));
    CKF(env, cudaStreamSynchronize(st));
    E = (long long)last[0] + last[1];
  }
  m->stats.last_expanded += E;
  // expand, sort by (query, candidate), sum each run that passes the filters, order each query's rows
  const int bits_q = ceil_log2((uint64_t)n), bits_i = ceil_log2((uint64_t)m->n_items);
  SortBufs sb;
  int* row_q = nullptr;
  int* row_item = nullptr;
  long long* row_score = nullptr;
  long long R = 0;
  if (E > 0) {
    for (int b = 0; b < 2; ++b) {
      CKF(env, tmp.alloc(&sb.k[b], (size_t)E));
      CKF(env, tmp.alloc(&sb.v[b], (size_t)E));
    }
    rc = env_launch(env, cp_expand_kernel, T * 32, ql.keys, (const uint32_t*)size, (const uint32_t*)off, T,
                    (const int*)m->d_items, (const int*)m->d_counts, m->topn, bits_i, sb.keys(), sb.vals());
    if (rc) return rc;
    CKF(env, radix_sort_pairs(sb, (size_t)E, bits_q + bits_i, st, env.launches));
    uint32_t *pass = nullptr, *pos = nullptr;
    CKF(env, tmp.alloc(&pass, (size_t)E));
    CKF(env, tmp.alloc(&pos, (size_t)E));
    rc = env_launch(env, cp_pass_kernel, E, (const uint64_t*)sb.keys(), E, bits_i, L, qf, pass);
    if (rc) return rc;
    CKF(env, scan_exclusive_u32(pass, pos, (size_t)E, st, env.launches));
    uint32_t last[2] = {0, 0};
    CKF(env, cudaMemcpyAsync(&last[0], pos + E - 1, 4, cudaMemcpyDeviceToHost, st));
    CKF(env, cudaMemcpyAsync(&last[1], pass + E - 1, 4, cudaMemcpyDeviceToHost, st));
    CKF(env, cudaStreamSynchronize(st));
    R = (long long)last[0] + last[1];
    if (R > 0) {
      CKF(env, tmp.alloc(&row_q, (size_t)R));
      CKF(env, tmp.alloc(&row_item, (size_t)R));
      CKF(env, tmp.alloc(&row_score, (size_t)R));
      rc = env_launch(env, cp_rows_kernel, E, (const uint64_t*)sb.keys(), (const uint32_t*)sb.vals(), E, bits_i,
                      (const uint32_t*)pass, (const uint32_t*)pos, (uint64_t)bound, row_q, row_item, row_score,
                      sb.spare_keys(), sb.spare_vals());
      if (rc) return rc;
      sb.flip();
      // stable LSD: by score descending, then by query; rows enter in (query, item) order, so equal scores stay
      // item-ascending
      const int sbits = bound ? 64 - __builtin_clzll(bound) : 0;
      CKF(env, radix_sort_pairs(sb, (size_t)R, sbits, st, env.launches));
      rc = env_launch(env, cp_query_keys_kernel, R, (const uint32_t*)sb.vals(), R, (const int*)row_q, sb.spare_keys(),
                      sb.spare_vals());
      if (rc) return rc;
      sb.flip();
      CKF(env, radix_sort_pairs(sb, (size_t)R, bits_q, st, env.launches));
    }
  }
  m->stats.last_rows += R;
  int* d_oi = nullptr;
  long long* d_os = nullptr;
  int* d_oc = nullptr;
  CKF(env, tmp.alloc(&d_oi, (size_t)n * topk));
  CKF(env, tmp.alloc(&d_os, (size_t)n * topk));
  CKF(env, tmp.alloc(&d_oc, (size_t)n));
  cp_take_kernel<<<n, 128, 0, st>>>((const uint64_t*)sb.keys(), (const uint32_t*)sb.vals(), R, topk, row_item, row_score,
                                    d_oi, d_os, d_oc);
  ++*env.launches;
  CKF(env, cudaGetLastError());
  CKF(env, cudaMemcpyAsync(out_items + (size_t)j0 * topk, d_oi, sizeof(int) * (size_t)n * topk, cudaMemcpyDeviceToHost, st));
  CKF(env, cudaMemcpyAsync(out_scores + (size_t)j0 * topk, d_os, sizeof(long long) * (size_t)n * topk,
                           cudaMemcpyDeviceToHost, st));
  if (out_count) CKF(env, cudaMemcpyAsync(out_count + j0, d_oc, sizeof(int) * (size_t)n, cudaMemcpyDeviceToHost, st));
  CKF(env, cudaStreamSynchronize(st));
  return PIO_ALS_OK;
}

}  // namespace pio

extern "C" {

int pio_cooc_model_create(int device, int32_t n_items, int32_t topn, const int32_t* top_items, const int32_t* top_counts,
                          const int32_t* top_n, pio_cooc_model** out) {
  if (!out || !top_items || !top_counts || !top_n || n_items < 1 || topn < 1)
    return fail(nullptr, PIO_ALS_ERR_ARG, "bad pio_cooc_model_create arguments");
  *out = nullptr;
  for (int32_t i = 0; i < n_items; ++i) {
    if (top_n[i] < 0 || top_n[i] > topn)
      return fail(nullptr, PIO_ALS_ERR_ARG, "item %d: top_n %d is outside [0, %d]", i, top_n[i], topn);
    for (int32_t t = 0; t < top_n[i]; ++t) {
      const size_t c = (size_t)i * topn + t;
      if (top_items[c] < 0 || top_items[c] >= n_items)
        return fail(nullptr, PIO_ALS_ERR_ARG, "item %d, slot %d: item %d is outside [0, %d)", i, t, top_items[c], n_items);
      if (top_counts[c] < 0)
        return fail(nullptr, PIO_ALS_ERR_ARG, "item %d, slot %d: count %d is negative", i, t, top_counts[c]);
    }
  }
  std::unique_ptr<pio_cooc_model> m;
  try {   // bad_alloc must not cross the C boundary
    m.reset(new pio_cooc_model);
    const size_t cells = (size_t)n_items * topn;
    m->device = device, m->n_items = n_items, m->topn = topn;
    m->items.assign(top_items, top_items + cells);
    m->counts.assign(top_counts, top_counts + cells);
    m->top_n.assign(top_n, top_n + n_items);
    m->row_sum.assign((size_t)n_items, 0);
  } catch (const std::bad_alloc&) {
    return fail(nullptr, PIO_ALS_ERR_NOMEM, "pio_cooc_model_create: out of host memory");
  }
  for (int32_t i = 0; i < n_items; ++i)
    for (int32_t t = 0; t < top_n[i]; ++t) m->row_sum[i] += top_counts[(size_t)i * topn + t];
  *out = m.release();
  return PIO_ALS_OK;
}

int pio_cooc_model_destroy(pio_cooc_model* m) {
  if (!m) return PIO_ALS_OK;
  if (m->st) {
    cudaSetDevice(m->device);
    cudaStreamSynchronize(m->st);
    cudaStreamDestroy(m->st);
  }
  for (int* p : {m->d_items, m->d_counts, m->d_n})
    if (p) cudaFree(p);
  delete m;
  return PIO_ALS_OK;
}

}  // extern "C"

namespace pio {
static int cooc_predict(pio_cooc_model* m, const int64_t* q_ptr, const int32_t* q_items, int32_t n_queries, int32_t topk,
                        const pio_als_query_filter* f, int32_t* out_items, int64_t* out_scores, int32_t* out_count) {
  pio_cooc_stats& s = m->stats;
  s.last_expanded = s.last_rows = s.last_budget = 0;
  s.last_parts = s.last_max_part_queries = 0;
  if (n_queries < 0 || topk < 1) return fail(nullptr, PIO_ALS_ERR_ARG, "topk must be >= 1 and n_queries >= 0");
  if (n_queries == 0) return PIO_ALS_OK;
  if (!q_ptr || !out_items || !out_scores) return fail(nullptr, PIO_ALS_ERR_ARG, "null argument");
  if (q_ptr[0] < 0) return fail(nullptr, PIO_ALS_ERR_ARG, "q_ptr must be non-decreasing offsets into q_items");
  for (int j = 0; j < n_queries; ++j)
    if (q_ptr[j + 1] < q_ptr[j] || (q_ptr[j + 1] > q_ptr[j] && !q_items))
      return fail(nullptr, PIO_ALS_ERR_ARG, "q_ptr must be non-decreasing offsets into q_items");
  if (f)
    if (const char* what = query_filter_error(f, n_queries)) return fail(nullptr, PIO_ALS_ERR_ARG, "%s", what);
  // PIO_COOC_PREDICT_BUDGET: expanded entries per part; capped so that a part's offsets fit the 32-bit scan
  const char* env_b = getenv("PIO_COOC_PREDICT_BUDGET");
  const long long budget = std::min<long long>(env_b && atoll(env_b) > 0 ? atoll(env_b) : PIO_COOC_PREDICT_BUDGET,
                                               (1ll << 32) - 1);
  CoocPlan plan;
  int rc = cooc_plan(m, q_ptr, q_items, n_queries, budget, &plan);
  if (rc) return rc;
  CK0(cudaSetDevice(m->device));
  const FilterEnv env{nullptr, m->n_items, &s.kernel_launches, &g_create_error};
  rc = cooc_upload(m, env);
  if (rc) return rc;
  FilterEnv penv = env;
  penv.st = m->st;
  s.last_budget = budget;
  Scratch tmp(m->st);
  CallFilter cf;
  if (f) {
    rc = upload_set_rows(penv, f, tmp, &cf);
    if (rc) return rc;
  }
  const int parts = (int)plan.first.size() - 1;
  for (int p = 0; p < parts; ++p) {
    const int j0 = plan.first[p], j1 = plan.first[p + 1];
    s.last_parts = p + 1;
    s.last_max_part_queries = std::max(s.last_max_part_queries, j1 - j0);
    rc = cooc_part(m, penv, q_ptr, q_items, j0, j1, topk, plan.bound[p], f, cf, out_items, out_scores, out_count);
    if (rc) return rc;
  }
  return PIO_ALS_OK;
}
}  // namespace pio

extern "C" {

int pio_cooc_predict_filtered(pio_cooc_model* m, const int64_t* q_ptr, const int32_t* q_items, int32_t n_queries,
                              int32_t topk, const pio_als_query_filter* f, int32_t* out_items, int64_t* out_scores,
                              int32_t* out_count) {
  if (!m) return fail(nullptr, PIO_ALS_ERR_ARG, "null model");
  std::lock_guard<std::mutex> lk(m->mu);
  try {   // bad_alloc must not cross the C boundary; Scratch releases a part's device memory on the way out
    return cooc_predict(m, q_ptr, q_items, n_queries, topk, f, out_items, out_scores, out_count);
  } catch (const std::bad_alloc&) {
    return fail(nullptr, PIO_ALS_ERR_NOMEM, "pio_cooc_predict_filtered: out of host memory");
  }
}

int pio_cooc_model_get_stats(const pio_cooc_model* m, pio_cooc_stats* out) {
  if (!m || !out) return fail(nullptr, PIO_ALS_ERR_ARG, "null argument");
  std::lock_guard<std::mutex> lk(m->mu);
  *out = m->stats;
  return PIO_ALS_OK;
}

}  // extern "C"

// ---- popularity top-N (ecommerce ECommAlgorithm.predictDefault) ------------------------------------------------------------
struct pio_popular_model {
  int device = 0, n_items = 0;
  std::vector<double> scores;           // host copy until the first call ranks it on the device
  cudaStream_t st = nullptr;
  int *d_order = nullptr, *d_rank = nullptr;   // set together with d_sorted, once the ranked order has landed
  double* d_sorted = nullptr;
  mutable std::mutex mu;                // serialises the calls, and guards stats
  pio_popular_stats stats{};
};

namespace pio {

// A call's parts: consecutive queries [first[p], first[p + 1]).  A part closes before the query that would take its
// entries (exclusion and white-list entries, plus topk output slots per query) over the budget; each part holds at
// least one query.
static int popular_plan(const pio_als_query_filter* f, int n, int topk, long long budget, std::vector<int>* first) {
  long long acc = 0;
  for (int j = 0; j < n; ++j) {
    long long ent = topk;
    if (f && f->ex_ptr) ent += f->ex_ptr[j + 1] - f->ex_ptr[j];
    if (f && f->wl_ptr) ent += f->wl_ptr[j + 1] - f->wl_ptr[j];
    if (ent >= (1ll << 32))
      return fail(nullptr, PIO_ALS_ERR_ARG, "query %d has %lld list entries and output slots: at most 2^32 - 1 fit one part",
                  j, ent);
    if (j == 0 || acc + ent > budget) {
      first->push_back(j);
      acc = 0;
    }
    acc += ent;
  }
  first->push_back(n);
  return PIO_ALS_OK;
}

// the ranked order of m's scores into order / sorted / rank, on env's stream, complete when it returns OK
static int popular_rank(pio_popular_model* m, const FilterEnv& env, int* order, double* sorted, int* rank) {
  const int n = m->n_items;
  Scratch tmp(env.st);
  double* d_scores = nullptr;
  SortBufs sb;
  CKF(env, tmp.alloc(&d_scores, (size_t)n));
  for (int b = 0; b < 2; ++b) {
    CKF(env, tmp.alloc(&sb.k[b], (size_t)n));
    CKF(env, tmp.alloc(&sb.v[b], (size_t)n));
  }
  CKF(env, cudaMemcpyAsync(d_scores, m->scores.data(), sizeof(double) * (size_t)n, cudaMemcpyHostToDevice, env.st));
  int rc = env_launch(env, pp_rank_keys_kernel, n, (const double*)d_scores, n, sb.keys(), sb.vals());
  if (rc) return rc;
  CKF(env, radix_sort_pairs(sb, (size_t)n, 64, env.st, env.launches));
  rc = env_launch(env, pp_ranked_kernel, n, (const uint32_t*)sb.vals(), (const double*)d_scores, n, order, sorted, rank);
  if (rc) return rc;
  CKF(env, cudaStreamSynchronize(env.st));   // the host scores are read until here
  return PIO_ALS_OK;
}

// The model's ranked order, made on its own stream by the first call.  The device pointers are published only after it
// has completed, so a failed upload leaves nothing half made: its allocations are freed and the next call starts over.
static int popular_upload(pio_popular_model* m, FilterEnv env) {
  if (m->d_order) return PIO_ALS_OK;
  if (!m->st) CKF(env, cudaStreamCreateWithFlags(&m->st, cudaStreamNonBlocking));
  env.st = m->st;
  const size_t n = (size_t)m->n_items;
  int *order = nullptr, *rank = nullptr;
  double* sorted = nullptr;
  cudaError_t e = cudaMalloc((void**)&order, sizeof(int) * n);
  if (e == cudaSuccess) e = cudaMalloc((void**)&rank, sizeof(int) * n);
  if (e == cudaSuccess) e = cudaMalloc((void**)&sorted, sizeof(double) * n);
  const int rc = e == cudaSuccess ? popular_rank(m, env, order, sorted, rank) : PIO_ALS_OK;
  if (e != cudaSuccess || rc) {
    cudaStreamSynchronize(m->st);
    for (void* p : {(void*)order, (void*)rank, (void*)sorted})
      if (p) cudaFree(p);
    return rc ? rc : fail_to(env.err, PIO_ALS_ERR_CUDA, "uploading the popularity model: %s", cudaGetErrorString(e));
  }
  m->d_order = order, m->d_rank = rank, m->d_sorted = sorted;
  std::vector<double>().swap(m->scores);
  return PIO_ALS_OK;
}

// the queries [j0, j1) of a call: rows j0 .. j1 - 1 of the caller's outputs
static int popular_part(pio_popular_model* m, const FilterEnv& env, int j0, int j1, int topk,
                        const pio_als_query_filter* f, const CallFilter& cf, int32_t* out_items, double* out_scores,
                        int32_t* out_count) {
  const int n = j1 - j0;
  cudaStream_t st = env.st;
  Scratch tmp(st);
  std::vector<int> idx((size_t)n);
  for (int i = 0; i < n; ++i) idx[i] = j0 + i;
  QueryFilterDev qf;
  PopularLists L;
  long long listed = 0;
  if (f) {
    int rc = upload_part_filter(env, f, cf, idx, tmp, &qf);
    if (rc) return rc;
    if (f->has_wl && std::any_of(f->has_wl + j0, f->has_wl + j1, [](uint8_t x) { return x != 0; })) {
      // the white lists as (query << 32 | rank position) keys, sorted: each query's list in rank order
      DevLists wl;
      rc = upload_lists(env, f->wl_ptr, f->wl_items, idx, tmp, &wl);
      if (rc) return rc;
      listed = f->wl_ptr ? f->wl_ptr[j1] - f->wl_ptr[j0] : 0;
      SortBufs sb;
      if (listed > 0) {
        for (int b = 0; b < 2; ++b) {
          CKF(env, tmp.alloc(&sb.k[b], (size_t)listed));
          CKF(env, tmp.alloc(&sb.v[b], (size_t)listed));
        }
        rc = env_launch(env, pp_list_keys_kernel, listed, wl.keys, listed, (const int*)m->d_rank, m->n_items, sb.keys(),
                        sb.vals());
        if (rc) return rc;
        CKF(env, radix_sort_pairs(sb, (size_t)listed, 32 + ceil_log2((uint64_t)n), st, env.launches));
      }
      uint8_t* d_has = nullptr;
      CKF(env, tmp.alloc(&d_has, (size_t)n));
      CKF(env, cudaMemcpyAsync(d_has, f->has_wl + j0, (size_t)n, cudaMemcpyHostToDevice, st));
      L.has_wl = d_has;
      L.keys = sb.keys();
      L.ptr = wl.ptr;
    }
  }
  m->stats.last_listed += listed;
  int* d_oi = nullptr;
  double* d_os = nullptr;
  int* d_oc = nullptr;
  unsigned long long* d_walked = nullptr;
  CKF(env, tmp.alloc(&d_oi, (size_t)n * topk));
  CKF(env, tmp.alloc(&d_os, (size_t)n * topk));
  CKF(env, tmp.alloc(&d_oc, (size_t)n));
  CKF(env, tmp.alloc(&d_walked, 1));
  CKF(env, cudaMemsetAsync(d_walked, 0, sizeof(unsigned long long), st));
  PopularRanked R;
  R.order = m->d_order;
  R.sorted = m->d_sorted;
  R.n_items = m->n_items;
  const int rc = env_launch(env, pp_take_kernel, (long long)n * 32, R, n, topk, qf, L, d_oi, d_os, d_oc, d_walked);
  if (rc) return rc;
  unsigned long long walked = 0;
  CKF(env, cudaMemcpyAsync(out_items + (size_t)j0 * topk, d_oi, sizeof(int) * (size_t)n * topk, cudaMemcpyDeviceToHost, st));
  CKF(env, cudaMemcpyAsync(out_scores + (size_t)j0 * topk, d_os, sizeof(double) * (size_t)n * topk, cudaMemcpyDeviceToHost,
                           st));
  CKF(env, cudaMemcpyAsync(out_count + j0, d_oc, sizeof(int) * (size_t)n, cudaMemcpyDeviceToHost, st));
  CKF(env, cudaMemcpyAsync(&walked, d_walked, sizeof walked, cudaMemcpyDeviceToHost, st));
  CKF(env, cudaStreamSynchronize(st));
  m->stats.last_walked += (int64_t)walked;
  return PIO_ALS_OK;
}

static int popular_predict(pio_popular_model* m, int32_t n_queries, int32_t topk, const pio_als_query_filter* f,
                           int32_t* out_items, double* out_scores, int32_t* out_count) {
  pio_popular_stats& s = m->stats;
  s.last_walked = s.last_listed = 0;
  s.last_parts = s.last_max_part_queries = 0;
  if (n_queries < 0 || topk < 1) return fail(nullptr, PIO_ALS_ERR_ARG, "topk must be >= 1 and n_queries >= 0");
  if (n_queries == 0) return PIO_ALS_OK;
  if (!out_items || !out_scores || !out_count) return fail(nullptr, PIO_ALS_ERR_ARG, "null argument");
  if (f)
    if (const char* what = query_filter_error(f, n_queries)) return fail(nullptr, PIO_ALS_ERR_ARG, "%s", what);
  // PIO_POPULAR_PREDICT_BUDGET: entries per part; capped so that a part's entries are numbered in 32 bits
  const char* env_b = getenv("PIO_POPULAR_PREDICT_BUDGET");
  const long long budget = std::min<long long>(env_b && atoll(env_b) > 0 ? atoll(env_b) : PIO_POPULAR_PREDICT_BUDGET,
                                               (1ll << 32) - 1);
  std::vector<int> first;
  int rc = popular_plan(f, n_queries, topk, budget, &first);
  if (rc) return rc;
  CK0(cudaSetDevice(m->device));
  FilterEnv env{nullptr, m->n_items, &s.kernel_launches, &g_create_error};
  rc = popular_upload(m, env);
  if (rc) return rc;
  env.st = m->st;
  Scratch tmp(m->st);
  CallFilter cf;
  if (f) {
    rc = upload_set_rows(env, f, tmp, &cf);
    if (rc) return rc;
  }
  const int parts = (int)first.size() - 1;
  for (int p = 0; p < parts; ++p) {
    const int j0 = first[p], j1 = first[p + 1];
    s.last_parts = p + 1;
    s.last_max_part_queries = std::max(s.last_max_part_queries, j1 - j0);
    rc = popular_part(m, env, j0, j1, topk, f, cf, out_items, out_scores, out_count);
    if (rc) return rc;
  }
  return PIO_ALS_OK;
}

}  // namespace pio

extern "C" {

int pio_popular_model_create(int device, int32_t n_items, const double* scores, pio_popular_model** out) {
  if (!out || !scores || n_items < 1) return fail(nullptr, PIO_ALS_ERR_ARG, "bad pio_popular_model_create arguments");
  *out = nullptr;
  for (int32_t i = 0; i < n_items; ++i)
    if (std::isnan(scores[i])) return fail(nullptr, PIO_ALS_ERR_ARG, "item %d: score is NaN", i);
  std::unique_ptr<pio_popular_model> m;
  try {   // bad_alloc must not cross the C boundary
    m.reset(new pio_popular_model);
    m->device = device, m->n_items = n_items;
    m->scores.assign(scores, scores + n_items);
  } catch (const std::bad_alloc&) {
    return fail(nullptr, PIO_ALS_ERR_NOMEM, "pio_popular_model_create: out of host memory");
  }
  *out = m.release();
  return PIO_ALS_OK;
}

int pio_popular_model_destroy(pio_popular_model* m) {
  if (!m) return PIO_ALS_OK;
  if (m->st) {
    cudaSetDevice(m->device);
    cudaStreamSynchronize(m->st);
    cudaStreamDestroy(m->st);
  }
  for (void* p : {(void*)m->d_order, (void*)m->d_rank, (void*)m->d_sorted})
    if (p) cudaFree(p);
  delete m;
  return PIO_ALS_OK;
}

int pio_popular_predict_filtered(pio_popular_model* m, int32_t n_queries, int32_t topk, const pio_als_query_filter* f,
                                 int32_t* out_items, double* out_scores, int32_t* out_count) {
  if (!m) return fail(nullptr, PIO_ALS_ERR_ARG, "null model");
  std::lock_guard<std::mutex> lk(m->mu);
  try {   // bad_alloc must not cross the C boundary; Scratch releases a part's device memory on the way out
    return popular_predict(m, n_queries, topk, f, out_items, out_scores, out_count);
  } catch (const std::bad_alloc&) {
    return fail(nullptr, PIO_ALS_ERR_NOMEM, "pio_popular_predict_filtered: out of host memory");
  }
}

int pio_popular_model_get_stats(const pio_popular_model* m, pio_popular_stats* out) {
  if (!m || !out) return fail(nullptr, PIO_ALS_ERR_ARG, "null argument");
  std::lock_guard<std::mutex> lk(m->mu);
  *out = m->stats;
  return PIO_ALS_OK;
}

}  // extern "C"

// ---- z-score serving merge (similarproduct Serving.serve) ------------------------------------------------------------------
namespace pio {

// what the last pio_serve_zscore_merge on this thread did (pio_serve_merge_debug_stats)
struct ServeMergeStats {
  long long parts = 0, max_part_queries = 0, entries = 0, rows = 0, budget = 0;
  double device_ms = 0.0;
};
static thread_local ServeMergeStats g_sm_stats;

// The queries [j0, j1) of a call on stream st: rows j0 .. j1 - 1 of the caller's outputs.
static int sm_part(cudaStream_t st, int n_algos, int n_items, const int32_t* const* items, const double* const* scores,
                   const int32_t* const* counts, const int32_t* widths, const int32_t* num, int j0, int j1, int topk,
                   int32_t* out_items, double* out_scores, int32_t* out_count) {
  const int n = j1 - j0;
  const long long NL = (long long)n * n_algos;
  std::vector<uint32_t> h_cnt((size_t)NL), h_off((size_t)NL);
  long long E = 0;
  for (int q = 0; q < n; ++q)
    for (int a = 0; a < n_algos; ++a) {
      const size_t l = (size_t)q * n_algos + a;
      h_cnt[l] = (uint32_t)counts[a][j0 + q];
      h_off[l] = (uint32_t)E;
      E += h_cnt[l];
    }
  Scratch tmp(st);
  std::vector<const int*> h_items((size_t)n_algos, nullptr);
  std::vector<const double*> h_scores((size_t)n_algos, nullptr);
  for (int a = 0; a < n_algos; ++a) {
    const size_t cells = (size_t)n * widths[a];
    if (cells == 0) continue;
    int* di = nullptr;
    double* ds = nullptr;
    CK0(tmp.alloc(&di, cells));
    CK0(tmp.alloc(&ds, cells));
    CK0(cudaMemcpyAsync(di, items[a] + (size_t)j0 * widths[a], sizeof(int) * cells, cudaMemcpyHostToDevice, st));
    CK0(cudaMemcpyAsync(ds, scores[a] + (size_t)j0 * widths[a], sizeof(double) * cells, cudaMemcpyHostToDevice, st));
    h_items[a] = di, h_scores[a] = ds;
  }
  const int** d_items = nullptr;
  const double** d_scores = nullptr;
  int *d_w = nullptr, *d_num = nullptr;
  uint32_t *d_cnt = nullptr, *d_off = nullptr;
  double *d_mean = nullptr, *d_sd = nullptr;
  CK0(tmp.alloc(&d_items, (size_t)n_algos));
  CK0(tmp.alloc(&d_scores, (size_t)n_algos));
  CK0(tmp.alloc(&d_w, (size_t)n_algos));
  CK0(tmp.alloc(&d_num, (size_t)n));
  CK0(tmp.alloc(&d_cnt, (size_t)NL));
  CK0(tmp.alloc(&d_off, (size_t)NL));
  CK0(tmp.alloc(&d_mean, (size_t)NL));
  CK0(tmp.alloc(&d_sd, (size_t)NL));
  CK0(cudaMemcpyAsync(d_items, h_items.data(), sizeof(int*) * n_algos, cudaMemcpyHostToDevice, st));
  CK0(cudaMemcpyAsync(d_scores, h_scores.data(), sizeof(double*) * n_algos, cudaMemcpyHostToDevice, st));
  CK0(cudaMemcpyAsync(d_w, widths, sizeof(int) * n_algos, cudaMemcpyHostToDevice, st));
  CK0(cudaMemcpyAsync(d_num, num + j0, sizeof(int) * n, cudaMemcpyHostToDevice, st));
  CK0(cudaMemcpyAsync(d_cnt, h_cnt.data(), sizeof(uint32_t) * NL, cudaMemcpyHostToDevice, st));
  CK0(cudaMemcpyAsync(d_off, h_off.data(), sizeof(uint32_t) * NL, cudaMemcpyHostToDevice, st));
  const MergeLists L{d_items, d_scores, d_w, n_algos};
  sm_stats_kernel<<<nblk(NL, 128), 128, 0, st>>>(L, d_cnt, NL, d_num, d_mean, d_sd);
  CK0(cudaGetLastError());
  const int bits_q = ceil_log2((uint64_t)n), bits_i = ceil_log2((uint64_t)n_items);
  SortBufs sb;
  uint64_t* row_key = nullptr;
  double* row_sum = nullptr;
  long long R = 0;
  if (E > 0) {
    for (int b = 0; b < 2; ++b) {
      CK0(tmp.alloc(&sb.k[b], (size_t)E));
      CK0(tmp.alloc(&sb.v[b], (size_t)E));
    }
    double *z = nullptr, *head_sum = nullptr;
    uint64_t* head_key = nullptr;
    uint32_t *head = nullptr, *pos = nullptr;
    CK0(tmp.alloc(&z, (size_t)E));
    CK0(tmp.alloc(&head_sum, (size_t)E));
    CK0(tmp.alloc(&head_key, (size_t)E));
    CK0(tmp.alloc(&head, (size_t)E));
    CK0(tmp.alloc(&pos, (size_t)E));
    CK0(cudaMemsetAsync(head, 0, sizeof(uint32_t) * E, st));
    sm_entries_kernel<<<(unsigned)std::min<long long>(nblk(NL * 32, 256), 132 * 64), 256, 0, st>>>(
        L, d_cnt, d_off, NL, d_mean, d_sd, bits_i, sb.keys(), sb.vals(), z);
    CK0(cudaGetLastError());
    CK0(radix_sort_pairs(sb, (size_t)E, bits_q + bits_i, st, nullptr));
    sm_sum_kernel<<<nblk(E, 256), 256, 0, st>>>(sb.keys(), sb.vals(), E, z, head, head_key, head_sum);
    CK0(cudaGetLastError());
    CK0(scan_exclusive_u32(head, pos, (size_t)E, st, nullptr));
    uint32_t last[2] = {0, 0};
    CK0(cudaMemcpyAsync(&last[0], pos + E - 1, 4, cudaMemcpyDeviceToHost, st));
    CK0(cudaMemcpyAsync(&last[1], head + E - 1, 4, cudaMemcpyDeviceToHost, st));
    CK0(cudaStreamSynchronize(st));
    R = (long long)last[0] + last[1];
    CK0(tmp.alloc(&row_key, (size_t)R));
    CK0(tmp.alloc(&row_sum, (size_t)R));
    sm_rows_kernel<<<nblk(E, 256), 256, 0, st>>>(head, pos, E, head_key, head_sum, row_key, row_sum, sb.spare_keys(),
                                                 sb.spare_vals());
    CK0(cudaGetLastError());
    sb.flip();
    // stable LSD: by sum descending, then by query; rows enter in (query, first appearance) order, so equal sums keep it
    CK0(radix_sort_pairs(sb, (size_t)R, 64, st, nullptr));
    sm_query_keys_kernel<<<nblk(R, 256), 256, 0, st>>>(sb.vals(), R, row_key, bits_i, sb.spare_keys(), sb.spare_vals());
    CK0(cudaGetLastError());
    sb.flip();
    CK0(radix_sort_pairs(sb, (size_t)R, bits_q, st, nullptr));
  }
  int* d_oi = nullptr;
  double* d_os = nullptr;
  int* d_oc = nullptr;
  CK0(tmp.alloc(&d_oi, (size_t)n * topk));
  CK0(tmp.alloc(&d_os, (size_t)n * topk));
  CK0(tmp.alloc(&d_oc, (size_t)n));
  sm_take_kernel<<<n, 128, 0, st>>>(sb.keys(), sb.vals(), R, topk, d_num, row_key, bits_i, row_sum, d_oi, d_os, d_oc);
  CK0(cudaGetLastError());
  CK0(cudaMemcpyAsync(out_items + (size_t)j0 * topk, d_oi, sizeof(int) * (size_t)n * topk, cudaMemcpyDeviceToHost, st));
  CK0(cudaMemcpyAsync(out_scores + (size_t)j0 * topk, d_os, sizeof(double) * (size_t)n * topk, cudaMemcpyDeviceToHost,
                      st));
  CK0(cudaMemcpyAsync(out_count + j0, d_oc, sizeof(int) * (size_t)n, cudaMemcpyDeviceToHost, st));
  CK0(cudaStreamSynchronize(st));
  g_sm_stats.entries += E;
  g_sm_stats.rows += R;
  return PIO_ALS_OK;
}

static int serve_zscore_merge(int device, int32_t n_queries, int32_t n_algos, int32_t n_items,
                              const int32_t* const* items, const double* const* scores, const int32_t* const* counts,
                              const int32_t* widths, const int32_t* num, int32_t topk, int32_t* out_items,
                              double* out_scores, int32_t* out_count) {
  g_sm_stats = ServeMergeStats{};
  if (n_queries < 0 || n_algos < 1 || n_items < 1 || topk < 1)
    return fail(nullptr, PIO_ALS_ERR_ARG, "n_queries must be >= 0, n_algos, n_items and topk >= 1");
  if (n_queries == 0) return PIO_ALS_OK;
  if (!items || !scores || !counts || !widths || !num || !out_items || !out_scores || !out_count)
    return fail(nullptr, PIO_ALS_ERR_ARG, "null argument");
  for (int a = 0; a < n_algos; ++a) {
    if (widths[a] < 0) return fail(nullptr, PIO_ALS_ERR_ARG, "algorithm %d: width %d is negative", a, widths[a]);
    if (!counts[a] || (widths[a] > 0 && (!items[a] || !scores[a])))
      return fail(nullptr, PIO_ALS_ERR_ARG, "algorithm %d: null items, scores or counts", a);
  }
  // every query's lists: counts within the widths, ids in the numbering, finite scores; entries per query under 2^32
  std::vector<unsigned long long> ent((size_t)n_queries, 0);
  for (int j = 0; j < n_queries; ++j) {
    if (num[j] < 1) return fail(nullptr, PIO_ALS_ERR_ARG, "query %d: num %d is below 1", j, num[j]);
    for (int a = 0; a < n_algos; ++a) {
      const int32_t c = counts[a][j];
      if (c < 0 || c > widths[a])
        return fail(nullptr, PIO_ALS_ERR_ARG, "query %d, algorithm %d: count %d is outside [0, %d]", j, a, c, widths[a]);
      const size_t row = (size_t)j * widths[a];
      for (int32_t t = 0; t < c; ++t) {
        if (items[a][row + t] < 0 || items[a][row + t] >= n_items)
          return fail(nullptr, PIO_ALS_ERR_ARG, "query %d, algorithm %d, entry %d: item %d is outside [0, %d)", j, a, t,
                      items[a][row + t], n_items);
        if (!isfinite(scores[a][row + t]))
          return fail(nullptr, PIO_ALS_ERR_ARG, "query %d, algorithm %d, entry %d: the score is not finite", j, a, t);
      }
      ent[j] += (unsigned)c;
    }
    if (ent[j] >= (1ull << 32))
      return fail(nullptr, PIO_ALS_ERR_ARG, "query %d has %llu entries: at most 2^32 - 1 fit one part", j, ent[j]);
  }
  // PIO_SERVE_MERGE_BUDGET: entries per part; capped so that a part's offsets fit the 32-bit scan
  const char* env_b = getenv("PIO_SERVE_MERGE_BUDGET");
  const long long budget = std::min<long long>(env_b && atoll(env_b) > 0 ? atoll(env_b) : PIO_SERVE_MERGE_BUDGET,
                                               (1ll << 32) - 1);
  std::vector<int> first;
  long long acc = 0;
  for (int j = 0; j < n_queries; ++j) {
    if (j == 0 || acc + (long long)ent[j] > budget) {
      first.push_back(j);
      acc = 0;
    }
    acc += (long long)ent[j];
  }
  first.push_back(n_queries);
  g_sm_stats.budget = budget;
  CK0(cudaSetDevice(device));
  CallMem mem;
  cudaStream_t st = nullptr;
  cudaEvent_t t0 = nullptr, t1 = nullptr;
  CK0(mem.stream(&st));
  CK0(mem.event(&t0));
  CK0(mem.event(&t1));
  CK0(cudaEventRecord(t0, st));
  for (size_t p = 0; p + 1 < first.size(); ++p) {
    g_sm_stats.parts = (long long)p + 1;
    g_sm_stats.max_part_queries = std::max<long long>(g_sm_stats.max_part_queries, first[p + 1] - first[p]);
    const int rc = sm_part(st, n_algos, n_items, items, scores, counts, widths, num, first[p], first[p + 1], topk,
                           out_items, out_scores, out_count);
    if (rc) return rc;
  }
  CK0(cudaEventRecord(t1, st));
  CK0(cudaEventSynchronize(t1));
  float ms = 0.f;
  CK0(cudaEventElapsedTime(&ms, t0, t1));
  g_sm_stats.device_ms = ms;
  return PIO_ALS_OK;
}

}  // namespace pio

extern "C" {

int pio_serve_zscore_merge(int device, int32_t n_queries, int32_t n_algos, int32_t n_items, const int32_t* const* items,
                           const double* const* scores, const int32_t* const* counts, const int32_t* widths,
                           const int32_t* num, int32_t topk, int32_t* out_items, double* out_scores, int32_t* out_count) {
  try {   // bad_alloc must not cross the C boundary; Scratch and CallMem release device memory on the way out
    return serve_zscore_merge(device, n_queries, n_algos, n_items, items, scores, counts, widths, num, topk, out_items,
                              out_scores, out_count);
  } catch (const std::bad_alloc&) {
    return fail(nullptr, PIO_ALS_ERR_NOMEM, "pio_serve_zscore_merge: out of host memory");
  }
}

/* debug only (not in pio_als.h): out[0] parts, out[1] most queries in one part, out[2] entries, out[3] distinct (query,
 * item) rows, out[4] the entries budget, out[5] device milliseconds from the first upload to the last copy back -- of the
 * last pio_serve_zscore_merge on this thread.  Used by the tests and tools/serve_merge_bench.py. */
__attribute__((visibility("default"))) int pio_serve_merge_debug_stats(double out[6]) {
  if (!out) return PIO_ALS_ERR_ARG;
  const ServeMergeStats& s = g_sm_stats;
  out[0] = (double)s.parts, out[1] = (double)s.max_part_queries, out[2] = (double)s.entries, out[3] = (double)s.rows;
  out[4] = (double)s.budget, out[5] = s.device_ms;
  return PIO_ALS_OK;
}

// ---- NaiveBayes ---------------------------------------------------------------------------------
}  // extern "C"

namespace pio {

static int nb_check_width(int n_feat, int n_class) {
  if ((size_t)n_class * (n_feat + 1) * 8 * sizeof(double) > 200 * 1024)
    return fail(nullptr, PIO_ALS_ERR_ARG, "n_class*(n_feat+1) too large");
  return PIO_ALS_OK;
}

// pi / theta of n device rows (class index dl, float32 features dx) on stream st: the per-class sums on the device, the
// log-probabilities on the host.  pio_nb_train and pio_cls_folds_nb_train both end here.
static int nb_fit(CallMem& tmp, cudaStream_t st, const int* dl, const float* dx, int64_t n, int n_feat, int n_class,
                  double lambda, double* pi, double* theta) {
  const int width = n_class * (n_feat + 1);
  double *dp = nullptr, *dout = nullptr;
  const int nb = 296;
  CK0(tmp.device(&dp, (size_t)nb * width));
  CK0(tmp.device(&dout, (size_t)width));
  const size_t smem = sizeof(double) * 8 * width;
  CK0(cudaFuncSetAttribute(nb_partial_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  nb_partial_kernel<<<nb, 256, smem, st>>>(dl, dx, n, n_feat, n_class, dp);
  nb_reduce_kernel<<<nblk(width, 128), 128, 0, st>>>(dp, nb, width, dout);
  CK0(cudaGetLastError());
  std::vector<double> acc(width);
  CK0(cudaMemcpyAsync(acc.data(), dout, sizeof(double) * width, cudaMemcpyDeviceToHost, st));
  CK0(cudaStreamSynchronize(st));
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

}  // namespace pio

extern "C" {

int pio_nb_train(int device, const int32_t* label, const float* x, int64_t n, int n_feat, int n_class, double lambda,
                 double* pi, double* theta) {
  if (!label || !x || !pi || !theta || n <= 0 || n_feat < 1 || n_class < 1)
    return fail(nullptr, PIO_ALS_ERR_ARG, "bad NaiveBayes arguments");
  EVF(nb_check_width(n_feat, n_class));
  CK0(cudaSetDevice(device));
  for (int64_t r = 0; r < n; ++r)
    if (label[r] < 0 || label[r] >= n_class) return fail(nullptr, PIO_ALS_ERR_ARG, "label out of range at row %lld", (long long)r);
  CallMem tmp(0);
  int* dl = nullptr;
  float* dx = nullptr;
  CK0(tmp.device(&dl, (size_t)n));
  CK0(tmp.device(&dx, (size_t)n * n_feat));
  CK0(cudaMemcpy(dl, label, sizeof(int) * n, cudaMemcpyHostToDevice));
  CK0(cudaMemcpy(dx, x, sizeof(float) * n * n_feat, cudaMemcpyHostToDevice));
  return nb_fit(tmp, 0, dl, dx, n, n_feat, n_class, lambda, pi, theta);
}

int pio_nb_predict(int device, const float* x, int64_t n, int n_feat, int n_class, const double* pi, const double* theta,
                   int32_t* out_label) {
  if (!x || !pi || !theta || !out_label || n <= 0) return fail(nullptr, PIO_ALS_ERR_ARG, "bad NaiveBayes arguments");
  CK0(cudaSetDevice(device));
  CallMem tmp(0);
  float* dx = nullptr;
  double *dpi = nullptr, *dth = nullptr;
  int* dout = nullptr;
  CK0(tmp.device(&dx, (size_t)n * n_feat));
  CK0(tmp.device(&dpi, (size_t)n_class));
  CK0(tmp.device(&dth, (size_t)n_class * n_feat));
  CK0(tmp.device(&dout, (size_t)n));
  CK0(cudaMemcpy(dx, x, sizeof(float) * n * n_feat, cudaMemcpyHostToDevice));
  CK0(cudaMemcpy(dpi, pi, sizeof(double) * n_class, cudaMemcpyHostToDevice));
  CK0(cudaMemcpy(dth, theta, sizeof(double) * n_class * n_feat, cudaMemcpyHostToDevice));
  nb_predict_kernel<<<nblk(n, 256), 256>>>(dx, n, n_feat, n_class, dpi, dth, dout);
  CK0(cudaGetLastError());
  CK0(cudaMemcpy(out_label, dout, sizeof(int) * n, cudaMemcpyDeviceToHost));
  return PIO_ALS_OK;
}

// ---- RandomForest (csrc/forest.cuh, csrc/forest_splits.h; rules: tests/forest_ref.py) ------------------------------
struct pio_rf_forest {
  int32_t n_trees = 0, n_class = 0;
  std::vector<int32_t> tree_off, feature, left, right, prediction;
  std::vector<double> threshold, impurity, gain;
  std::vector<int64_t> count;
  bool regression = false;              // pio_rf_train_regressor: the fields below, prediction all 0
  std::vector<double> value;            // per node: its mean label
  std::vector<int64_t> cat_off;         // [n_nodes + 1] left categories of each categorical node ...
  std::vector<int32_t> cat_ids;         // ... ascending
};

}  // extern "C"

namespace pio {

constexpr int64_t RF_NODE_BUDGET = 1ll << 30;   // node ids of one tree group (int32 per tree and row)
constexpr int64_t RF_HIST_BUDGET = 1ll << 29;   // the global histogram of one chunk of a level's node slots
constexpr int RF_SMEM = 96 * 1024;              // shared-memory histogram of one pass (two blocks per SM)

// where the last pio_rf_train on this thread spent its time (wall ms; every phase ends in a stream synchronise), and
// which paths it took
struct RfTiming {
  double h2d = 0, split = 0, bin = 0, hist = 0, sel = 0, upd = 0;
  int levels = 0, groups = 0;
  double hist_l[RF_MAX_DEPTH + 1] = {}, sel_l[RF_MAX_DEPTH + 1] = {};
  int bin_bytes = 0, staged = 0;                 // bin code width; thresholds staged in shared memory
  int64_t smem_launches = 0, global_launches = 0;  // hist_kernel<BinT, true> / <BinT, false> launches
  int64_t max_chunks = 0, max_passes = 0;        // most chunks in one level, most shared-memory passes in one chunk
};
static thread_local RfTiming g_rf_timing;

struct RfRec {
  bool leaf;
  int feature;
  double thr, imp, gain;
  int pred;
  int64_t count;
  double value;                         // regressor: the node's mean label
  std::vector<int32_t> cats;            // regressor: left categories of a categorical split, ascending
};
using RfTree = std::map<int64_t, RfRec>;

// a double as the error messages print it: the shortest %g that reads back, '.0' on an integral value
static std::string rf_fmt(double v) {
  char b[64];
  for (int p = 1; p <= 17; ++p) {
    snprintf(b, sizeof b, "%.*g", p, v);
    if (strtod(b, nullptr) == v) break;
  }
  std::string s(b);
  if (s.find_first_of(".en") == std::string::npos) s += ".0";
  return s;
}

// the row checks' messages, row r being the r-th row of the training set: a non-finite label, else the first non-finite
// feature of the row
static int rf_fail_finite(int64_t r, double label, const double* xr, int F) {
  if (!isfinite(label))
    return fail(nullptr, PIO_ALS_ERR_ARG, "label of row %lld is not finite (%s).", (long long)r, rf_fmt(label).c_str());
  for (int f = 0; f < F; ++f)
    if (!isfinite(xr[f]))
      return fail(nullptr, PIO_ALS_ERR_ARG, "feature %d of row %lld is not finite (%s).", f, (long long)r,
                  rf_fmt(xr[f]).c_str());
  return PIO_ALS_OK;
}
static int rf_fail_label(const pio_rf_params* p, double label) {
  const char* agg = p->impurity == RF_GINI ? "GiniAggregator" : "EntropyAggregator";
  if (label >= p->num_classes)
    return fail(nullptr, PIO_ALS_ERR_ARG, "%s given label %s but requires label < numClasses (= %d).", agg,
                rf_fmt(label).c_str(), p->num_classes);
  if (label < 0)
    return fail(nullptr, PIO_ALS_ERR_ARG, "%s given label %sbut requires label is non-negative.", agg,
                rf_fmt(label).c_str());
  return PIO_ALS_OK;
}

// the parameters and the shape (n rows, F features), before any row is read
static int rf_check_params(const pio_rf_params* p, int64_t n, int F) {
  const int C = p->num_classes;
  if (C < 2)
    return fail(nullptr, PIO_ALS_ERR_ARG, "DecisionTree Strategy for Classification must have numClasses >= 2, but "
                "numClasses = %d.", C);
  if (C > RF_MAX_CLASSES)
    return fail(nullptr, PIO_ALS_ERR_ARG, "numClasses = %d: at most %d classes are supported.", C, RF_MAX_CLASSES);
  if (p->num_trees < 1)
    return fail(nullptr, PIO_ALS_ERR_ARG, "RandomForest requires numTrees > 0, but was given numTrees = %d.",
                p->num_trees);
  if (rf_subset_size(p->feature_subset_strategy, F > 1 ? F : 1, p->num_trees) == 0)
    return fail(nullptr, PIO_ALS_ERR_ARG, "RandomForest given invalid featureSubsetStrategy: %s. Supported values: "
                "auto, all, onethird, sqrt, log2, (0.0-1.0], [1-n].",
                p->feature_subset_strategy ? p->feature_subset_strategy : "null");
  if (p->max_depth < 0)
    return fail(nullptr, PIO_ALS_ERR_ARG, "DecisionTree Strategy given invalid maxDepth parameter: %d.  Valid values "
                "are integers >= 0.", p->max_depth);
  if (p->max_depth > RF_MAX_DEPTH)
    return fail(nullptr, PIO_ALS_ERR_ARG, "DecisionTree currently only supports maxDepth <= 30, but was given maxDepth "
                "= %d.", p->max_depth);
  if (p->max_bins < 2)
    return fail(nullptr, PIO_ALS_ERR_ARG, "DecisionTree Strategy given invalid maxBins parameter: %d.  Valid values are "
                "integers >= 2.", p->max_bins);
  if (p->max_bins > RF_MAX_BINS)
    return fail(nullptr, PIO_ALS_ERR_ARG, "maxBins = %d: at most %d bins are supported.", p->max_bins, RF_MAX_BINS);
  if (p->impurity != RF_GINI && p->impurity != RF_ENTROPY)
    return fail(nullptr, PIO_ALS_ERR_ARG, "unknown impurity code %d", p->impurity);
  if (n < 1 || F < 1) return fail(nullptr, PIO_ALS_ERR_ARG, "RandomForest requires at least one row and one feature.");
  if (n >= (1ll << 31)) return fail(nullptr, PIO_ALS_ERR_ARG, "at most 2^31 - 1 rows are supported.");
  return PIO_ALS_OK;
}

// the regressor's checks (tests/forest_reg_ref.py check_args / check_data), all before any device work; *shift: s
static int rf_check_reg(const pio_rf_params* p, const int32_t* arity, const double* label, const double* x, int64_t n,
                        int F, int* shift) {
  if (p->impurity != RF_VARIANCE) {
    if (p->impurity == RF_GINI || p->impurity == RF_ENTROPY)
      return fail(nullptr, PIO_ALS_ERR_ARG, "DecisionTree Strategy given invalid impurity for Regression: %s.  Valid "
                  "settings: Variance", p->impurity == RF_GINI ? "gini" : "entropy");
    return fail(nullptr, PIO_ALS_ERR_ARG, "unknown impurity code %d", p->impurity);
  }
  for (int f = 0; arity && f < F; ++f)
    if (arity[f] != 0 && arity[f] < 2)
      return fail(nullptr, PIO_ALS_ERR_ARG, "DecisionTree Strategy given invalid categoricalFeaturesInfo setting: "
                  "feature %d has %d categories.  The number of categories should be >= 2.", f, arity[f]);
  if (p->num_trees < 1)
    return fail(nullptr, PIO_ALS_ERR_ARG, "RandomForest requires numTrees > 0, but was given numTrees = %d.",
                p->num_trees);
  if (rf_subset_size_reg(p->feature_subset_strategy, F > 1 ? F : 1, p->num_trees) == 0)
    return fail(nullptr, PIO_ALS_ERR_ARG, "RandomForest given invalid featureSubsetStrategy: %s. Supported values: "
                "auto, all, onethird, sqrt, log2, (0.0-1.0], [1-n].",
                p->feature_subset_strategy ? p->feature_subset_strategy : "null");
  pio_rf_params q = *p;                                   // the classifier's remaining numeric and shape checks
  q.num_classes = 2, q.impurity = RF_GINI, q.feature_subset_strategy = "all";
  EVF(rf_check_params(&q, n, F));
  if (!label || !x) return fail(nullptr, PIO_ALS_ERR_ARG, "bad pio_rf_train_regressor arguments");
  for (int64_t r = 0; r < n; ++r) EVF(rf_fail_finite(r, label[r], x + r * F, F));
  double m = 0.0;
  int64_t rm = 0;
  for (int64_t r = 0; r < n; ++r)
    if (fabs(label[r]) > m) m = fabs(label[r]), rm = r;
  if (m >= ldexp(1.0, RF_LABEL_EXP_MAX) || (m > 0.0 && m < ldexp(1.0, -RF_LABEL_EXP_MAX)))
    return fail(nullptr, PIO_ALS_ERR_ARG, "label of row %lld is out of range (%s): the largest |label| must be 0 or in "
                "[2^-%d, 2^%d).", (long long)rm, rf_fmt(label[rm]).c_str(), RF_LABEL_EXP_MAX, RF_LABEL_EXP_MAX);
  *shift = rf_label_shift(m);
  if (!arity) return PIO_ALS_OK;
  int amax = 0, fmax = -1;
  for (int f = 0; f < F; ++f)
    if (arity[f] > amax) amax = arity[f], fmax = f;
  const int64_t nb = std::min<int64_t>(p->max_bins, n);
  if (amax > nb)
    return fail(nullptr, PIO_ALS_ERR_ARG, "DecisionTree requires maxBins (= %lld) to be at least as large as the number "
                "of values in each categorical feature, but categorical feature %d has %d values. Consider removing "
                "this and other categorical features with a large number of values, or add more training examples.",
                (long long)nb, fmax, amax);
  for (int64_t r = 0; r < n; ++r)
    for (int f = 0; f < F; ++f) {
      const double v = x[r * F + f];
      if (arity[f] > 0 && !(v >= 0.0 && v < (double)arity[f]))
        return fail(nullptr, PIO_ALS_ERR_ARG, "DecisionTree given invalid data: Feature %d is categorical with values "
                    "in {0,...,%d}, but a data point gives it value %s.", f, arity[f] - 1, rf_fmt(v).c_str());
    }
  return PIO_ALS_OK;
}

static int rf_check(const pio_rf_params* p, const double* label, const double* x, int64_t n, int F) {
  EVF(rf_check_params(p, n, F));
  if (!label || !x) return fail(nullptr, PIO_ALS_ERR_ARG, "bad pio_rf_train arguments");
  for (int64_t r = 0; r < n; ++r) EVF(rf_fail_finite(r, label[r], x + r * F, F));
  for (int64_t r = 0; r < n; ++r) EVF(rf_fail_label(p, label[r]));
  return PIO_ALS_OK;
}

static double rf_ms(std::chrono::steady_clock::time_point& t0) {
  const auto t = std::chrono::steady_clock::now();
  const double ms = std::chrono::duration<double, std::milli>(t - t0).count();
  t0 = t;
  return ms;
}

// LearningNode.toNode(prune = true): an internal node whose two children end as leaves with the same prediction becomes
// a leaf; returns the node's prediction
// (the regressor compares its fp64 predictions with ==; the collapsed leaf keeps the left child's)
static int rf_prune(RfTree& t, int64_t i) {
  RfRec& r = t[i];
  if (r.leaf) return r.pred;
  const int a = rf_prune(t, 2 * i), b = rf_prune(t, 2 * i + 1);
  const RfRec &L = t[2 * i], &R = t[2 * i + 1];
  if (L.leaf && R.leaf && a == b && L.value == R.value) {
    r.leaf = true, r.pred = a, r.value = L.value, r.feature = -1, r.thr = 0.0, r.gain = 0.0;
    r.cats.clear();
  }
  return r.pred;
}
// preorder: the node, its left subtree, its right subtree; returns the node's index in the flat arrays
static int32_t rf_emit(const RfTree& t, int64_t i, pio_rf_forest* o) {
  const RfRec& r = t.at(i);
  const int32_t me = (int32_t)o->feature.size();
  o->feature.push_back(r.leaf ? -1 : r.feature);
  o->threshold.push_back(r.leaf ? 0.0 : r.thr);
  o->left.push_back(-1);
  o->right.push_back(-1);
  o->prediction.push_back(r.pred);
  o->impurity.push_back(r.imp);
  o->gain.push_back(r.leaf ? 0.0 : r.gain);
  o->count.push_back(r.count);
  if (o->regression) {
    o->value.push_back(r.value);
    if (!r.leaf) o->cat_ids.insert(o->cat_ids.end(), r.cats.begin(), r.cats.end());
    o->cat_off.push_back((int64_t)o->cat_ids.size());
  }
  if (!r.leaf) {
    const int32_t l = rf_emit(t, 2 * i, o);
    o->left[me] = l;
    const int32_t rr = rf_emit(t, 2 * i + 1, o);
    o->right[me] = rr;
  }
  return me;
}

struct RfCtx {
  CallMem* tmp;
  cudaStream_t st;
  int sm;
  const pio_rf_params* p;
  int64_t n;
  int F, K, C, NB;
  const double* dx;
  const uint8_t* dcls;
  const double* dthr;
  const int* doff;
  const int* dnthr;
  const std::vector<std::vector<double>>* thr;
  pio_rf_forest* out;
  // the regressor (else nullptr / empty): quantised labels, categories per feature (0: continuous), 2^-s and 2^-2s
  const long long* dyq;
  const int* darity;
  const std::vector<int>* arity;
  double scale1, scale2;
};

// the fp64 statistics of integer sums (tests/forest_reg_ref.py to_f64), and the node record they give
static RfRec rf_var_rec(const unsigned long long* e, double scale1, double scale2) {
  const unsigned __int128 sq = ((unsigned __int128)e[2] << 64) | e[1], qq = ((unsigned __int128)e[4] << 64) | e[3];
  const double W = (double)e[0], S = (double)(__int128)sq * scale1, Q = (double)qq * scale2;
  RfRec r{true, -1, 0.0, rf_variance(W, S, Q), 0.0, 0, (int64_t)e[0]};
  r.value = W == 0.0 ? 0.0 : S / W;
  return r;
}

using RfActive = std::vector<std::pair<int, int64_t>>;   // (tree of the group, heap index) of each slot of a level

// The regressor's split selection for the slots [c0, c1) of a level whose histogram chunk is in dhist: the centroid
// order of wide categorical features, select_var_kernel, then on the host each slot's first maximum over its subset
// features (hbest[S * K + s]: its subset position, -1 for none) and, for a categorical split, its left categories
// (hcats[s], ascending), read before the next chunk overwrites the split order.
static int rf_select_var(const RfCtx& c, int level, const RfActive& active, const std::vector<int>& hsub, int64_t c0,
                         int64_t c1, const unsigned long long* dhist, const int* dsub, uint32_t* dorder, double* dcen,
                         int2* dseg, double* dgain, int* dbest, unsigned long long* dleft, unsigned long long* dtot,
                         std::vector<double>& hgain, std::vector<int>& hbest,
                         std::vector<std::vector<int32_t>>& hcats) {
  const int K = c.K, NB = c.NB;
  const int64_t S = (int64_t)active.size();
  const cudaStream_t st = c.st;
  const std::vector<int>& ar = *c.arity;
  std::vector<int2> seg;
  int amax = 0;
  for (int64_t s = c0; s < c1; ++s)
    for (int kk = 0; kk < K; ++kk) {
      const int f = hsub[(size_t)s * K + kk];
      if (ar[f] > rf::CAT_SMEM_ARITY) seg.push_back(make_int2((int)(s - c0), kk)), amax = std::max(amax, ar[f]);
    }
  if (!seg.empty()) {
    CK0(cudaMemcpyAsync(dseg, seg.data(), sizeof(int2) * seg.size(), cudaMemcpyHostToDevice, st));
    const dim3 g((unsigned)((amax + 255) / 256), (unsigned)seg.size());
    rf::cat_centroid_kernel<<<g, 256, 0, st>>>(dhist, dseg, dsub, c.darity, K, NB, (int)c0, c.scale1, dcen);
    rf::cat_rank_kernel<<<g, 256, 0, st>>>(dcen, dseg, dsub, c.darity, K, NB, (int)c0, dorder);
  }
  rf::VarSelArgs sa{dhist, dsub, c.dnthr, c.darity, dorder, dgain, dbest, dleft, dtot, c.scale1, c.scale2, K, NB,
                    (int)c0, (int)c0};
  rf::select_var_kernel<<<(unsigned)((c1 - c0) * K), rf::SEL_WARPS * 32, 0, st>>>(sa);
  CK0(cudaGetLastError());
  const size_t m = (size_t)(c1 - c0) * K;
  CK0(cudaMemcpyAsync(&hgain[c0 * K], dgain + c0 * K, 8 * m, cudaMemcpyDeviceToHost, st));
  CK0(cudaMemcpyAsync(&hbest[c0 * K], dbest + c0 * K, 4 * m, cudaMemcpyDeviceToHost, st));
  CK0(cudaStreamSynchronize(st));
  for (int64_t s = c0; s < c1; ++s) {
    int pick = -1;
    for (int kk = 0; kk < K; ++kk)                       // the first maximum: earlier subset features win ties
      if (hbest[s * K + kk] >= 0 && (pick < 0 || hgain[s * K + kk] > hgain[s * K + pick])) pick = kk;
    hbest[S * K + s] = pick;
    if (pick < 0 || !(hgain[s * K + pick] > 0.0) || level == c.p->max_depth) continue;
    const int f = hsub[(size_t)s * K + pick], j = hbest[s * K + pick];
    if (ar[f] == 0) continue;
    hcats[s].resize((size_t)j + 1);
    CK0(cudaMemcpyAsync(hcats[s].data(), dorder + ((s - c0) * K + pick) * (int64_t)NB, 4 * ((size_t)j + 1),
                        cudaMemcpyDeviceToHost, st));
  }
  CK0(cudaStreamSynchronize(st));
  for (int64_t s = c0; s < c1; ++s) std::sort(hcats[s].begin(), hcats[s].end());
  return PIO_ALS_OK;
}

// The regressor's decisions for a level (tests/forest_reg_ref.py _decide): node records, leaves, children, the next
// level's slots (`next`) and the rows' moves (update_kernel<BinT, true>, with a bit mask per categorical split).
template <typename BinT>
static int rf_decide_var(const RfCtx& c, int level, const RfActive& active, const std::vector<int>& hsub,
                         const std::vector<double>& hgain, const std::vector<int>& hbest,
                         const std::vector<std::vector<int32_t>>& hcats, const unsigned long long* dleft,
                         const unsigned long long* dtot, int* dnode, const BinT* dbins, int G, unsigned ugrid, Scratch& lv,
                         std::vector<RfTree>& trees, std::chrono::steady_clock::time_point& t0, RfActive& next) {
  const int K = c.K, W = rf::VAR_WORDS, max_depth = c.p->max_depth;
  const int64_t S = (int64_t)active.size();
  const cudaStream_t st = c.st;
  std::vector<unsigned long long> hleft((size_t)S * K * W), htot((size_t)S * W);
  CK0(cudaMemcpyAsync(hleft.data(), dleft, 8 * hleft.size(), cudaMemcpyDeviceToHost, st));
  CK0(cudaMemcpyAsync(htot.data(), dtot, 8 * htot.size(), cudaMemcpyDeviceToHost, st));
  CK0(cudaStreamSynchronize(st));
  std::vector<int4> upd(S);
  std::vector<long long> moff(S, -1);
  std::vector<uint32_t> mask;
  for (int64_t s = 0; s < S; ++s) {
    const int g = active[s].first;
    const int64_t i = active[s].second;
    const unsigned long long* tot = &htot[(size_t)s * W];
    RfRec rec = rf_var_rec(tot, c.scale1, c.scale2);
    const int kk = hbest[S * K + s];
    if (kk < 0 || !(hgain[s * K + kk] > 0.0) || level == max_depth) {
      trees[g][i] = rec;
      upd[s] = make_int4(-1, 0, -1, -1);
      continue;
    }
    const int f = hsub[(size_t)s * K + kk], j = hbest[s * K + kk], ar = (*c.arity)[f];
    rec.leaf = false, rec.feature = f, rec.gain = hgain[s * K + kk];
    if (ar > 0) {
      rec.cats = hcats[s];
      moff[s] = (long long)mask.size();
      mask.resize(mask.size() + (size_t)(ar + 31) / 32, 0u);
      for (int32_t cat : rec.cats) mask[moff[s] + (cat >> 5)] |= 1u << (cat & 31);
    } else {
      rec.thr = (*c.thr)[f][j];
    }
    trees[g][i] = rec;
    unsigned long long side_st[2][rf::VAR_WORDS];
    const unsigned long long* L = &hleft[((size_t)s * K + kk) * W];
    memcpy(side_st[0], L, sizeof side_st[0]);
    const unsigned __int128 ts = ((unsigned __int128)tot[2] << 64) | tot[1], tq = ((unsigned __int128)tot[4] << 64) | tot[3];
    const unsigned __int128 ls = ((unsigned __int128)L[2] << 64) | L[1], lq = ((unsigned __int128)L[4] << 64) | L[3];
    const unsigned __int128 rs = ts - ls, rq = tq - lq;
    side_st[1][0] = tot[0] - L[0];
    side_st[1][1] = (unsigned long long)rs, side_st[1][2] = (unsigned long long)(rs >> 64);
    side_st[1][3] = (unsigned long long)rq, side_st[1][4] = (unsigned long long)(rq >> 64);
    int child_slot[2];
    for (int side = 0; side < 2; ++side) {
      const RfRec cr = rf_var_rec(side_st[side], c.scale1, c.scale2);
      const int64_t child = 2 * i + side;
      if (level + 1 == max_depth || cr.imp == 0.0) {
        trees[g][child] = cr;
        child_slot[side] = -1;
      } else {
        child_slot[side] = (int)next.size();
        next.push_back({g, child});
      }
    }
    upd[s] = make_int4(f, j, child_slot[0], child_slot[1]);
  }
  if (!next.empty()) {
    int4* dupd = nullptr;
    long long* dmoff = nullptr;
    uint32_t* dmask = nullptr;
    CK0(lv.alloc(&dupd, (size_t)S));
    CK0(lv.alloc(&dmoff, (size_t)S));
    CK0(lv.alloc(&dmask, std::max<size_t>(1, mask.size())));
    CK0(cudaMemcpyAsync(dupd, upd.data(), sizeof(int4) * (size_t)S, cudaMemcpyHostToDevice, st));
    CK0(cudaMemcpyAsync(dmoff, moff.data(), 8 * (size_t)S, cudaMemcpyHostToDevice, st));
    if (!mask.empty()) CK0(cudaMemcpyAsync(dmask, mask.data(), 4 * mask.size(), cudaMemcpyHostToDevice, st));
    rf::update_kernel<BinT, true><<<ugrid, rf::THREADS, 0, st>>>(dnode, c.n, G, dbins, c.F, dupd, dmoff, dmask);
    CK0(cudaGetLastError());
    CK0(cudaStreamSynchronize(st));
    g_rf_timing.upd += rf_ms(t0);
  }
  return PIO_ALS_OK;
}

// bin codes, then every tree group level by level; REG: the regressor's statistics and splits (forest.cuh)
template <typename BinT, bool REG = false>
static int rf_bin_and_grow(const RfCtx& c) {
  CallMem& tmp = *c.tmp;
  const cudaStream_t st = c.st;
  const int64_t n = c.n;
  const int F = c.F, K = c.K, C = c.C, NB = c.NB, T = c.p->num_trees, max_depth = c.p->max_depth;
  const int64_t seed = c.p->seed;
  RfTiming& tm = g_rf_timing;
  auto t0 = std::chrono::steady_clock::now();
  BinT* dbins = nullptr;
  CK0(tmp.device(&dbins, (size_t)n * F));
  std::vector<int> hoff(F + 1, 0);
  for (int f = 0; f < F; ++f) hoff[f + 1] = hoff[f] + (int)(*c.thr)[f].size();
  const size_t thr_bytes = sizeof(double) * (size_t)hoff[F];
  const int staged = thr_bytes <= 48 * 1024 ? 1 : 0;
  const unsigned bgrid = (unsigned)std::min<int64_t>(nblk(n * F, rf::THREADS), (int64_t)c.sm * 16);
  rf::bin_kernel<BinT><<<bgrid, rf::THREADS, staged ? thr_bytes : 0, st>>>(c.dx, n, F, c.dthr, c.doff, staged, dbins,
                                                                           c.darity);
  CK0(cudaGetLastError());
  CK0(cudaStreamSynchronize(st));
  tm.bin = rf_ms(t0);
  tm.bin_bytes = (int)sizeof(BinT), tm.staged = staged;

  // PIO_RF_TREES_PER_PASS / PIO_RF_HIST_BUDGET (bytes): tree grouping and histogram chunking for tests; neither changes
  // the forest
  const char* env = getenv("PIO_RF_TREES_PER_PASS");
  const char* env_hb = getenv("PIO_RF_HIST_BUDGET");
  const int64_t hist_budget = env_hb && atoll(env_hb) > 0 ? atoll(env_hb) : RF_HIST_BUDGET;
  const auto groups = rf_plan_groups(T, n, RF_NODE_BUDGET, env ? atoi(env) : 0);
  int gmax = 0;
  for (const auto& g : groups) gmax = std::max(gmax, g.second - g.first);
  int* dnode = nullptr;
  uint64_t* dbag = nullptr;
  CK0(tmp.device(&dnode, (size_t)n * gmax));
  CK0(tmp.device(&dbag, (size_t)gmax));
  rf::Cdf cdf;
  rf_poisson_table(cdf.v);
  // a histogram entry: C class counts (8 bytes global, 4 in shared memory), or one variance entry of 5 words in both
  const int64_t slot_bytes = REG ? (int64_t)K * NB * rf::VAR_WORDS * 8 : (int64_t)K * NB * C * 8;
  const int64_t smem_slot = REG ? slot_bytes : (int64_t)K * NB * C * 4;
  bool any_cat = false, wide_cat = false;
  if (REG)
    for (int a : *c.arity) any_cat |= a > 0, wide_cat |= a > rf::CAT_SMEM_ARITY;
  // the regressor's chunk also holds the split order (4 bytes per bin) and, for wide categorical features, the centroids
  // (8 bytes per bin) of each slot
  const int64_t chunk_slot_bytes = slot_bytes + (any_cat ? (int64_t)K * NB * 4 : 0) + (wide_cat ? (int64_t)K * NB * 8 : 0);
  const int64_t chunk_max = std::max<int64_t>(1, hist_budget / chunk_slot_bytes);
  const int64_t pass_slots = RF_SMEM / smem_slot;
  if (pass_slots >= 1) {
    CK0(cudaFuncSetAttribute(rf::hist_kernel<BinT, true, REG>, cudaFuncAttributeMaxDynamicSharedMemorySize, RF_SMEM));
  }
  const unsigned ugrid = (unsigned)std::min<int64_t>(nblk(n * gmax, rf::THREADS), (int64_t)c.sm * 16);
  tm.groups = (int)groups.size();
  for (const auto& grp : groups) {
    const int t_first = grp.first, G = grp.second - grp.first;
    rf::root_kernel<<<ugrid, rf::THREADS, 0, st>>>(dnode, n, G);
    std::vector<uint64_t> hbag(G);
    for (int g = 0; g < G; ++g) hbag[g] = rf_stream(seed, RF_TAG_BAG, (uint64_t)(t_first + g));
    CK0(cudaMemcpyAsync(dbag, hbag.data(), 8 * (size_t)G, cudaMemcpyHostToDevice, st));
    std::vector<RfTree> trees(G);
    std::vector<std::pair<int, int64_t>> active;
    for (int g = 0; g < G; ++g) active.push_back({g, 1});
    for (int level = 0; !active.empty(); ++level) {
      const int64_t S = (int64_t)active.size();
      if (S >= (1ll << 31) / std::max(K, C)) return fail(nullptr, PIO_ALS_ERR_ARG, "too many nodes in one level");
      std::vector<int> hsub((size_t)S * K);
      for (int64_t s = 0; s < S; ++s)
        rf_node_subset(rf_stream(seed, RF_TAG_SUBSET, (uint64_t)(t_first + active[s].first)), active[s].second, F, K,
                       &hsub[(size_t)s * K]);
      Scratch lv(st);
      int *dsub = nullptr, *dbest = nullptr;
      double* dgain = nullptr;
      long long *dleft = nullptr, *dtot = nullptr;
      unsigned long long* dhist = nullptr;
      const int64_t cap = std::min<int64_t>(S, chunk_max);
      // the classifier: best split and class counts per slot; the regressor: the best split of every subset feature,
      // variance entries, and the split order of categorical features
      const int64_t per_sel = REG ? K : 1, words = REG ? rf::VAR_WORDS : C;
      CK0(lv.alloc(&dsub, (size_t)S * K));
      CK0(lv.alloc(&dbest, (size_t)S * per_sel * 2));
      CK0(lv.alloc(&dgain, (size_t)S * per_sel));
      CK0(lv.alloc(&dleft, (size_t)S * per_sel * words));
      CK0(lv.alloc(&dtot, (size_t)S * words));
      CK0(lv.alloc(&dhist, (size_t)cap * K * NB * words));
      uint32_t* dorder = nullptr;
      double* dcen = nullptr;
      int2* dseg = nullptr;
      if (REG && any_cat) CK0(lv.alloc(&dorder, (size_t)cap * K * NB));
      if (REG && wide_cat) {
        CK0(lv.alloc(&dcen, (size_t)cap * K * NB));
        CK0(lv.alloc(&dseg, (size_t)cap * K));
      }
      std::vector<double> hgain(S * per_sel);
      std::vector<int> hbest(2 * S * per_sel);
      std::vector<std::vector<int32_t>> hcats(REG ? S : 0);
      CK0(cudaMemcpyAsync(dsub, hsub.data(), 4 * hsub.size(), cudaMemcpyHostToDevice, st));
      CK0(cudaStreamSynchronize(st));
      rf_ms(t0);
      tm.max_chunks = std::max(tm.max_chunks, (S + cap - 1) / cap);
      for (int64_t c0 = 0; c0 < S; c0 += cap) {
        const int64_t c1 = std::min(S, c0 + cap);
        CK0(cudaMemsetAsync(dhist, 0, (size_t)(c1 - c0) * slot_bytes, st));
        rf::HistArgs a{c.dcls, dbins, dnode, T > 1 ? dbag : nullptr, dsub, dhist, n, F, G, K, NB, C,
                       (int)c0, (int)c1, (int)c0, active[c0].first, active[c1 - 1].first, cdf, c.dyq};
        if (pass_slots >= 1) {
          const unsigned grid = (unsigned)std::min<int64_t>(nblk(n, rf::THREADS), (int64_t)c.sm * 2);
          for (int64_t p0 = c0; p0 < c1; p0 += pass_slots) {
            a.s0 = (int)p0;
            a.s1 = (int)std::min(c1, p0 + pass_slots);
            a.g0 = active[a.s0].first;
            a.g1 = active[a.s1 - 1].first;
            rf::hist_kernel<BinT, true, REG><<<grid, rf::THREADS, (size_t)(a.s1 - a.s0) * smem_slot, st>>>(a);
          }
          const int64_t passes = (c1 - c0 + pass_slots - 1) / pass_slots;
          tm.smem_launches += passes, tm.max_passes = std::max(tm.max_passes, passes);
        } else {
          const unsigned grid = (unsigned)std::min<int64_t>(nblk(n, rf::THREADS), (int64_t)c.sm * 8);
          rf::hist_kernel<BinT, false, REG><<<grid, rf::THREADS, 0, st>>>(a);
          ++tm.global_launches;
        }
        CK0(cudaGetLastError());
        CK0(cudaStreamSynchronize(st));
        const double hm = rf_ms(t0);
        tm.hist += hm, tm.hist_l[level] += hm;
        if constexpr (REG) {
          EVF(rf_select_var(c, level, active, hsub, c0, c1, dhist, dsub, dorder, dcen, dseg, dgain, dbest,
                            (unsigned long long*)dleft, (unsigned long long*)dtot, hgain, hbest, hcats));
        } else {
          rf::SelArgs sa{dhist, dsub, c.dnthr, dgain, dbest, dleft, dtot, K, NB, C, c.p->impurity, (int)c0, (int)c0};
          rf::select_kernel<<<(unsigned)(c1 - c0), rf::SEL_WARPS * 32, 0, st>>>(sa);
        }
        CK0(cudaGetLastError());
        CK0(cudaStreamSynchronize(st));
        const double sm_ = rf_ms(t0);
        tm.sel += sm_, tm.sel_l[level] += sm_;
      }
      if constexpr (REG) {
        std::vector<std::pair<int, int64_t>> next;
        EVF(rf_decide_var<BinT>(c, level, active, hsub, hgain, hbest, hcats, (const unsigned long long*)dleft,
                                (const unsigned long long*)dtot, dnode, dbins, G, ugrid, lv, trees, t0, next));
        tm.levels = std::max(tm.levels, level + 1);
        active.swap(next);
        continue;
      }
      std::vector<int64_t> hleft(S * C), htot(S * C);
      CK0(cudaMemcpyAsync(hgain.data(), dgain, 8 * (size_t)S, cudaMemcpyDeviceToHost, st));
      CK0(cudaMemcpyAsync(hbest.data(), dbest, 8 * (size_t)S, cudaMemcpyDeviceToHost, st));
      CK0(cudaMemcpyAsync(hleft.data(), dleft, 8 * (size_t)S * C, cudaMemcpyDeviceToHost, st));
      CK0(cudaMemcpyAsync(htot.data(), dtot, 8 * (size_t)S * C, cudaMemcpyDeviceToHost, st));
      CK0(cudaStreamSynchronize(st));
      // the level's decisions (tests/forest_ref.py train): leaves, splits, children and the next level's slots
      std::vector<int4> upd(S);
      std::vector<std::pair<int, int64_t>> next;
      std::vector<int64_t> cc(C);
      for (int64_t s = 0; s < S; ++s) {
        const int g = active[s].first;
        const int64_t i = active[s].second;
        const int64_t* tot = &htot[s * C];
        int64_t cnt = 0;
        for (int k = 0; k < C; ++k) cnt += tot[k];
        RfRec rec{true, -1, 0.0, rf_impurity(tot, C, c.p->impurity), 0.0, rf_argmax(tot, C), cnt};
        const int kk = hbest[2 * s];
        if (kk < 0 || !(hgain[s] > 0.0) || level == max_depth) {
          trees[g][i] = rec;
          upd[s] = make_int4(-1, 0, -1, -1);
          continue;
        }
        const int f = hsub[(size_t)s * K + kk], j = hbest[2 * s + 1];
        rec.leaf = false, rec.feature = f, rec.thr = (*c.thr)[f][j], rec.gain = hgain[s];
        trees[g][i] = rec;
        int child_slot[2];
        for (int side = 0; side < 2; ++side) {
          int64_t ccount = 0;
          for (int k = 0; k < C; ++k) {
            cc[k] = side == 0 ? hleft[s * C + k] : tot[k] - hleft[s * C + k];
            ccount += cc[k];
          }
          const double ci = rf_impurity(cc.data(), C, c.p->impurity);
          const int64_t child = 2 * i + side;
          if (level + 1 == max_depth || ci == 0.0) {
            trees[g][child] = RfRec{true, -1, 0.0, ci, 0.0, rf_argmax(cc.data(), C), ccount};
            child_slot[side] = -1;
          } else {
            child_slot[side] = (int)next.size();
            next.push_back({g, child});
          }
        }
        upd[s] = make_int4(f, j, child_slot[0], child_slot[1]);
      }
      if (!next.empty()) {
        int4* dupd = nullptr;
        CK0(lv.alloc(&dupd, (size_t)S));
        CK0(cudaMemcpyAsync(dupd, upd.data(), sizeof(int4) * (size_t)S, cudaMemcpyHostToDevice, st));
        rf::update_kernel<BinT><<<ugrid, rf::THREADS, 0, st>>>(dnode, n, G, dbins, F, dupd);
        CK0(cudaGetLastError());
        CK0(cudaStreamSynchronize(st));
        tm.upd += rf_ms(t0);
      }
      tm.levels = std::max(tm.levels, level + 1);
      active.swap(next);
    }
    for (int g = 0; g < G; ++g) {
      rf_prune(trees[g], 1);
      rf_emit(trees[g], 1, c.out);
      c.out->tree_off.push_back((int32_t)c.out->feature.size());
    }
  }
  return PIO_ALS_OK;
}

// what the regressor adds to rf_fit: device quantised labels and categories per feature (host and device), 2^-s, 2^-2s
struct RfReg {
  const long long* dyq;
  const int* darity;
  std::vector<int> arity;
  double scale1, scale2;
};

// The forest from n rows already on the device (dx: n x F fp64, dcls: class bytes, or reg for the regressor) on stream
// st: split search, bin codes, then every tree group level by level.  pio_rf_train, pio_rf_train_regressor and
// pio_cls_folds_rf_train end here; g_rf_timing's later phases are timed from t0.
static int rf_fit(const pio_rf_params* p, const double* dx, const uint8_t* dcls, int64_t n, int F, int sm, CallMem& tmp,
                  cudaStream_t st, std::chrono::steady_clock::time_point t0, pio_rf_forest** out,
                  const RfReg* reg = nullptr) {
  const int C = reg ? 1 : p->num_classes;
  const int K = reg ? rf_subset_size_reg(p->feature_subset_strategy, F, p->num_trees)
                    : rf_subset_size(p->feature_subset_strategy, F, p->num_trees);
  RfTiming& tm = g_rf_timing;
  // split sample, then per feature its sorted distinct values: thresholds on the host (findSplitsForContinuousFeature)
  const double frac = rf_sample_fraction(n, p->max_bins);
  uint32_t* rows = nullptr;
  int64_t m = n;
  if (frac < 1.0) {
    uint32_t *flag = nullptr, *pos = nullptr;
    CK0(tmp.device(&flag, (size_t)n));
    CK0(tmp.device(&pos, (size_t)n));
    rf::sample_flag_kernel<<<nblk(n, 256), 256, 0, st>>>(n, rf_stream(p->seed, RF_TAG_SAMPLE, 0), frac, flag);
    CK0(scan_exclusive_u32(flag, pos, (size_t)n, st, nullptr));
    uint32_t lf = 0, lp = 0;
    CK0(cudaMemcpyAsync(&lf, flag + n - 1, 4, cudaMemcpyDeviceToHost, st));
    CK0(cudaMemcpyAsync(&lp, pos + n - 1, 4, cudaMemcpyDeviceToHost, st));
    CK0(cudaStreamSynchronize(st));
    m = (int64_t)lp + lf;
    CK0(tmp.device(&rows, (size_t)m));
    rf::sample_compact_kernel<<<nblk(n, 256), 256, 0, st>>>(flag, pos, n, rows);
    CK0(cudaGetLastError());
  }
  std::vector<std::vector<double>> thr(F);
  if (m > 0) {
    SortBufs sb;
    uint32_t *head = nullptr, *rpos = nullptr, *rstart = nullptr;
    uint64_t* rkey = nullptr;
    for (int i : {0, 1}) {
      CK0(tmp.device(&sb.k[i], (size_t)m));
      CK0(tmp.device(&sb.v[i], (size_t)m));
    }
    CK0(tmp.device(&head, (size_t)m));
    CK0(tmp.device(&rpos, (size_t)m));
    CK0(tmp.device(&rkey, (size_t)m));
    CK0(tmp.device(&rstart, (size_t)m));
    std::vector<uint64_t> hk;
    std::vector<uint32_t> hs;
    std::vector<double> vals;
    std::vector<int64_t> cnts;
    for (int f = 0; f < F; ++f) {
      if (reg && reg->arity[f] > 0) continue;             // categorical: no thresholds, its bins are its categories
      sb.live = 0;
      rf::sample_keys_kernel<<<nblk(m, 256), 256, 0, st>>>(dx, F, f, rows, m, sb.keys(), sb.vals());
      CK0(radix_sort_pairs(sb, (size_t)m, 64, st, nullptr));
      rf::run_head_kernel<<<nblk(m, 256), 256, 0, st>>>(sb.keys(), m, head);
      CK0(scan_exclusive_u32(head, rpos, (size_t)m, st, nullptr));
      rf::run_compact_kernel<<<nblk(m, 256), 256, 0, st>>>(sb.keys(), head, rpos, m, rkey, rstart);
      CK0(cudaGetLastError());
      uint32_t lh = 0, lp = 0;
      CK0(cudaMemcpyAsync(&lh, head + m - 1, 4, cudaMemcpyDeviceToHost, st));
      CK0(cudaMemcpyAsync(&lp, rpos + m - 1, 4, cudaMemcpyDeviceToHost, st));
      CK0(cudaStreamSynchronize(st));
      const int64_t runs = (int64_t)lp + lh;
      hk.resize(runs);
      hs.resize(runs);
      CK0(cudaMemcpyAsync(hk.data(), rkey, 8 * (size_t)runs, cudaMemcpyDeviceToHost, st));
      CK0(cudaMemcpyAsync(hs.data(), rstart, 4 * (size_t)runs, cudaMemcpyDeviceToHost, st));
      CK0(cudaStreamSynchronize(st));
      vals.resize(runs);
      cnts.resize(runs);
      for (int64_t i = 0; i < runs; ++i) {
        const uint64_t b = (hk[i] >> 63) ? (hk[i] & ~(1ull << 63)) : ~hk[i];
        memcpy(&vals[i], &b, 8);
        cnts[i] = (i + 1 < runs ? (int64_t)hs[i + 1] : m) - (int64_t)hs[i];
      }
      rf_thresholds(vals.data(), cnts.data(), runs, std::min<int64_t>(p->max_bins, n), thr[f]);
    }
  }
  std::vector<double> hthr;
  std::vector<int> hoff(F + 1, 0), hnthr(F);
  for (int f = 0; f < F; ++f) {
    hthr.insert(hthr.end(), thr[f].begin(), thr[f].end());
    hnthr[f] = (int)thr[f].size();
    hoff[f + 1] = (int)hthr.size();
  }
  int NB = *std::max_element(hnthr.begin(), hnthr.end()) + 1;
  if (reg)
    for (int a : reg->arity) NB = std::max(NB, a);
  double* dthr = nullptr;
  int *doff = nullptr, *dnthr = nullptr;
  CK0(tmp.device(&dthr, hthr.size()));
  CK0(tmp.device(&doff, (size_t)F + 1));
  CK0(tmp.device(&dnthr, (size_t)F));
  if (!hthr.empty())
    CK0(cudaMemcpyAsync(dthr, hthr.data(), 8 * hthr.size(), cudaMemcpyHostToDevice, st));
  CK0(cudaMemcpyAsync(doff, hoff.data(), 4 * hoff.size(), cudaMemcpyHostToDevice, st));
  CK0(cudaMemcpyAsync(dnthr, hnthr.data(), 4 * hnthr.size(), cudaMemcpyHostToDevice, st));
  CK0(cudaStreamSynchronize(st));
  tm.split = rf_ms(t0);

  pio_rf_forest* fo = new pio_rf_forest();
  fo->n_trees = p->num_trees;
  fo->n_class = C;
  fo->tree_off.push_back(0);
  fo->regression = reg != nullptr;
  if (reg) fo->n_class = 0, fo->cat_off.push_back(0);
  RfCtx ctx{&tmp, st, sm, p, n, F, K, C, NB, dx, dcls, dthr, doff, dnthr, &thr, fo,
            reg ? reg->dyq : nullptr, reg ? reg->darity : nullptr, reg ? &reg->arity : nullptr,
            reg ? reg->scale1 : 0.0, reg ? reg->scale2 : 0.0};
  const int rc2 = reg ? (NB <= 256 ? rf_bin_and_grow<uint8_t, true>(ctx) : rf_bin_and_grow<uint16_t, true>(ctx))
                      : (NB <= 256 ? rf_bin_and_grow<uint8_t>(ctx) : rf_bin_and_grow<uint16_t>(ctx));
  if (rc2 != PIO_ALS_OK) {
    delete fo;
    return rc2;
  }
  *out = fo;
  return PIO_ALS_OK;
}

// a forest as the flat arrays of pio_rf_forest_get (HOST)
struct RfFlat {
  int32_t n_trees;
  const int32_t* tree_off;
  int64_t n_nodes;
  const int32_t *feature;
  const double* threshold;
  const int32_t *left, *right, *prediction;
  int32_t num_classes;
};

// a walk must end: children come after their parent (preorder) and stay in their tree
static int rf_check_flat(const RfFlat& a, int32_t n_feat) {
  if (!a.tree_off || !a.feature || !a.threshold || !a.left || !a.right || !a.prediction || a.n_trees < 1 ||
      a.n_nodes < 1 || a.n_nodes >= (1ll << 31) || a.num_classes < 1 || a.num_classes > RF_MAX_CLASSES || n_feat < 1)
    return fail(nullptr, PIO_ALS_ERR_ARG, "bad pio_rf_predict arguments");
  for (int32_t t = 0; t < a.n_trees; ++t) {
    const int64_t lo = a.tree_off[t], hi = t + 1 < a.n_trees ? a.tree_off[t + 1] : a.n_nodes;
    if (lo < 0 || lo >= hi || hi > a.n_nodes) return fail(nullptr, PIO_ALS_ERR_ARG, "bad tree offsets");
    for (int64_t i = lo; i < hi; ++i) {
      if (a.prediction[i] < 0 || a.prediction[i] >= a.num_classes) return fail(nullptr, PIO_ALS_ERR_ARG, "bad prediction");
      if (a.feature[i] >= n_feat) return fail(nullptr, PIO_ALS_ERR_ARG, "node %lld uses feature %d of %d", (long long)i,
                                              a.feature[i], n_feat);
      if (a.feature[i] >= 0 && (a.left[i] <= i || a.left[i] >= hi || a.right[i] <= i || a.right[i] >= hi))
        return fail(nullptr, PIO_ALS_ERR_ARG, "bad children at node %lld", (long long)i);
    }
  }
  return PIO_ALS_OK;
}

// the vote (class index) of n >= 1 device rows dx (n x F) into dout, on stream st
static int rf_predict_device(CallMem& tmp, cudaStream_t st, const RfFlat& a, const double* dx, int64_t n, int F,
                             int* dout) {
  const int64_t nn = a.n_nodes;
  int *dto = nullptr, *df = nullptr, *dl = nullptr, *dr = nullptr, *dp = nullptr;
  double* dt = nullptr;
  CK0(tmp.device(&dto, (size_t)a.n_trees));
  CK0(tmp.device(&df, (size_t)nn));
  CK0(tmp.device(&dl, (size_t)nn));
  CK0(tmp.device(&dr, (size_t)nn));
  CK0(tmp.device(&dp, (size_t)nn));
  CK0(tmp.device(&dt, (size_t)nn));
  CK0(cudaMemcpyAsync(dto, a.tree_off, 4 * (size_t)a.n_trees, cudaMemcpyHostToDevice, st));
  CK0(cudaMemcpyAsync(df, a.feature, 4 * (size_t)nn, cudaMemcpyHostToDevice, st));
  CK0(cudaMemcpyAsync(dl, a.left, 4 * (size_t)nn, cudaMemcpyHostToDevice, st));
  CK0(cudaMemcpyAsync(dr, a.right, 4 * (size_t)nn, cudaMemcpyHostToDevice, st));
  CK0(cudaMemcpyAsync(dp, a.prediction, 4 * (size_t)nn, cudaMemcpyHostToDevice, st));
  CK0(cudaMemcpyAsync(dt, a.threshold, 8 * (size_t)nn, cudaMemcpyHostToDevice, st));
  rf::predict_kernel<<<nblk(n, 128), 128, sizeof(int) * 128 * (size_t)a.num_classes, st>>>(
      dto, a.n_trees, df, dt, dl, dr, dp, a.num_classes, dx, n, F, dout);
  CK0(cudaGetLastError());
  return PIO_ALS_OK;
}

}  // namespace pio

extern "C" {

int pio_rf_train(int device, const pio_rf_params* p, const double* label, const double* x, int64_t n, int32_t n_feat,
                 pio_rf_forest** out) {
  if (!p || !out) return fail(nullptr, PIO_ALS_ERR_ARG, "bad pio_rf_train arguments");
  *out = nullptr;
  const int rc = rf_check(p, label, x, n, n_feat);
  if (rc != PIO_ALS_OK) return rc;
  g_rf_timing = RfTiming();
  RfTiming& tm = g_rf_timing;
  auto t0 = std::chrono::steady_clock::now();
  CK0(cudaSetDevice(device));
  int sm = 0;
  CK0(cudaDeviceGetAttribute(&sm, cudaDevAttrMultiProcessorCount, device));
  std::vector<uint8_t> hcls((size_t)n);
  for (int64_t r = 0; r < n; ++r) hcls[r] = (uint8_t)(int)trunc(label[r]);
  CallMem tmp;
  cudaStream_t st;
  CK0(tmp.stream(&st));
  double* dx = nullptr;
  uint8_t* dcls = nullptr;
  CK0(tmp.device(&dx, (size_t)n * n_feat));
  CK0(tmp.device(&dcls, (size_t)n));
  rf_ms(t0);
  CK0(cudaMemcpyAsync(dx, x, sizeof(double) * (size_t)n * n_feat, cudaMemcpyHostToDevice, st));
  CK0(cudaMemcpyAsync(dcls, hcls.data(), (size_t)n, cudaMemcpyHostToDevice, st));
  CK0(cudaStreamSynchronize(st));
  tm.h2d = rf_ms(t0);
  return rf_fit(p, dx, dcls, n, n_feat, sm, tmp, st, t0, out);
}

int pio_rf_forest_size(const pio_rf_forest* f, int32_t* n_trees, int64_t* n_nodes) {
  if (!f) return fail(nullptr, PIO_ALS_ERR_ARG, "null forest");
  if (n_trees) *n_trees = f->n_trees;
  if (n_nodes) *n_nodes = (int64_t)f->feature.size();
  return PIO_ALS_OK;
}

int pio_rf_forest_get(const pio_rf_forest* f, int32_t* tree_off, int32_t* feature, double* threshold, int32_t* left,
                      int32_t* right, int32_t* prediction, double* impurity, double* gain, int64_t* count) {
  if (!f) return fail(nullptr, PIO_ALS_ERR_ARG, "null forest");
  auto put = [](auto* dst, const auto& v) {
    if (dst && !v.empty()) memcpy(dst, v.data(), v.size() * sizeof(v[0]));
  };
  put(tree_off, f->tree_off);
  put(feature, f->feature);
  put(threshold, f->threshold);
  put(left, f->left);
  put(right, f->right);
  put(prediction, f->prediction);
  put(impurity, f->impurity);
  put(gain, f->gain);
  put(count, f->count);
  return PIO_ALS_OK;
}

int pio_rf_forest_destroy(pio_rf_forest* f) {
  delete f;
  return PIO_ALS_OK;
}

int pio_rf_predict(int device, int32_t n_trees, const int32_t* tree_off, int64_t n_nodes, const int32_t* feature,
                   const double* threshold, const int32_t* left, const int32_t* right, const int32_t* prediction,
                   int32_t num_classes, const double* x, int64_t n, int32_t n_feat, int32_t* out) {
  if (!out || n < 0 || (n > 0 && !x)) return fail(nullptr, PIO_ALS_ERR_ARG, "bad pio_rf_predict arguments");
  const RfFlat fl{n_trees, tree_off, n_nodes, feature, threshold, left, right, prediction, num_classes};
  EVF(rf_check_flat(fl, n_feat));
  if (n == 0) return PIO_ALS_OK;
  CK0(cudaSetDevice(device));
  CallMem tmp;
  cudaStream_t st;
  CK0(tmp.stream(&st));
  int* dout = nullptr;
  double* dx = nullptr;
  CK0(tmp.device(&dx, (size_t)n * n_feat));
  CK0(tmp.device(&dout, (size_t)n));
  CK0(cudaMemcpyAsync(dx, x, 8 * (size_t)n * n_feat, cudaMemcpyHostToDevice, st));
  EVF(rf_predict_device(tmp, st, fl, dx, n, n_feat, dout));
  CK0(cudaMemcpyAsync(out, dout, 4 * (size_t)n, cudaMemcpyDeviceToHost, st));
  CK0(cudaStreamSynchronize(st));
  return PIO_ALS_OK;
}

int pio_rf_train_regressor(int device, const pio_rf_params* p, const int32_t* arity, const double* label,
                           const double* x, int64_t n, int32_t n_feat, pio_rf_forest** out) {
  if (!p || !out) return fail(nullptr, PIO_ALS_ERR_ARG, "bad pio_rf_train_regressor arguments");
  *out = nullptr;
  int shift = 0;
  EVF(rf_check_reg(p, arity, label, x, n, n_feat, &shift));
  g_rf_timing = RfTiming();
  RfTiming& tm = g_rf_timing;
  auto t0 = std::chrono::steady_clock::now();
  CK0(cudaSetDevice(device));
  int sm = 0;
  CK0(cudaDeviceGetAttribute(&sm, cudaDevAttrMultiProcessorCount, device));
  RfReg reg;
  if (arity) reg.arity.assign(arity, arity + n_feat);
  else reg.arity.assign((size_t)n_feat, 0);
  reg.scale1 = ldexp(1.0, -shift), reg.scale2 = ldexp(1.0, -2 * shift);
  std::vector<long long> hyq((size_t)n);
  for (int64_t r = 0; r < n; ++r) hyq[r] = (long long)nearbyint(ldexp(label[r], shift));   // ties to even
  CallMem tmp;
  cudaStream_t st;
  CK0(tmp.stream(&st));
  double* dx = nullptr;
  long long* dyq = nullptr;
  int* dar = nullptr;
  CK0(tmp.device(&dx, (size_t)n * n_feat));
  CK0(tmp.device(&dyq, (size_t)n));
  CK0(tmp.device(&dar, (size_t)n_feat));
  rf_ms(t0);
  CK0(cudaMemcpyAsync(dx, x, sizeof(double) * (size_t)n * n_feat, cudaMemcpyHostToDevice, st));
  CK0(cudaMemcpyAsync(dyq, hyq.data(), 8 * (size_t)n, cudaMemcpyHostToDevice, st));
  CK0(cudaMemcpyAsync(dar, reg.arity.data(), 4 * (size_t)n_feat, cudaMemcpyHostToDevice, st));
  CK0(cudaStreamSynchronize(st));
  tm.h2d = rf_ms(t0);
  reg.dyq = dyq, reg.darity = dar;
  return rf_fit(p, dx, nullptr, n, n_feat, sm, tmp, st, t0, out, &reg);
}

int pio_rf_forest_reg_size(const pio_rf_forest* f, int64_t* n_cat_ids) {
  if (!f) return fail(nullptr, PIO_ALS_ERR_ARG, "null forest");
  if (!f->regression) return fail(nullptr, PIO_ALS_ERR_ARG, "not a regression forest");
  if (n_cat_ids) *n_cat_ids = (int64_t)f->cat_ids.size();
  return PIO_ALS_OK;
}

int pio_rf_forest_reg_get(const pio_rf_forest* f, double* value, int64_t* cat_off, int32_t* cat_ids) {
  if (!f) return fail(nullptr, PIO_ALS_ERR_ARG, "null forest");
  if (!f->regression) return fail(nullptr, PIO_ALS_ERR_ARG, "not a regression forest");
  auto put = [](auto* dst, const auto& v) {
    if (dst && !v.empty()) memcpy(dst, v.data(), v.size() * sizeof(v[0]));
  };
  put(value, f->value);
  put(cat_off, f->cat_off);
  put(cat_ids, f->cat_ids);
  return PIO_ALS_OK;
}

int pio_rf_predict_regression(int device, int32_t n_trees, const int32_t* tree_off, int64_t n_nodes,
                              const int32_t* feature, const double* threshold, const int32_t* left,
                              const int32_t* right, const double* value, const int64_t* cat_off,
                              const int32_t* cat_ids, const double* x, int64_t n, int32_t n_feat, double* out) {
  if (!out || !value || !cat_off || n < 0 || (n > 0 && !x) || n_nodes < 1 || n_nodes >= (1ll << 31))
    return fail(nullptr, PIO_ALS_ERR_ARG, "bad pio_rf_predict_regression arguments");
  const std::vector<int32_t> zero((size_t)n_nodes, 0);   // rf_check_flat's class check, with one class
  const RfFlat fl{n_trees, tree_off, n_nodes, feature, threshold, left, right, zero.data(), 1};
  EVF(rf_check_flat(fl, n_feat));
  const int64_t nc = cat_off[n_nodes];
  if (cat_off[0] != 0 || nc < 0 || (nc > 0 && !cat_ids)) return fail(nullptr, PIO_ALS_ERR_ARG, "bad category offsets");
  for (int64_t i = 0; i < n_nodes; ++i) {
    if (cat_off[i + 1] < cat_off[i] || cat_off[i + 1] > nc)
      return fail(nullptr, PIO_ALS_ERR_ARG, "bad category offsets at node %lld", (long long)i);
    if (cat_off[i + 1] > cat_off[i] && feature[i] < 0)
      return fail(nullptr, PIO_ALS_ERR_ARG, "leaf %lld has categories", (long long)i);
    for (int64_t k = cat_off[i]; k < cat_off[i + 1]; ++k)
      if (cat_ids[k] < 0 || (k > cat_off[i] && cat_ids[k] <= cat_ids[k - 1]))
        return fail(nullptr, PIO_ALS_ERR_ARG, "categories of node %lld are not ascending non-negative ids", (long long)i);
  }
  if (n == 0) return PIO_ALS_OK;
  CK0(cudaSetDevice(device));
  CallMem tmp;
  cudaStream_t st;
  CK0(tmp.stream(&st));
  const int64_t nn = n_nodes;
  int *dto = nullptr, *df = nullptr, *dl = nullptr, *dr = nullptr, *dci = nullptr;
  double *dt = nullptr, *dv = nullptr, *dx = nullptr, *dout = nullptr;
  long long* dco = nullptr;
  CK0(tmp.device(&dto, (size_t)n_trees));
  CK0(tmp.device(&df, (size_t)nn));
  CK0(tmp.device(&dl, (size_t)nn));
  CK0(tmp.device(&dr, (size_t)nn));
  CK0(tmp.device(&dt, (size_t)nn));
  CK0(tmp.device(&dv, (size_t)nn));
  CK0(tmp.device(&dco, (size_t)nn + 1));
  CK0(tmp.device(&dci, (size_t)std::max<int64_t>(1, nc)));
  CK0(tmp.device(&dx, (size_t)n * n_feat));
  CK0(tmp.device(&dout, (size_t)n));
  CK0(cudaMemcpyAsync(dto, tree_off, 4 * (size_t)n_trees, cudaMemcpyHostToDevice, st));
  CK0(cudaMemcpyAsync(df, feature, 4 * (size_t)nn, cudaMemcpyHostToDevice, st));
  CK0(cudaMemcpyAsync(dl, left, 4 * (size_t)nn, cudaMemcpyHostToDevice, st));
  CK0(cudaMemcpyAsync(dr, right, 4 * (size_t)nn, cudaMemcpyHostToDevice, st));
  CK0(cudaMemcpyAsync(dt, threshold, 8 * (size_t)nn, cudaMemcpyHostToDevice, st));
  CK0(cudaMemcpyAsync(dv, value, 8 * (size_t)nn, cudaMemcpyHostToDevice, st));
  CK0(cudaMemcpyAsync(dco, cat_off, 8 * ((size_t)nn + 1), cudaMemcpyHostToDevice, st));
  if (nc > 0) CK0(cudaMemcpyAsync(dci, cat_ids, 4 * (size_t)nc, cudaMemcpyHostToDevice, st));
  CK0(cudaMemcpyAsync(dx, x, 8 * (size_t)n * n_feat, cudaMemcpyHostToDevice, st));
  rf::predict_reg_kernel<<<nblk(n, 128), 128, 0, st>>>(dto, n_trees, df, dt, dl, dr, dv, dco, dci, dx, n, n_feat, dout);
  CK0(cudaGetLastError());
  CK0(cudaMemcpyAsync(out, dout, 8 * (size_t)n, cudaMemcpyDeviceToHost, st));
  CK0(cudaStreamSynchronize(st));
  return PIO_ALS_OK;
}

int pio_lead_sessions(int device, const int32_t* session, const uint8_t* is_buy, const int64_t* t_ms, int64_t n,
                      int32_t n_sessions, int64_t* landing, uint8_t* buy) {
  if (n < 0 || n_sessions < 0 || (n > 0 && (!session || !is_buy || !t_ms)) || (n_sessions > 0 && (!landing || !buy)))
    return fail(nullptr, PIO_ALS_ERR_ARG, "bad pio_lead_sessions arguments");
  for (int64_t r = 0; r < n; ++r)
    if (session[r] < 0 || session[r] >= n_sessions)
      return fail(nullptr, PIO_ALS_ERR_ARG, "event %lld has session %d of %d", (long long)r, session[r], n_sessions);
  if (n_sessions == 0) return PIO_ALS_OK;
  CK0(cudaSetDevice(device));
  CallMem tmp;
  cudaStream_t st;
  CK0(tmp.stream(&st));
  int* ds = nullptr;
  uint8_t *db = nullptr, *dbuy = nullptr;
  long long *dt = nullptr, *dland = nullptr;
  unsigned long long* dmin = nullptr;
  CK0(tmp.device(&ds, (size_t)std::max<int64_t>(n, 1)));
  CK0(tmp.device(&db, (size_t)std::max<int64_t>(n, 1)));
  CK0(tmp.device(&dt, (size_t)std::max<int64_t>(n, 1)));
  CK0(tmp.device(&dmin, (size_t)n_sessions));
  CK0(tmp.device(&dland, (size_t)n_sessions));
  CK0(tmp.device(&dbuy, (size_t)n_sessions));
  if (n > 0) {
    CK0(cudaMemcpyAsync(ds, session, 4 * (size_t)n, cudaMemcpyHostToDevice, st));
    CK0(cudaMemcpyAsync(db, is_buy, (size_t)n, cudaMemcpyHostToDevice, st));
    CK0(cudaMemcpyAsync(dt, t_ms, 8 * (size_t)n, cudaMemcpyHostToDevice, st));
  }
  CK0(cudaMemsetAsync(dmin, 0xff, 8 * (size_t)n_sessions, st));
  CK0(cudaMemsetAsync(dland, 0xff, 8 * (size_t)n_sessions, st));          // -1: no view
  CK0(cudaMemsetAsync(dbuy, 0, (size_t)n_sessions, st));
  if (n > 0) {
    lead::landing_time_kernel<<<nblk(n, 256), 256, 0, st>>>(ds, db, dt, n, dmin);
    lead::landing_pick_kernel<<<nblk(n, 256), 256, 0, st>>>(ds, db, dt, n, dmin, dland);
    lead::buy_flag_kernel<<<nblk(n, 256), 256, 0, st>>>(ds, db, dt, n, dmin, dland, dbuy);
    CK0(cudaGetLastError());
  }
  CK0(cudaMemcpyAsync(landing, dland, 8 * (size_t)n_sessions, cudaMemcpyDeviceToHost, st));
  CK0(cudaMemcpyAsync(buy, dbuy, (size_t)n_sessions, cudaMemcpyDeviceToHost, st));
  CK0(cudaStreamSynchronize(st));
  return PIO_ALS_OK;
}

/* debug only (not in pio_als.h): where the last pio_rf_train on this thread spent its time, wall ms of phases that each
 * end in a stream synchronise: out[0] host-to-device copy, [1] split search, [2] binning, [3] histograms, [4] split
 * selection, [5] node update, [6] levels, [7] tree groups, [8 + l] histograms of level l, [39 + l] selection of level l
 * (l < 31).  Used by tools/forest_bench.py. */
__attribute__((visibility("default"))) int pio_rf_debug_timing(double out[70]) {
  if (!out) return PIO_ALS_ERR_ARG;
  const RfTiming& t = g_rf_timing;
  out[0] = t.h2d, out[1] = t.split, out[2] = t.bin, out[3] = t.hist, out[4] = t.sel, out[5] = t.upd;
  out[6] = t.levels, out[7] = t.groups;
  for (int l = 0; l <= RF_MAX_DEPTH; ++l) out[8 + l] = t.hist_l[l], out[39 + l] = t.sel_l[l];
  return PIO_ALS_OK;
}

/* debug only (not in pio_als.h): which paths the last pio_rf_train on this thread took: out[0] bin code bytes (1 or 2),
 * [1] thresholds staged in shared memory (0 / 1), [2] shared-memory hist_kernel launches, [3] global hist_kernel
 * launches, [4] most histogram chunks in one level, [5] most shared-memory passes in one chunk, [6] levels, [7] tree
 * groups.  Used by tests/test_gpu_forest_bounds.py. */
__attribute__((visibility("default"))) int pio_rf_debug_paths(int64_t out[8]) {
  if (!out) return PIO_ALS_ERR_ARG;
  const RfTiming& t = g_rf_timing;
  out[0] = t.bin_bytes, out[1] = t.staged, out[2] = t.smem_launches, out[3] = t.global_launches;
  out[4] = t.max_chunks, out[5] = t.max_passes, out[6] = t.levels, out[7] = t.groups;
  return PIO_ALS_OK;
}

}  // extern "C"

// ---- k-fold evaluation (eval_folds.cuh; DESIGN.md 4.11) ----------------------------------------------------------------
struct pio_eval_folds {
  struct Fold {
    int n_users = 0, n_items = 0, nq = 0;
    long long n_train = 0, n_test = 0;
    int *uloc = nullptr, *iloc = nullptr;   // global -> fold-local (-1: not in the training set)
    int *ul2g = nullptr, *il2g = nullptr;   // fold-local -> global
    int *q2g = nullptr, *qtrain = nullptr;  // per query: global user, fold-local training user or -1
    int *qptr = nullptr;                    // [nq + 1] test ratings of query q, sorted by global item: raw[qptr[q] ..)
    double* raw = nullptr;
    int *dptr = nullptr, *ditem = nullptr;  // [nq + 1] distinct test items of query q: ditem / dmax[dptr[q] ..)
    double* dmax = nullptr;
  };
  struct Result {
    int fold = 0, nq = 0, num = 0;
    int *items = nullptr, *count = nullptr;
  };
  int device = 0, k_fold = 1, n_users = 0, n_items = 0;   // n_users / n_items: global index ranges
  long long n = 0;
  cudaStream_t st = nullptr;
  int *gu = nullptr, *gi = nullptr;
  double* r = nullptr;
  std::vector<Fold> folds;
  std::map<int32_t, Result> results;
  int32_t next_result = 0;
  std::vector<void*> mem;   // the object's device memory, results excepted
};

namespace pio {

__global__ void evf_fill_kernel(int* __restrict__ p, long long n, int v) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) p[i] = v;
}

template <class T>
static int evf_alloc(pio_eval_folds* ef, T** p, size_t n) {
  CK0(cudaMalloc((void**)p, (n ? n : 1) * sizeof(T)));
  ef->mem.push_back((void*)*p);
  return PIO_ALS_OK;
}

static int evf_read(const uint32_t* d, cudaStream_t st, uint32_t* out) {
  CK0(cudaMemcpyAsync(out, d, sizeof(uint32_t), cudaMemcpyDeviceToHost, st));
  CK0(cudaStreamSynchronize(st));
  return PIO_ALS_OK;
}

// Fold f's maps of one side (global ids 0 .. n_ids): loc (global -> local), l2g and their count.  flag: n + 1 entries.
static int evf_side(pio_eval_folds* ef, int f, const int* e1, const int* e2, int n_ids, uint32_t* flag, int** loc,
                    int** l2g, int* count) {
  const cudaStream_t st = ef->st;
  const long long n = ef->n;
  CK0(cudaMemsetAsync(flag, 0, sizeof(uint32_t) * (size_t)(n + 1), st));
  evf::train_flag_kernel<<<nblk(n_ids, 256), 256, 0, st>>>(e1, e2, n_ids, ef->k_fold, f, flag);
  CK0(scan_exclusive_u32(flag, flag, (size_t)n + 1, st, nullptr));
  uint32_t total = 0;
  EVF(evf_read(flag + n, st, &total));
  *count = (int)total;
  EVF(evf_alloc(ef, loc, (size_t)n_ids));
  EVF(evf_alloc(ef, l2g, (size_t)total));
  evf::train_index_kernel<<<nblk(n_ids, 256), 256, 0, st>>>(e1, e2, n_ids, ef->k_fold, f, flag, *loc, *l2g);
  CK0(cudaGetLastError());
  return PIO_ALS_OK;
}

// Uploads the ratings and builds every fold: maps, queries and sorted test lists.
static int evf_build(pio_eval_folds* ef, const int32_t* user, const int32_t* item, const double* rating) {
  const cudaStream_t st = ef->st;
  const long long n = ef->n;
  const int K = ef->k_fold;
  EVF(evf_alloc(ef, &ef->gu, (size_t)n));
  EVF(evf_alloc(ef, &ef->gi, (size_t)n));
  EVF(evf_alloc(ef, &ef->r, (size_t)n));
  CK0(cudaMemcpyAsync(ef->gu, user, sizeof(int) * (size_t)n, cudaMemcpyHostToDevice, st));
  CK0(cudaMemcpyAsync(ef->gi, item, sizeof(int) * (size_t)n, cudaMemcpyHostToDevice, st));
  CK0(cudaMemcpyAsync(ef->r, rating, sizeof(double) * (size_t)n, cudaMemcpyHostToDevice, st));
  CallMem tmp(st);
  int *ue1, *ue2, *ie1, *ie2, *qfirst;
  uint32_t *uflag, *iflag, *qflag, *dflag;
  const long long m_max = (n + K - 1) / K;   // fold 0 has the most test ratings
  for (int** p : {&ue1, &ue2, &qfirst}) CK0(tmp.device(p, (size_t)ef->n_users));
  for (int** p : {&ie1, &ie2}) CK0(tmp.device(p, (size_t)ef->n_items));
  for (uint32_t** p : {&uflag, &iflag}) CK0(tmp.device(p, (size_t)n + 1));
  for (uint32_t** p : {&qflag, &dflag}) CK0(tmp.device(p, (size_t)m_max + 1));
  SortBufs sb;
  for (int i : {0, 1}) {
    CK0(tmp.device(&sb.k[i], (size_t)m_max));
    CK0(tmp.device(&sb.v[i], (size_t)m_max));
  }
  struct { const int* g; int* e1; int* e2; int n_ids; } sides[2] = {{ef->gu, ue1, ue2, ef->n_users},
                                                                    {ef->gi, ie1, ie2, ef->n_items}};
  for (auto& s : sides) {
    for (int* p : {s.e1, s.e2}) evf_fill_kernel<<<nblk(s.n_ids, 256), 256, 0, st>>>(p, s.n_ids, evf::NONE);
    evf::first_pos_kernel<<<nblk(n, 256), 256, 0, st>>>(s.g, n, s.e1);
    evf::second_pos_kernel<<<nblk(n, 256), 256, 0, st>>>(s.g, n, K, s.e1, s.e2);
  }
  CK0(cudaGetLastError());
  const int ibits = ceil_log2((uint64_t)ef->n_items);
  ef->folds.resize(K);
  for (int f = 0; f < K; ++f) {
    pio_eval_folds::Fold& F = ef->folds[f];
    const long long m = (n + K - 1 - f) / K;
    F.n_test = m;
    F.n_train = n - m;
    EVF(evf_side(ef, f, ue1, ue2, ef->n_users, uflag, &F.uloc, &F.ul2g, &F.n_users));
    EVF(evf_side(ef, f, ie1, ie2, ef->n_items, iflag, &F.iloc, &F.il2g, &F.n_items));
    if (m == 0) continue;
    evf_fill_kernel<<<nblk(ef->n_users, 256), 256, 0, st>>>(qfirst, ef->n_users, evf::NONE);
    evf::query_first_kernel<<<nblk(m, 256), 256, 0, st>>>(ef->gu, K, f, m, qfirst);
    evf::query_flag_kernel<<<nblk(m + 1, 256), 256, 0, st>>>(ef->gu, K, f, m, qfirst, qflag);
    CK0(scan_exclusive_u32(qflag, qflag, (size_t)m + 1, st, nullptr));
    uint32_t nq = 0;
    EVF(evf_read(qflag + m, st, &nq));
    F.nq = (int)nq;
    EVF(evf_alloc(ef, &F.q2g, nq));
    EVF(evf_alloc(ef, &F.qtrain, nq));
    EVF(evf_alloc(ef, &F.qptr, (size_t)nq + 1));
    EVF(evf_alloc(ef, &F.dptr, (size_t)nq + 1));
    EVF(evf_alloc(ef, &F.raw, (size_t)m));
    sb.live = 0;
    evf::query_index_kernel<<<nblk(m, 256), 256, 0, st>>>(ef->gu, ef->gi, K, f, m, qfirst, qflag, F.uloc, ibits, F.q2g,
                                                         F.qtrain, sb.keys(), sb.vals());
    CK0(radix_sort_pairs(sb, (size_t)m, ceil_log2(nq) + ibits, st, nullptr));
    evf::test_slots_kernel<<<nblk(m + 1, 256), 256, 0, st>>>(sb.keys(), sb.vals(), m, K, f, ef->r, ibits, (int)nq, F.raw,
                                                            F.qptr, dflag);
    CK0(scan_exclusive_u32(dflag, dflag, (size_t)m + 1, st, nullptr));
    uint32_t nd = 0;
    EVF(evf_read(dflag + m, st, &nd));
    EVF(evf_alloc(ef, &F.ditem, nd));
    EVF(evf_alloc(ef, &F.dmax, nd));
    evf::test_distinct_kernel<<<nblk(m, 256), 256, 0, st>>>(sb.keys(), m, F.raw, dflag, (1ull << ibits) - 1ull, F.ditem,
                                                           F.dmax);
    evf::test_dptr_kernel<<<nblk((long long)nq + 1, 256), 256, 0, st>>>(F.qptr, dflag, (int)nq, F.dptr);
    CK0(cudaGetLastError());
  }
  CK0(cudaStreamSynchronize(st));
  return PIO_ALS_OK;
}

static int evf_fold(const pio_eval_folds* ef, int32_t fold, const char* what) {
  if (!ef) return fail(nullptr, PIO_ALS_ERR_ARG, "%s: null object", what);
  if (fold < 0 || fold >= ef->k_fold)
    return fail(nullptr, PIO_ALS_ERR_ARG, "%s: fold %d outside 0..%d", what, fold, ef->k_fold - 1);
  return PIO_ALS_OK;
}

}  // namespace pio

extern "C" {

int pio_eval_folds_create(int device, const int32_t* user, const int32_t* item, const double* rating, int64_t n,
                          int32_t k_fold, pio_eval_folds** out) {
  if (!out) return fail(nullptr, PIO_ALS_ERR_ARG, "bad pio_eval_folds_create arguments");
  *out = nullptr;
  if (!user || !item || !rating || n < 1 || k_fold < 1)
    return fail(nullptr, PIO_ALS_ERR_ARG, "bad pio_eval_folds_create arguments (n >= 1 and k_fold >= 1)");
  if (n >= (1ll << 31)) return fail(nullptr, PIO_ALS_ERR_ARG, "n must be < 2^31");
  int32_t mu = -1, mi = -1;
  for (int64_t e = 0; e < n; ++e) {
    if (user[e] < 0 || item[e] < 0)
      return fail(nullptr, PIO_ALS_ERR_ARG, "rating %lld: negative user or item index", (long long)e);
    mu = std::max(mu, user[e]);
    mi = std::max(mi, item[e]);
  }
  CK0(cudaSetDevice(device));
  auto* ef = new pio_eval_folds;
  ef->device = device;
  ef->k_fold = k_fold;
  ef->n = n;
  ef->n_users = mu + 1;
  ef->n_items = mi + 1;
  const cudaError_t e = cudaStreamCreateWithFlags(&ef->st, cudaStreamNonBlocking);
  if (e != cudaSuccess) {
    delete ef;
    return fail(nullptr, PIO_ALS_ERR_CUDA, "cudaStreamCreate: %s", cudaGetErrorString(e));
  }
  const int rc = evf_build(ef, user, item, rating);
  if (rc != PIO_ALS_OK) {
    pio_eval_folds_destroy(ef);
    return rc;
  }
  *out = ef;
  return PIO_ALS_OK;
}

int pio_eval_folds_sizes(const pio_eval_folds* ef, int32_t fold, int64_t out[4]) {
  EVF(evf_fold(ef, fold, "pio_eval_folds_sizes"));
  if (!out) return fail(nullptr, PIO_ALS_ERR_ARG, "pio_eval_folds_sizes: null out");
  const pio_eval_folds::Fold& F = ef->folds[fold];
  out[0] = F.n_users, out[1] = F.n_items, out[2] = F.n_train, out[3] = F.nq;
  return PIO_ALS_OK;
}

int pio_eval_folds_maps(const pio_eval_folds* ef, int32_t fold, int32_t* user, int32_t* item, int32_t* query_user,
                        int32_t* query_train_user) {
  EVF(evf_fold(ef, fold, "pio_eval_folds_maps"));
  CK0(cudaSetDevice(ef->device));
  const pio_eval_folds::Fold& F = ef->folds[fold];
  const struct { int32_t* to; const int* from; int count; } jobs[4] = {
      {user, F.ul2g, F.n_users}, {item, F.il2g, F.n_items}, {query_user, F.q2g, F.nq}, {query_train_user, F.qtrain, F.nq}};
  for (const auto& j : jobs)
    if (j.to && j.count) CK0(cudaMemcpyAsync(j.to, j.from, sizeof(int32_t) * (size_t)j.count, cudaMemcpyDeviceToHost, ef->st));
  CK0(cudaStreamSynchronize(ef->st));
  return PIO_ALS_OK;
}

int pio_eval_folds_set_ratings(pio_eval_folds* ef, int32_t fold, pio_als_handle* h) {
  EVF(evf_fold(ef, fold, "pio_eval_folds_set_ratings"));
  const pio_eval_folds::Fold& F = ef->folds[fold];
  if (!h) return fail(nullptr, PIO_ALS_ERR_ARG, "pio_eval_folds_set_ratings: null handle");
  if (h->cfg.device != ef->device || h->cfg.world_size != 1 || h->cfg.n_users != F.n_users || h->cfg.n_items != F.n_items)
    return fail(nullptr, PIO_ALS_ERR_ARG, "pio_eval_folds_set_ratings: the handle (device %d, world_size %d, %d users, "
                "%d items) does not match fold %d (device %d, %d users, %d items)", h->cfg.device, h->cfg.world_size,
                h->cfg.n_users, h->cfg.n_items, fold, ef->device, F.n_users, F.n_items);
  if (F.n_train == 0) return fail(nullptr, PIO_ALS_ERR_ARG, "fold %d has no training ratings", fold);
  CK0(cudaSetDevice(ef->device));
  int rc;
  {
    CallMem tmp(ef->st);
    int *du = nullptr, *di = nullptr;
    float* dv = nullptr;
    CK0(tmp.device(&du, (size_t)F.n_train));
    CK0(tmp.device(&di, (size_t)F.n_train));
    CK0(tmp.device(&dv, (size_t)F.n_train));
    evf::train_coo_kernel<<<nblk(ef->n, 256), 256, 0, ef->st>>>(ef->gu, ef->gi, ef->r, ef->n, ef->k_fold, fold, F.uloc,
                                                               F.iloc, du, di, dv);
    CK0(cudaGetLastError());
    CK0(cudaStreamSynchronize(ef->st));
    rc = pio_als_set_ratings_coo_device(h, du, di, dv, F.n_train, PIO_ALS_DEDUP_NONE, nullptr);
  }
  if (rc != PIO_ALS_OK) return fail(nullptr, rc, "%s", h->err.c_str());
  return PIO_ALS_OK;
}

int pio_eval_folds_result_add(pio_eval_folds* ef, int32_t fold, const int32_t* items, const int32_t* count,
                              int32_t n_queries, int32_t num, int32_t* out_result) {
  EVF(evf_fold(ef, fold, "pio_eval_folds_result_add"));
  const pio_eval_folds::Fold& F = ef->folds[fold];
  if (!out_result || num < 1 || n_queries != F.nq || (n_queries > 0 && (!items || !count)))
    return fail(nullptr, PIO_ALS_ERR_ARG, "bad pio_eval_folds_result_add arguments (fold %d has %d queries)", fold, F.nq);
  for (int32_t q = 0; q < n_queries; ++q) {
    if (count[q] < 0 || count[q] > num)
      return fail(nullptr, PIO_ALS_ERR_ARG, "query %d: count %d outside 0..%d", q, count[q], num);
    for (int32_t j = 0; j < count[q]; ++j) {
      const int32_t it = items[(int64_t)q * num + j];
      if (it < 0 || it >= F.n_items)
        return fail(nullptr, PIO_ALS_ERR_ARG, "query %d: item %d outside the fold's %d items", q, it, F.n_items);
    }
  }
  CK0(cudaSetDevice(ef->device));
  pio_eval_folds::Result R;
  R.fold = fold, R.nq = n_queries, R.num = num;
  cudaError_t e = cudaMalloc((void**)&R.items, sizeof(int32_t) * ((size_t)n_queries * num + 1));
  if (e == cudaSuccess) e = cudaMalloc((void**)&R.count, sizeof(int32_t) * ((size_t)n_queries + 1));
  if (e == cudaSuccess && n_queries > 0)
    e = cudaMemcpyAsync(R.items, items, sizeof(int32_t) * (size_t)n_queries * num, cudaMemcpyHostToDevice, ef->st);
  if (e == cudaSuccess && n_queries > 0)
    e = cudaMemcpyAsync(R.count, count, sizeof(int32_t) * (size_t)n_queries, cudaMemcpyHostToDevice, ef->st);
  if (e == cudaSuccess) e = cudaStreamSynchronize(ef->st);
  if (e != cudaSuccess) {
    cudaFree(R.items);
    cudaFree(R.count);
    return fail(nullptr, PIO_ALS_ERR_CUDA, "pio_eval_folds_result_add: %s", cudaGetErrorString(e));
  }
  *out_result = ef->next_result++;
  ef->results[*out_result] = R;
  return PIO_ALS_OK;
}

int pio_eval_folds_result_free(pio_eval_folds* ef, int32_t result) {
  if (!ef) return fail(nullptr, PIO_ALS_ERR_ARG, "pio_eval_folds_result_free: null object");
  auto it = ef->results.find(result);
  if (it == ef->results.end()) return fail(nullptr, PIO_ALS_ERR_ARG, "no result %d", result);
  cudaSetDevice(ef->device);
  cudaFree(it->second.items);
  cudaFree(it->second.count);
  ef->results.erase(it);
  return PIO_ALS_OK;
}

int pio_eval_folds_rank_counts(pio_eval_folds* ef, int32_t result, int32_t k, double threshold, int32_t* hits,
                               int32_t* npos, int32_t* nraw) {
  if (!ef) return fail(nullptr, PIO_ALS_ERR_ARG, "pio_eval_folds_rank_counts: null object");
  auto it = ef->results.find(result);
  if (it == ef->results.end()) return fail(nullptr, PIO_ALS_ERR_ARG, "no result %d", result);
  const pio_eval_folds::Result& R = it->second;
  if (k < 1 || (R.nq > 0 && (!hits || !npos || !nraw)))
    return fail(nullptr, PIO_ALS_ERR_ARG, "bad pio_eval_folds_rank_counts arguments (k >= 1)");
  if (R.nq == 0) return PIO_ALS_OK;
  CK0(cudaSetDevice(ef->device));
  const pio_eval_folds::Fold& F = ef->folds[R.fold];
  const cudaStream_t st = ef->st;
  CallMem tmp(st);
  int* d = nullptr;
  CK0(tmp.device(&d, 3 * (size_t)R.nq));
  evf::rank_counts_kernel<<<nblk(R.nq, evf::RC_WARPS), 32 * evf::RC_WARPS, 0, st>>>(
      R.items, R.count, R.num, R.nq, k, threshold, F.il2g, F.qptr, F.raw, F.dptr, F.ditem, F.dmax, d, d + R.nq,
      d + 2 * (size_t)R.nq);
  CK0(cudaGetLastError());
  int32_t* outs[3] = {hits, npos, nraw};
  for (int j = 0; j < 3; ++j)
    CK0(cudaMemcpyAsync(outs[j], d + (size_t)j * R.nq, sizeof(int32_t) * (size_t)R.nq, cudaMemcpyDeviceToHost, st));
  CK0(cudaStreamSynchronize(st));
  return PIO_ALS_OK;
}

int pio_eval_folds_destroy(pio_eval_folds* ef) {
  if (!ef) return PIO_ALS_OK;
  cudaSetDevice(ef->device);
  if (ef->st) cudaStreamSynchronize(ef->st);
  for (auto& kv : ef->results) {
    cudaFree(kv.second.items);
    cudaFree(kv.second.count);
  }
  for (void* p : ef->mem) cudaFree(p);
  if (ef->st) cudaStreamDestroy(ef->st);
  delete ef;
  return PIO_ALS_OK;
}

}  // extern "C"

// ---- k-fold evaluation of the classification template (cls_folds.cuh; DESIGN.md 4.12) -----------------------------------
struct pio_cls_folds {
  struct Result {
    int fold = 0;
    long long m = 0;
    double* pred = nullptr;   // [m] predicted label of every test row of the fold
  };
  int device = 0, k = 1, F = 1, C = 0;   // C: distinct labels of all rows
  long long n = 0;
  cudaStream_t st = nullptr;
  double *label = nullptr, *x = nullptr;
  int* cls = nullptr;                    // [n] index of the row's label among the distinct labels
  std::vector<double> classes;           // the distinct labels, ascending
  std::vector<int> fmin, fmax;           // per class: smallest / largest fold holding one of its rows
  std::map<int32_t, Result> results;
  int32_t next_result = 0;
  std::vector<void*> mem;                // the object's device memory, results excepted
};

namespace pio {

static long long clf_n_test(const pio_cls_folds* cf, int f) { return (cf->n + cf->k - 1 - f) / cf->k; }

static int clf_fold(const pio_cls_folds* cf, int32_t fold, const char* what) {
  if (!cf) return fail(nullptr, PIO_ALS_ERR_ARG, "%s: null object", what);
  if (fold < 0 || fold >= cf->k)
    return fail(nullptr, PIO_ALS_ERR_ARG, "%s: fold %d outside 0..%d", what, fold, cf->k - 1);
  return PIO_ALS_OK;
}

// fold f's training classes: lmap[c] = index of class c among them (-1: every row of c tests in fold f); returns their
// number
static int clf_train_classes(const pio_cls_folds* cf, int f, std::vector<int>* lmap, std::vector<double>* labels) {
  int nc = 0;
  if (lmap) lmap->assign(cf->C, -1);
  for (int c = 0; c < cf->C; ++c) {
    if (cf->fmin[c] == f && cf->fmax[c] == f) continue;
    if (lmap) (*lmap)[c] = nc;
    if (labels) labels->push_back(cf->classes[c]);
    ++nc;
  }
  return nc;
}

// grid of the grid-stride kernels: one thread per row up to 16 blocks per SM of an H100
static unsigned clf_grid(long long n) { return (unsigned)std::max<long long>(1, std::min<long long>(nblk(n, clf::THREADS), 132 * 16)); }

// the first training row of fold f failing check `mode` (cls_folds.cuh): its row, or -1 (none)
static int clf_first_bad(pio_cls_folds* cf, int f, int mode, int num_classes, CallMem& tmp, long long* row) {
  unsigned long long* d = nullptr;
  CK0(tmp.device(&d, 1));
  const unsigned long long none = (unsigned long long)cf->n;
  CK0(cudaMemcpyAsync(d, &none, 8, cudaMemcpyHostToDevice, cf->st));
  clf::first_bad_kernel<<<clf_grid(cf->n), clf::THREADS, 0, cf->st>>>(cf->label, cf->x, cf->n, cf->F, cf->k, f, mode,
                                                                      num_classes, d);
  CK0(cudaGetLastError());
  unsigned long long e = 0;
  CK0(cudaMemcpyAsync(&e, d, 8, cudaMemcpyDeviceToHost, cf->st));
  CK0(cudaStreamSynchronize(cf->st));
  *row = e == none ? -1 : (long long)e;
  return PIO_ALS_OK;
}

// label and features of row e, to the host
static int clf_row(const pio_cls_folds* cf, long long e, double* label, std::vector<double>* xr) {
  xr->resize(cf->F);
  CK0(cudaMemcpyAsync(label, cf->label + e, 8, cudaMemcpyDeviceToHost, cf->st));
  CK0(cudaMemcpyAsync(xr->data(), cf->x + e * cf->F, 8 * (size_t)cf->F, cudaMemcpyDeviceToHost, cf->st));
  CK0(cudaStreamSynchronize(cf->st));
  return PIO_ALS_OK;
}

static long long clf_train_pos(const pio_cls_folds* cf, long long e, int f) { return e - (e + cf->k - 1 - f) / cf->k; }

// Uploads the rows and encodes the labels: distinct labels, each row's class, each class's fold range.
static int clf_build(pio_cls_folds* cf, const double* label, const double* x) {
  const cudaStream_t st = cf->st;
  const long long n = cf->n;
  for (double** p : {&cf->label, &cf->x}) {
    const size_t cnt = p == &cf->label ? (size_t)n : (size_t)n * cf->F;
    CK0(cudaMalloc((void**)p, 8 * cnt));
    cf->mem.push_back(*p);
  }
  CK0(cudaMalloc((void**)&cf->cls, 4 * (size_t)n));
  cf->mem.push_back(cf->cls);
  CK0(cudaMemcpyAsync(cf->label, label, 8 * (size_t)n, cudaMemcpyHostToDevice, st));
  CK0(cudaMemcpyAsync(cf->x, x, 8 * (size_t)n * cf->F, cudaMemcpyHostToDevice, st));
  CallMem tmp(st);
  SortBufs sb;
  uint32_t *head = nullptr, *pos = nullptr;
  uint64_t* ukey = nullptr;
  for (int i : {0, 1}) {
    CK0(tmp.device(&sb.k[i], (size_t)n));
    CK0(tmp.device(&sb.v[i], (size_t)n));
  }
  CK0(tmp.device(&head, (size_t)n));
  CK0(tmp.device(&pos, (size_t)n));
  CK0(tmp.device(&ukey, (size_t)n));
  clf::label_keys_kernel<<<nblk(n, 256), 256, 0, st>>>(cf->label, n, sb.keys(), sb.vals());
  CK0(radix_sort_pairs(sb, (size_t)n, 64, st, nullptr));
  rf::run_head_kernel<<<nblk(n, 256), 256, 0, st>>>(sb.keys(), n, head);
  CK0(scan_exclusive_u32(head, pos, (size_t)n, st, nullptr));
  clf::class_index_kernel<<<nblk(n, 256), 256, 0, st>>>(sb.keys(), sb.vals(), head, pos, n, cf->cls, ukey);
  CK0(cudaGetLastError());
  uint32_t lh = 0, lp = 0;
  CK0(cudaMemcpyAsync(&lh, head + n - 1, 4, cudaMemcpyDeviceToHost, st));
  CK0(cudaMemcpyAsync(&lp, pos + n - 1, 4, cudaMemcpyDeviceToHost, st));
  CK0(cudaStreamSynchronize(st));
  cf->C = (int)(lp + lh);
  std::vector<uint64_t> hk(cf->C);
  CK0(cudaMemcpyAsync(hk.data(), ukey, 8 * (size_t)cf->C, cudaMemcpyDeviceToHost, st));
  int *dmin = nullptr, *dmax = nullptr;
  CK0(tmp.device(&dmin, (size_t)cf->C));
  CK0(tmp.device(&dmax, (size_t)cf->C));
  cf->fmin.assign(cf->C, cf->k);
  cf->fmax.assign(cf->C, -1);
  CK0(cudaMemcpyAsync(dmin, cf->fmin.data(), 4 * (size_t)cf->C, cudaMemcpyHostToDevice, st));
  CK0(cudaMemcpyAsync(dmax, cf->fmax.data(), 4 * (size_t)cf->C, cudaMemcpyHostToDevice, st));
  clf::class_folds_kernel<<<clf_grid(n), clf::THREADS, 0, st>>>(cf->cls, n, cf->k, dmin, dmax);
  CK0(cudaGetLastError());
  CK0(cudaMemcpyAsync(cf->fmin.data(), dmin, 4 * (size_t)cf->C, cudaMemcpyDeviceToHost, st));
  CK0(cudaMemcpyAsync(cf->fmax.data(), dmax, 4 * (size_t)cf->C, cudaMemcpyDeviceToHost, st));
  CK0(cudaStreamSynchronize(st));
  cf->classes.resize(cf->C);
  for (int c = 0; c < cf->C; ++c) {
    const uint64_t b = (hk[c] >> 63) ? (hk[c] & ~(1ull << 63)) : ~hk[c];
    memcpy(&cf->classes[c], &b, 8);
    if (!isfinite(cf->classes[c]))
      return fail(nullptr, PIO_ALS_ERR_ARG, "pio_cls_folds_create: labels must be finite (%s)", rf_fmt(cf->classes[c]).c_str());
  }
  return PIO_ALS_OK;
}

// keeps the predicted labels of fold f's m test rows, class_label[idx] with idx on the device; *out_result names them
static int clf_keep_result(pio_cls_folds* cf, int f, long long m, CallMem& tmp, const int* didx, const double* class_label,
                           int n_labels, int32_t* out_result) {
  double* dlab = nullptr;
  CK0(tmp.device(&dlab, (size_t)n_labels));
  CK0(cudaMemcpyAsync(dlab, class_label, 8 * (size_t)n_labels, cudaMemcpyHostToDevice, cf->st));
  pio_cls_folds::Result R;
  R.fold = f, R.m = m;
  CK0(cudaMalloc((void**)&R.pred, 8 * (size_t)(m ? m : 1)));
  if (m > 0) clf::pred_label_kernel<<<nblk(m, 256), 256, 0, cf->st>>>(didx, m, dlab, R.pred);
  const cudaError_t e0 = cudaGetLastError(), e1 = cudaStreamSynchronize(cf->st);
  if (e0 != cudaSuccess || e1 != cudaSuccess) {
    cudaFree(R.pred);
    return fail(nullptr, PIO_ALS_ERR_CUDA, "predicted labels: %s", cudaGetErrorString(e0 != cudaSuccess ? e0 : e1));
  }
  *out_result = cf->next_result++;
  cf->results[*out_result] = R;
  return PIO_ALS_OK;
}

}  // namespace pio

extern "C" {

int pio_cls_folds_create(int device, const double* label, const double* x, int64_t n, int32_t n_feat, int32_t k_fold,
                         pio_cls_folds** out) {
  if (!out) return fail(nullptr, PIO_ALS_ERR_ARG, "bad pio_cls_folds_create arguments");
  *out = nullptr;
  if (!label || !x || n < 1 || n_feat < 1 || k_fold < 1)
    return fail(nullptr, PIO_ALS_ERR_ARG, "bad pio_cls_folds_create arguments (n >= 1, n_feat >= 1 and k_fold >= 1)");
  if (n >= (1ll << 31)) return fail(nullptr, PIO_ALS_ERR_ARG, "n must be < 2^31");
  CK0(cudaSetDevice(device));
  auto* cf = new pio_cls_folds;
  cf->device = device, cf->k = k_fold, cf->F = n_feat, cf->n = n;
  const cudaError_t e = cudaStreamCreateWithFlags(&cf->st, cudaStreamNonBlocking);
  if (e != cudaSuccess) {
    delete cf;
    return fail(nullptr, PIO_ALS_ERR_CUDA, "cudaStreamCreate: %s", cudaGetErrorString(e));
  }
  const int rc = clf_build(cf, label, x);
  if (rc != PIO_ALS_OK) {
    pio_cls_folds_destroy(cf);
    return rc;
  }
  *out = cf;
  return PIO_ALS_OK;
}

int pio_cls_folds_sizes(const pio_cls_folds* cf, int32_t fold, int64_t out[2]) {
  EVF(clf_fold(cf, fold, "pio_cls_folds_sizes"));
  if (!out) return fail(nullptr, PIO_ALS_ERR_ARG, "pio_cls_folds_sizes: null out");
  const long long m = clf_n_test(cf, fold);
  out[0] = cf->n - m, out[1] = m;
  return PIO_ALS_OK;
}

int pio_cls_folds_classes(const pio_cls_folds* cf, int32_t fold, int32_t* n_class, double* labels) {
  EVF(clf_fold(cf, fold, "pio_cls_folds_classes"));
  if (!n_class) return fail(nullptr, PIO_ALS_ERR_ARG, "pio_cls_folds_classes: null n_class");
  std::vector<double> v;
  *n_class = clf_train_classes(cf, fold, nullptr, &v);
  if (labels && !v.empty()) memcpy(labels, v.data(), 8 * v.size());
  return PIO_ALS_OK;
}

int pio_cls_folds_nb_train(pio_cls_folds* cf, int32_t fold, double lambda, int32_t n_class, double* pi, double* theta) {
  EVF(clf_fold(cf, fold, "pio_cls_folds_nb_train"));
  std::vector<int> lmap;
  const int nc = clf_train_classes(cf, fold, &lmap, nullptr);
  if (!pi || !theta || n_class != nc)
    return fail(nullptr, PIO_ALS_ERR_ARG, "bad pio_cls_folds_nb_train arguments (fold %d has %d training classes)", fold,
                nc);
  const long long nt = cf->n - clf_n_test(cf, fold);
  if (nt == 0) return fail(nullptr, PIO_ALS_ERR_ARG, "fold %d has no training rows", fold);
  EVF(nb_check_width(cf->F, nc));
  CK0(cudaSetDevice(cf->device));
  CallMem tmp(cf->st);
  long long bad = -1;
  EVF(clf_first_bad(cf, fold, clf::CHECK_NEG_F32, 0, tmp, &bad));
  if (bad >= 0) return fail(nullptr, PIO_ALS_ERR_NUMERIC, "Naive Bayes requires nonnegative feature values");
  int *dmap = nullptr, *dl = nullptr;
  float* dx = nullptr;
  CK0(tmp.device(&dmap, (size_t)cf->C));
  CK0(tmp.device(&dl, (size_t)nt));
  CK0(tmp.device(&dx, (size_t)nt * cf->F));
  CK0(cudaMemcpyAsync(dmap, lmap.data(), 4 * (size_t)cf->C, cudaMemcpyHostToDevice, cf->st));
  clf::nb_gather_kernel<<<clf_grid(cf->n), clf::THREADS, 0, cf->st>>>(cf->cls, cf->x, cf->n, cf->F, cf->k, fold, dmap,
                                                                     dl, dx);
  CK0(cudaGetLastError());
  return nb_fit(tmp, cf->st, dl, dx, nt, cf->F, nc, lambda, pi, theta);
}

int pio_cls_folds_rf_train(pio_cls_folds* cf, int32_t fold, const pio_rf_params* p, pio_rf_forest** out) {
  EVF(clf_fold(cf, fold, "pio_cls_folds_rf_train"));
  if (!p || !out) return fail(nullptr, PIO_ALS_ERR_ARG, "bad pio_cls_folds_rf_train arguments");
  *out = nullptr;
  const long long nt = cf->n - clf_n_test(cf, fold);
  EVF(rf_check_params(p, nt, cf->F));
  CK0(cudaSetDevice(cf->device));
  {
    CallMem chk(cf->st);
    for (int mode : {clf::CHECK_FINITE, clf::CHECK_LABEL}) {
      long long e = -1;
      EVF(clf_first_bad(cf, fold, mode, p->num_classes, chk, &e));
      if (e < 0) continue;
      double lab = 0;
      std::vector<double> xr;
      EVF(clf_row(cf, e, &lab, &xr));
      EVF(mode == clf::CHECK_FINITE ? rf_fail_finite(clf_train_pos(cf, e, fold), lab, xr.data(), cf->F)
                                    : rf_fail_label(p, lab));
    }
  }
  g_rf_timing = RfTiming();
  RfTiming& tm = g_rf_timing;
  auto t0 = std::chrono::steady_clock::now();
  int sm = 0;
  CK0(cudaDeviceGetAttribute(&sm, cudaDevAttrMultiProcessorCount, cf->device));
  CallMem tmp;
  cudaStream_t st;
  CK0(tmp.stream(&st));
  double* dx = nullptr;
  uint8_t* dcls = nullptr;
  CK0(tmp.device(&dx, (size_t)nt * cf->F));
  CK0(tmp.device(&dcls, (size_t)nt));
  rf_ms(t0);
  clf::rf_gather_kernel<<<clf_grid(cf->n), clf::THREADS, 0, st>>>(cf->label, cf->x, cf->n, cf->F, cf->k, fold, dcls, dx);
  CK0(cudaGetLastError());
  CK0(cudaStreamSynchronize(st));
  tm.h2d = rf_ms(t0);   // the gather stands where pio_rf_train copies the rows in
  return rf_fit(p, dx, dcls, nt, cf->F, sm, tmp, st, t0, out);
}

int pio_cls_folds_nb_predict(pio_cls_folds* cf, int32_t fold, int32_t n_class, const double* pi, const double* theta,
                             const double* class_label, int32_t* out_result) {
  EVF(clf_fold(cf, fold, "pio_cls_folds_nb_predict"));
  if (!pi || !theta || !class_label || !out_result || n_class < 1)
    return fail(nullptr, PIO_ALS_ERR_ARG, "bad pio_cls_folds_nb_predict arguments");
  CK0(cudaSetDevice(cf->device));
  const long long m = clf_n_test(cf, fold);
  CallMem tmp(cf->st);
  int* didx = nullptr;
  CK0(tmp.device(&didx, (size_t)m));
  if (m > 0) {
    float* dx = nullptr;
    double *dpi = nullptr, *dth = nullptr;
    CK0(tmp.device(&dx, (size_t)m * cf->F));
    CK0(tmp.device(&dpi, (size_t)n_class));
    CK0(tmp.device(&dth, (size_t)n_class * cf->F));
    CK0(cudaMemcpyAsync(dpi, pi, 8 * (size_t)n_class, cudaMemcpyHostToDevice, cf->st));
    CK0(cudaMemcpyAsync(dth, theta, 8 * (size_t)n_class * cf->F, cudaMemcpyHostToDevice, cf->st));
    clf::test_gather_kernel<float><<<nblk(m, 256), 256, 0, cf->st>>>(cf->x, cf->F, cf->k, fold, m, dx);
    nb_predict_kernel<<<nblk(m, 256), 256, 0, cf->st>>>(dx, m, cf->F, n_class, dpi, dth, didx);
    CK0(cudaGetLastError());
  }
  return clf_keep_result(cf, fold, m, tmp, didx, class_label, n_class, out_result);
}

int pio_cls_folds_rf_predict(pio_cls_folds* cf, int32_t fold, int32_t n_trees, const int32_t* tree_off, int64_t n_nodes,
                             const int32_t* feature, const double* threshold, const int32_t* left, const int32_t* right,
                             const int32_t* prediction, int32_t num_classes, int32_t* out_result) {
  EVF(clf_fold(cf, fold, "pio_cls_folds_rf_predict"));
  if (!out_result) return fail(nullptr, PIO_ALS_ERR_ARG, "bad pio_cls_folds_rf_predict arguments");
  const RfFlat fl{n_trees, tree_off, n_nodes, feature, threshold, left, right, prediction, num_classes};
  EVF(rf_check_flat(fl, cf->F));
  CK0(cudaSetDevice(cf->device));
  const long long m = clf_n_test(cf, fold);
  CallMem tmp(cf->st);
  int* didx = nullptr;
  CK0(tmp.device(&didx, (size_t)m));
  if (m > 0) {
    double* dx = nullptr;
    CK0(tmp.device(&dx, (size_t)m * cf->F));
    clf::test_gather_kernel<double><<<nblk(m, 256), 256, 0, cf->st>>>(cf->x, cf->F, cf->k, fold, m, dx);
    CK0(cudaGetLastError());
    EVF(rf_predict_device(tmp, cf->st, fl, dx, m, cf->F, didx));
  }
  std::vector<double> cl(num_classes);   // the forest predicts the class index as its label
  for (int c = 0; c < num_classes; ++c) cl[c] = c;
  return clf_keep_result(cf, fold, m, tmp, didx, cl.data(), num_classes, out_result);
}

int pio_cls_folds_result_labels(const pio_cls_folds* cf, int32_t result, double* out) {
  if (!cf) return fail(nullptr, PIO_ALS_ERR_ARG, "pio_cls_folds_result_labels: null object");
  auto it = cf->results.find(result);
  if (it == cf->results.end()) return fail(nullptr, PIO_ALS_ERR_ARG, "no result %d", result);
  const pio_cls_folds::Result& R = it->second;
  if (R.m == 0) return PIO_ALS_OK;
  if (!out) return fail(nullptr, PIO_ALS_ERR_ARG, "pio_cls_folds_result_labels: null out");
  CK0(cudaSetDevice(cf->device));
  CK0(cudaMemcpyAsync(out, R.pred, 8 * (size_t)R.m, cudaMemcpyDeviceToHost, cf->st));
  CK0(cudaStreamSynchronize(cf->st));
  return PIO_ALS_OK;
}

int pio_cls_folds_result_counts(const pio_cls_folds* cf, int32_t result, double label, int64_t out[4]) {
  if (!cf || !out) return fail(nullptr, PIO_ALS_ERR_ARG, "bad pio_cls_folds_result_counts arguments");
  auto it = cf->results.find(result);
  if (it == cf->results.end()) return fail(nullptr, PIO_ALS_ERR_ARG, "no result %d", result);
  const pio_cls_folds::Result& R = it->second;
  unsigned long long h[3] = {0, 0, 0};
  if (R.m > 0) {
    CK0(cudaSetDevice(cf->device));
    CallMem tmp(cf->st);
    unsigned long long* d = nullptr;
    CK0(tmp.device(&d, 3));
    CK0(cudaMemsetAsync(d, 0, 3 * 8, cf->st));
    clf::counts_kernel<<<clf_grid(R.m), clf::THREADS, 0, cf->st>>>(R.pred, cf->label, R.m, cf->k, R.fold, label, d);
    CK0(cudaGetLastError());
    CK0(cudaMemcpyAsync(h, d, 3 * 8, cudaMemcpyDeviceToHost, cf->st));
    CK0(cudaStreamSynchronize(cf->st));
  }
  out[0] = R.m, out[1] = (int64_t)h[0], out[2] = (int64_t)h[1], out[3] = (int64_t)h[2];
  return PIO_ALS_OK;
}

int pio_cls_folds_result_free(pio_cls_folds* cf, int32_t result) {
  if (!cf) return fail(nullptr, PIO_ALS_ERR_ARG, "pio_cls_folds_result_free: null object");
  auto it = cf->results.find(result);
  if (it == cf->results.end()) return fail(nullptr, PIO_ALS_ERR_ARG, "no result %d", result);
  cudaSetDevice(cf->device);
  cudaFree(it->second.pred);
  cf->results.erase(it);
  return PIO_ALS_OK;
}

int pio_cls_folds_destroy(pio_cls_folds* cf) {
  if (!cf) return PIO_ALS_OK;
  cudaSetDevice(cf->device);
  if (cf->st) cudaStreamSynchronize(cf->st);
  for (auto& kv : cf->results) cudaFree(kv.second.pred);
  for (void* p : cf->mem) cudaFree(p);
  if (cf->st) cudaStreamDestroy(cf->st);
  delete cf;
  return PIO_ALS_OK;
}

}  // extern "C"

// ---- association rules (complementary purchase template, DESIGN.md 4.15) ---------------------------------------------
struct pio_assoc_model {
  int64_t n_transactions = 0;
  std::vector<int64_t> level_off{0};   // the sets of level l + 1 are [level_off[l], level_off[l + 1])
  std::vector<int64_t> set_prefix, set_count;
  std::vector<int32_t> set_item;
  std::vector<int64_t> rule_cond;
  std::vector<int32_t> rule_conseq;
  std::vector<double> support, confidence, lift;
};

namespace pio {

// where the last pio_assoc_train on this thread spent its time (wall ms; every phase ends in a stream synchronise)
struct AssocTiming {
  double h2d = 0, baskets = 0, level1 = 0, levels = 0, rules = 0, rank = 0, d2h = 0, total = 0;
  int64_t n_baskets = 0, n_transactions = 0, levels_run = 0, rejected_level = 0;
  int64_t cand[ASSOC_MAX_LEN + 1] = {};   // candidates counted for level k >= 2, a rejected level's included
};
static thread_local AssocTiming g_assoc_timing;

static int assoc_check(const pio_assoc_params* p) {
  if (p->max_rule_length < 2)
    return fail(nullptr, PIO_ALS_ERR_ARG, "maxRuleLength must be at least 2 (got %d)", p->max_rule_length);
  if (p->min_basket_size < 2)
    return fail(nullptr, PIO_ALS_ERR_ARG, "minBasketSize must be at least 2 (got %d)", p->min_basket_size);
  if (!(p->min_support >= 0.0 && p->min_support <= 1.0))
    return fail(nullptr, PIO_ALS_ERR_ARG, "minSupport must be in [0, 1] (got %g)", p->min_support);
  if (!(p->min_confidence >= 0.0 && p->min_confidence <= 1.0))
    return fail(nullptr, PIO_ALS_ERR_ARG, "minConfidence must be in [0, 1] (got %g)", p->min_confidence);
  if (p->max_num_rules_per_cond < 1)
    return fail(nullptr, PIO_ALS_ERR_ARG, "maxNumRulesPerCond must be at least 1 (got %d)", p->max_num_rules_per_cond);
  return PIO_ALS_OK;
}

// exclusive scan of v[0, n) into pos, and *total = the sum (synchronises st)
static cudaError_t assoc_total(const uint32_t* v, uint32_t* pos, long long n, cudaStream_t st, long long* total) {
  *total = 0;
  if (n == 0) return cudaSuccess;
  cudaError_t e = scan_exclusive_u32(v, pos, (size_t)n, st, nullptr);
  uint32_t last[2] = {0, 0};
  if (e == cudaSuccess) e = cudaMemcpyAsync(&last[0], pos + n - 1, 4, cudaMemcpyDeviceToHost, st);
  if (e == cudaSuccess) e = cudaMemcpyAsync(&last[1], v + n - 1, 4, cudaMemcpyDeviceToHost, st);
  if (e == cudaSuccess) e = cudaStreamSynchronize(st);
  *total = (long long)last[0] + last[1];
  return e;
}

// a 64-bit device counter, read back (synchronises st)
static cudaError_t assoc_read(const unsigned long long* d, cudaStream_t st, unsigned long long* out) {
  cudaError_t e = cudaMemcpyAsync(out, d, sizeof(*out), cudaMemcpyDeviceToHost, st);
  return e == cudaSuccess ? cudaStreamSynchronize(st) : e;
}

static int assoc_fit(int device, const int32_t* user, const int32_t* item, const int64_t* t_ms, long long n,
                     int32_t n_users, int32_t n_items, const pio_assoc_params* p, pio_assoc_model* m) {
  AssocTiming& tm = g_assoc_timing;
  const auto t0 = Clock::now();
  auto tp = t0;
  auto lap = [&tp]() {
    const auto now = Clock::now();
    const double r = std::chrono::duration<double, std::milli>(now - tp).count();
    tp = now;
    return r;
  };
  CK0(cudaSetDevice(device));
  CallMem call;
  cudaStream_t st;
  CK0(call.stream(&st));
  const int bits_u = ceil_log2((uint64_t)n_users), bits_i = ceil_log2((uint64_t)n_items);
  Scratch base(st);   // the kept baskets and the level-1 arrays, until the levels are built
  int* k_item = nullptr;
  uint32_t *k_basket = nullptr, *cnt1 = nullptr;
  long long NB = 0, T = 0, M = 0;
  lap();
  {
    // 1. baskets: (user, t, event) order, heads at a user change or a gap over the window, distinct (basket, item)
    Scratch tmp(st);
    int *du = nullptr, *di = nullptr;
    long long* dt = nullptr;
    uint32_t *head = nullptr, *bscan = nullptr;
    SortBufs sb;
    CK0(tmp.alloc(&du, (size_t)n)); CK0(tmp.alloc(&di, (size_t)n)); CK0(tmp.alloc(&dt, (size_t)n));
    CK0(tmp.alloc(&head, (size_t)n)); CK0(tmp.alloc(&bscan, (size_t)n));
    for (int b : {0, 1}) {
      CK0(tmp.alloc(&sb.k[b], (size_t)n));
      CK0(tmp.alloc(&sb.v[b], (size_t)n));
    }
    CK0(cudaMemcpyAsync(du, user, 4 * (size_t)n, cudaMemcpyHostToDevice, st));
    CK0(cudaMemcpyAsync(di, item, 4 * (size_t)n, cudaMemcpyHostToDevice, st));
    CK0(cudaMemcpyAsync(dt, t_ms, 8 * (size_t)n, cudaMemcpyHostToDevice, st));
    CK0(cudaStreamSynchronize(st));
    tm.h2d = lap();
    fold_time_key_kernel<<<nblk(n, 256), 256, 0, st>>>(dt, n, sb.keys(), sb.vals());
    CK0(radix_sort_pairs(sb, (size_t)n, 64, st, nullptr));
    fold_entity_key_kernel<<<nblk(n, 256), 256, 0, st>>>(sb.vals(), du, n, sb.keys());
    CK0(radix_sort_pairs(sb, (size_t)n, bits_u, st, nullptr));
    assoc_basket_head_kernel<<<nblk(n, 256), 256, 0, st>>>(sb.keys(), sb.vals(), dt, n,
                                                          (long long)p->basket_window * 1000ll, head);
    CK0(cudaGetLastError());
    long long n_raw = 0;
    CK0(assoc_total(head, bscan, n, st, &n_raw));
    assoc_bi_key_kernel<<<nblk(n, 256), 256, 0, st>>>(head, bscan, sb.vals(), di, n, bits_i, sb.spare_keys(),
                                                     sb.spare_vals());
    sb.flip();
    CK0(radix_sort_pairs(sb, (size_t)n, ceil_log2((uint64_t)n_raw) + bits_i, st, nullptr));
    uint32_t *flag = head, *pos = bscan;
    cooc_head_kernel<<<nblk(n, 256), 256, 0, st>>>(sb.keys(), n, flag);
    long long D = 0;
    CK0(assoc_total(flag, pos, n, st, &D));
    uint64_t* dk = sb.spare_keys();
    cooc_compact_kernel<<<nblk(n, 256), 256, 0, st>>>(sb.keys(), flag, pos, n, dk);
    // 2. basket sizes, minBasketSize, T
    uint32_t *bh = nullptr, *bord = nullptr, *keep = nullptr, *kord = nullptr, *eflag = nullptr, *epos = nullptr;
    CK0(tmp.alloc(&bh, (size_t)D)); CK0(tmp.alloc(&bord, (size_t)D));
    cooc_user_head_kernel<<<nblk(D, 256), 256, 0, st>>>(dk, D, bits_i, bh);
    CK0(assoc_total(bh, bord, D, st, &NB));
    CK0(tmp.alloc(&keep, (size_t)NB)); CK0(tmp.alloc(&kord, (size_t)NB));
    assoc_basket_size_kernel<<<nblk(D, 256), 256, 0, st>>>(dk, bh, bord, D, bits_i, p->min_basket_size, keep);
    CK0(assoc_total(keep, kord, NB, st, &T));
    CK0(tmp.alloc(&eflag, (size_t)D)); CK0(tmp.alloc(&epos, (size_t)D));
    assoc_kept_flag_kernel<<<nblk(D, 256), 256, 0, st>>>(bh, bord, keep, D, eflag);
    CK0(assoc_total(eflag, epos, D, st, &M));
    CK0(base.alloc(&k_item, (size_t)M)); CK0(base.alloc(&k_basket, (size_t)M));
    CK0(base.alloc(&cnt1, (size_t)n_items));
    CK0(cudaMemsetAsync(cnt1, 0, 4 * (size_t)n_items, st));
    assoc_kept_kernel<<<nblk(D, 256), 256, 0, st>>>(dk, bh, bord, kord, eflag, epos, D, bits_i, k_item, k_basket, cnt1);
    CK0(cudaGetLastError());
    CK0(cudaStreamSynchronize(st));
  }
  tm.baskets = lap();
  tm.n_baskets = NB;
  tm.n_transactions = m->n_transactions = T;
  if (T == 0) {
    tm.total = std::chrono::duration<double, std::milli>(Clock::now() - t0).count();
    return PIO_ALS_OK;
  }
  const double thr = p->min_support * (double)T;   // count >= minSupport * T, compared in fp64
  // 3. level 1, and the baskets pruned to their frequent items: the occurrences of the level-1 sets
  Scratch sets(st);                                 // keys and counts of every level, until the rules are made
  std::vector<uint64_t*> lkeys{nullptr};
  std::vector<uint32_t*> lcount{nullptr};
  std::vector<long long> ln{0};
  auto occ_mem = std::make_unique<Scratch>(st);
  uint32_t *occ_pos = nullptr, *occ_id = nullptr, *end = nullptr;
  int* p_item = nullptr;
  long long NO = 0;
  {
    uint32_t *f1 = nullptr, *id1 = nullptr;
    CK0(base.alloc(&f1, (size_t)n_items)); CK0(base.alloc(&id1, (size_t)n_items));
    assoc_l1_flag_kernel<<<nblk(n_items, 256), 256, 0, st>>>(cnt1, n_items, thr, f1);
    long long L1 = 0;
    CK0(assoc_total(f1, id1, n_items, st, &L1));
    if (L1 > 0) {
      uint64_t* k1 = nullptr;
      uint32_t* c1 = nullptr;
      CK0(sets.alloc(&k1, (size_t)L1)); CK0(sets.alloc(&c1, (size_t)L1));
      assoc_l1_emit_kernel<<<nblk(n_items, 256), 256, 0, st>>>(cnt1, f1, id1, n_items, k1, c1);
      lkeys.push_back(k1), lcount.push_back(c1), ln.push_back(L1);
      Scratch tmp(st);
      uint32_t *pflag = nullptr, *ppos = nullptr, *p_basket = nullptr, *hd = nullptr, *sidx = nullptr, *seg = nullptr;
      CK0(tmp.alloc(&pflag, (size_t)M)); CK0(tmp.alloc(&ppos, (size_t)M));
      assoc_prune_flag_kernel<<<nblk(M, 256), 256, 0, st>>>(k_item, f1, M, pflag);
      CK0(assoc_total(pflag, ppos, M, st, &NO));
      CK0(base.alloc(&p_item, (size_t)NO)); CK0(base.alloc(&end, (size_t)NO));
      CK0(tmp.alloc(&p_basket, (size_t)NO)); CK0(tmp.alloc(&hd, (size_t)NO)); CK0(tmp.alloc(&sidx, (size_t)NO));
      CK0(occ_mem->alloc(&occ_pos, (size_t)NO)); CK0(occ_mem->alloc(&occ_id, (size_t)NO));
      assoc_prune_kernel<<<nblk(M, 256), 256, 0, st>>>(k_item, k_basket, pflag, ppos, id1, M, p_item, p_basket, occ_pos,
                                                       occ_id);
      assoc_seg_start_kernel<<<nblk(NO, 256), 256, 0, st>>>(p_basket, NO, hd);
      long long n_seg = 0;
      CK0(assoc_total(hd, sidx, NO, st, &n_seg));
      CK0(tmp.alloc(&seg, (size_t)n_seg + 1));
      const uint32_t np32 = (uint32_t)NO;
      CK0(cudaMemcpyAsync(seg + n_seg, &np32, 4, cudaMemcpyHostToDevice, st));
      assoc_seg_pos_kernel<<<nblk(NO, 256), 256, 0, st>>>(hd, sidx, NO, seg);
      assoc_seg_end_kernel<<<nblk(NO, 256), 256, 0, st>>>(hd, sidx, seg, NO, end);
      CK0(cudaGetLastError());
      CK0(cudaStreamSynchronize(st));
    }
  }
  tm.level1 = lap();
  // 4. levels 2 .. maxRuleLength: extend the occurrences of the frequent (k-1)-sets, count, keep the frequent sets
  long long n_sets = ln.back();
  for (int k = 2; k <= p->max_rule_length && (int)ln.size() == k && NO > 0; ++k) {
    Scratch tmp(st);
    uint32_t *ext = nullptr, *off = nullptr;
    unsigned long long* dtot = nullptr;
    CK0(tmp.alloc(&ext, (size_t)NO)); CK0(tmp.alloc(&off, (size_t)NO)); CK0(tmp.alloc(&dtot, 1));
    CK0(cudaMemsetAsync(dtot, 0, sizeof(unsigned long long), st));
    assoc_ext_kernel<<<nblk(NO, 256), 256, 0, st>>>(occ_pos, end, NO, ext, dtot);
    unsigned long long tot = 0;
    CK0(assoc_read(dtot, st, &tot));
    if (k <= ASSOC_MAX_LEN) tm.cand[k] = (int64_t)tot;
    if (tot > (unsigned long long)PIO_ASSOC_MAX_CANDIDATES) {
      tm.rejected_level = k;
      return fail(nullptr, PIO_ALS_ERR_ARG,
                  "the item sets of length %d have %llu candidates, more than the limit of %lld: raise minSupport, "
                  "lower maxRuleLength or shorten basketWindow", k, tot, (long long)PIO_ASSOC_MAX_CANDIDATES);
    }
    if (tot == 0) break;
    if (k > ASSOC_MAX_LEN)
      return fail(nullptr, PIO_ALS_ERR_ARG, "item sets longer than %d items are not supported", ASSOC_MAX_LEN);
    ++tm.levels_run;
    const long long C = (long long)tot;
    CK0(scan_exclusive_u32(ext, off, (size_t)NO, st, nullptr));
    SortBufs cs;
    uint32_t *cand_pos = nullptr, *hf = nullptr, *rix = nullptr;
    for (int b : {0, 1}) {
      CK0(tmp.alloc(&cs.k[b], (size_t)C));
      CK0(tmp.alloc(&cs.v[b], (size_t)C));
    }
    CK0(tmp.alloc(&cand_pos, (size_t)C)); CK0(tmp.alloc(&hf, (size_t)C)); CK0(tmp.alloc(&rix, (size_t)C));
    assoc_expand_kernel<<<nblk(NO, 256), 256, 0, st>>>(occ_pos, occ_id, ext, off, NO, p_item, bits_i, cs.keys(),
                                                       cs.vals(), cand_pos);
    CK0(radix_sort_pairs(cs, (size_t)C, ceil_log2((uint64_t)ln[k - 1]) + bits_i, st, nullptr));
    cooc_head_kernel<<<nblk(C, 256), 256, 0, st>>>(cs.keys(), C, hf);
    long long R = 0, Lk = 0;
    CK0(assoc_total(hf, rix, C, st, &R));
    uint64_t* rkey = nullptr;
    uint32_t *rcnt = nullptr, *rf = nullptr, *rid = nullptr;
    CK0(tmp.alloc(&rkey, (size_t)R)); CK0(tmp.alloc(&rcnt, (size_t)R)); CK0(tmp.alloc(&rf, (size_t)R));
    CK0(tmp.alloc(&rid, (size_t)R));
    assoc_runs_kernel<<<nblk(C, 256), 256, 0, st>>>(cs.keys(), hf, rix, C, thr, rkey, rcnt, rf);
    CK0(assoc_total(rf, rid, R, st, &Lk));
    if (Lk == 0) break;
    if (n_sets + Lk >= (1ll << 31)) return fail(nullptr, PIO_ALS_ERR_ARG, "2^31 or more frequent item sets");
    n_sets += Lk;
    uint64_t* kk = nullptr;
    uint32_t* ck = nullptr;
    CK0(sets.alloc(&kk, (size_t)Lk)); CK0(sets.alloc(&ck, (size_t)Lk));
    assoc_level_emit_kernel<<<nblk(R, 256), 256, 0, st>>>(rkey, rcnt, rf, rid, R, kk, ck);
    lkeys.push_back(kk), lcount.push_back(ck), ln.push_back(Lk);
    if (k < p->max_rule_length) {
      uint32_t *oflag = nullptr, *opos = nullptr;
      CK0(tmp.alloc(&oflag, (size_t)C)); CK0(tmp.alloc(&opos, (size_t)C));
      assoc_occ_flag_kernel<<<nblk(C, 256), 256, 0, st>>>(hf, rix, rf, C, oflag);
      long long NO2 = 0;
      CK0(assoc_total(oflag, opos, C, st, &NO2));
      auto next = std::make_unique<Scratch>(st);
      uint32_t *op2 = nullptr, *oi2 = nullptr;
      CK0(next->alloc(&op2, (size_t)NO2)); CK0(next->alloc(&oi2, (size_t)NO2));
      assoc_occ_kernel<<<nblk(C, 256), 256, 0, st>>>(cs.vals(), cand_pos, hf, rix, rid, oflag, opos, C, op2, oi2);
      occ_mem = std::move(next);
      occ_pos = op2, occ_id = oi2, NO = NO2;
    }
    CK0(cudaGetLastError());
    CK0(cudaStreamSynchronize(st));
  }
  tm.levels = lap();
  const int K = (int)ln.size() - 1;
  // 5. rules of every set of level k >= 2, counted per set, then written at their scanned offsets
  AssocLevels L{};
  for (int l = 1; l <= K; ++l) {
    L.keys[l] = lkeys[l], L.count[l] = lcount[l], L.n[l] = (uint32_t)ln[l];
    L.base[l] = l == 1 ? 0u : L.base[l - 1] + L.n[l - 1];
  }
  Scratch rules(st);
  std::vector<uint32_t*> roff((size_t)K + 1, nullptr);
  std::vector<long long> rbase((size_t)K + 2, 0);
  {
    unsigned long long* dtot = nullptr;
    CK0(rules.alloc(&dtot, 1));
    for (int k = 2; k <= K; ++k) {
      uint32_t* npass = nullptr;
      CK0(rules.alloc(&npass, (size_t)ln[k])); CK0(rules.alloc(&roff[k], (size_t)ln[k]));
      CK0(cudaMemsetAsync(dtot, 0, sizeof(unsigned long long), st));
      const AssocRuleArgs a{k, bits_i, (double)T, p->min_confidence, p->min_lift};
      assoc_rule_kernel<0><<<nblk(ln[k], ASSOC_RULE_THREADS), ASSOC_RULE_THREADS, 0, st>>>(
          L, a, npass, dtot, nullptr, nullptr, nullptr, nullptr, nullptr, nullptr);
      CK0(cudaGetLastError());
      unsigned long long tot = 0;
      CK0(assoc_read(dtot, st, &tot));
      if ((unsigned long long)rbase[k] + tot >= (1ull << 31))
        return fail(nullptr, PIO_ALS_ERR_ARG, "2^31 or more rules pass minConfidence and minLift");
      CK0(scan_exclusive_u32(npass, roff[k], (size_t)ln[k], st, nullptr));
      rbase[k + 1] = rbase[k] + (long long)tot;
    }
  }
  const long long RT = K >= 2 ? rbase[K + 1] : 0;
  uint32_t* r_cond = nullptr;
  int* r_conseq = nullptr;
  double *r_sup = nullptr, *r_conf = nullptr, *r_lift = nullptr;
  CK0(rules.alloc(&r_cond, (size_t)RT)); CK0(rules.alloc(&r_conseq, (size_t)RT));
  CK0(rules.alloc(&r_sup, (size_t)RT)); CK0(rules.alloc(&r_conf, (size_t)RT)); CK0(rules.alloc(&r_lift, (size_t)RT));
  for (int k = 2; k <= K; ++k) {
    if (rbase[k + 1] == rbase[k]) continue;
    const AssocRuleArgs a{k, bits_i, (double)T, p->min_confidence, p->min_lift};
    const long long b = rbase[k];
    assoc_rule_kernel<1><<<nblk(ln[k], ASSOC_RULE_THREADS), ASSOC_RULE_THREADS, 0, st>>>(
        L, a, nullptr, nullptr, roff[k], r_cond + b, r_conseq + b, r_sup + b, r_conf + b, r_lift + b);
    CK0(cudaGetLastError());
  }
  CK0(cudaStreamSynchronize(st));
  tm.rules = lap();
  // 6. ranking per condition: lift descending, then the conseq's item index; the first maxNumRulesPerCond
  long long RK = 0;
  uint32_t* o_cond = nullptr;
  int* o_conseq = nullptr;
  double *o_sup = nullptr, *o_conf = nullptr, *o_lift = nullptr;
  if (RT > 0) {
    SortBufs rs;
    for (int b : {0, 1}) {
      CK0(rules.alloc(&rs.k[b], (size_t)RT));
      CK0(rules.alloc(&rs.v[b], (size_t)RT));
    }
    assoc_rank_key_kernel<<<nblk(RT, 256), 256, 0, st>>>(nullptr, RT, 0, r_cond, r_conseq, r_lift, rs.keys(), rs.vals());
    CK0(radix_sort_pairs(rs, (size_t)RT, bits_i, st, nullptr));
    assoc_rank_key_kernel<<<nblk(RT, 256), 256, 0, st>>>(rs.vals(), RT, 1, r_cond, r_conseq, r_lift, rs.spare_keys(),
                                                         rs.spare_vals());
    rs.flip();
    CK0(radix_sort_pairs(rs, (size_t)RT, 64, st, nullptr));
    assoc_rank_key_kernel<<<nblk(RT, 256), 256, 0, st>>>(rs.vals(), RT, 2, r_cond, r_conseq, r_lift, rs.spare_keys(),
                                                         rs.spare_vals());
    rs.flip();
    CK0(radix_sort_pairs(rs, (size_t)RT, ceil_log2((uint64_t)n_sets), st, nullptr));
    uint32_t *ccount = nullptr, *cstart = nullptr, *kcount = nullptr, *kstart = nullptr;
    CK0(rules.alloc(&ccount, (size_t)n_sets)); CK0(rules.alloc(&cstart, (size_t)n_sets));
    CK0(rules.alloc(&kcount, (size_t)n_sets)); CK0(rules.alloc(&kstart, (size_t)n_sets));
    CK0(cudaMemsetAsync(ccount, 0, 4 * (size_t)n_sets, st));
    assoc_cond_count_kernel<<<nblk(RT, 256), 256, 0, st>>>(rs.keys(), RT, ccount);
    CK0(scan_exclusive_u32(ccount, cstart, (size_t)n_sets, st, nullptr));
    const uint32_t per = (uint32_t)p->max_num_rules_per_cond;
    assoc_cond_keep_kernel<<<nblk(n_sets, 256), 256, 0, st>>>(ccount, n_sets, per, kcount);
    CK0(assoc_total(kcount, kstart, n_sets, st, &RK));
    CK0(rules.alloc(&o_cond, (size_t)RK)); CK0(rules.alloc(&o_conseq, (size_t)RK));
    CK0(rules.alloc(&o_sup, (size_t)RK)); CK0(rules.alloc(&o_conf, (size_t)RK)); CK0(rules.alloc(&o_lift, (size_t)RK));
    assoc_take_kernel<<<nblk(RT, 256), 256, 0, st>>>(rs.keys(), rs.vals(), RT, cstart, kstart, per, r_cond, r_conseq,
                                                     r_sup, r_conf, r_lift, o_cond, o_conseq, o_sup, o_conf, o_lift);
    CK0(cudaGetLastError());
    CK0(cudaStreamSynchronize(st));
  }
  tm.rank = lap();
  // 7. the model on the host: sets as (global id of the prefix, last item, count), rules in ranked order
  m->level_off.assign((size_t)K + 1, 0);
  for (int l = 1; l <= K; ++l) m->level_off[l] = m->level_off[l - 1] + ln[l];
  m->set_prefix.resize((size_t)n_sets);
  m->set_item.resize((size_t)n_sets);
  m->set_count.resize((size_t)n_sets);
  {
    std::vector<uint64_t> hk;
    std::vector<uint32_t> hc;
    const uint64_t imask = (1ull << bits_i) - 1ull;
    for (int l = 1; l <= K; ++l) {
      hk.resize((size_t)ln[l]);
      hc.resize((size_t)ln[l]);
      CK0(cudaMemcpyAsync(hk.data(), lkeys[l], 8 * (size_t)ln[l], cudaMemcpyDeviceToHost, st));
      CK0(cudaMemcpyAsync(hc.data(), lcount[l], 4 * (size_t)ln[l], cudaMemcpyDeviceToHost, st));
      CK0(cudaStreamSynchronize(st));
      const int64_t o = m->level_off[l - 1];
      for (long long j = 0; j < ln[l]; ++j) {
        m->set_prefix[o + j] = l == 1 ? -1 : m->level_off[l - 2] + (int64_t)(hk[j] >> bits_i);
        m->set_item[o + j] = (int32_t)(l == 1 ? hk[j] : (hk[j] & imask));
        m->set_count[o + j] = hc[j];
      }
    }
  }
  std::vector<uint32_t> hcond((size_t)RK);
  m->rule_cond.resize((size_t)RK);
  m->rule_conseq.resize((size_t)RK);
  m->support.resize((size_t)RK);
  m->confidence.resize((size_t)RK);
  m->lift.resize((size_t)RK);
  if (RK > 0) {
    CK0(cudaMemcpyAsync(hcond.data(), o_cond, 4 * (size_t)RK, cudaMemcpyDeviceToHost, st));
    CK0(cudaMemcpyAsync(m->rule_conseq.data(), o_conseq, 4 * (size_t)RK, cudaMemcpyDeviceToHost, st));
    CK0(cudaMemcpyAsync(m->support.data(), o_sup, 8 * (size_t)RK, cudaMemcpyDeviceToHost, st));
    CK0(cudaMemcpyAsync(m->confidence.data(), o_conf, 8 * (size_t)RK, cudaMemcpyDeviceToHost, st));
    CK0(cudaMemcpyAsync(m->lift.data(), o_lift, 8 * (size_t)RK, cudaMemcpyDeviceToHost, st));
    CK0(cudaStreamSynchronize(st));
  }
  for (long long r = 0; r < RK; ++r) m->rule_cond[r] = hcond[r];
  tm.d2h = lap();
  tm.total = std::chrono::duration<double, std::milli>(Clock::now() - t0).count();
  return PIO_ALS_OK;
}

}  // namespace pio

extern "C" {

int pio_assoc_train(int device, const int32_t* user, const int32_t* item, const int64_t* t_ms, int64_t n,
                    int32_t n_users, int32_t n_items, const pio_assoc_params* p, pio_assoc_model** out) {
  if (!p || !out || n < 0 || (n > 0 && (!user || !item || !t_ms)) || n_users < 1 || n_items < 1)
    return fail(nullptr, PIO_ALS_ERR_ARG, "bad pio_assoc_train arguments");
  *out = nullptr;
  EVF(assoc_check(p));
  if (n >= (1ll << 32)) return fail(nullptr, PIO_ALS_ERR_ARG, "n must be < 2^32");
  for (int64_t e = 0; e < n; ++e)
    if (user[e] < 0 || user[e] >= n_users || item[e] < 0 || item[e] >= n_items)
      return fail(nullptr, PIO_ALS_ERR_ARG, "event %lld has a user/item index out of range", (long long)e);
  g_assoc_timing = AssocTiming();
  try {
    std::unique_ptr<pio_assoc_model> m(new pio_assoc_model());
    if (n > 0) EVF(assoc_fit(device, user, item, t_ms, (long long)n, n_users, n_items, p, m.get()));
    *out = m.release();
  } catch (const std::bad_alloc&) {
    return fail(nullptr, PIO_ALS_ERR_NOMEM, "pio_assoc_train: out of host memory");
  }
  return PIO_ALS_OK;
}

int pio_assoc_model_size(const pio_assoc_model* m, int32_t* n_levels, int64_t* n_sets, int64_t* n_rules,
                         int64_t* n_transactions) {
  if (!m) return fail(nullptr, PIO_ALS_ERR_ARG, "null association model");
  if (n_levels) *n_levels = (int32_t)m->level_off.size() - 1;
  if (n_sets) *n_sets = (int64_t)m->set_item.size();
  if (n_rules) *n_rules = (int64_t)m->rule_conseq.size();
  if (n_transactions) *n_transactions = m->n_transactions;
  return PIO_ALS_OK;
}

int pio_assoc_model_get(const pio_assoc_model* m, int64_t* level_off, int64_t* set_prefix, int32_t* set_item,
                        int64_t* set_count, int64_t* rule_cond, int32_t* rule_conseq, double* support,
                        double* confidence, double* lift) {
  if (!m) return fail(nullptr, PIO_ALS_ERR_ARG, "null association model");
  auto put = [](auto* dst, const auto& v) {
    if (dst && !v.empty()) memcpy(dst, v.data(), v.size() * sizeof(v[0]));
  };
  put(level_off, m->level_off);
  put(set_prefix, m->set_prefix);
  put(set_item, m->set_item);
  put(set_count, m->set_count);
  put(rule_cond, m->rule_cond);
  put(rule_conseq, m->rule_conseq);
  put(support, m->support);
  put(confidence, m->confidence);
  put(lift, m->lift);
  return PIO_ALS_OK;
}

int pio_assoc_model_destroy(pio_assoc_model* m) {
  delete m;
  return PIO_ALS_OK;
}

/* debug only (not in pio_als.h): the last pio_assoc_train on this thread, wall ms of phases that each end in a stream
 * synchronise: out[0] host-to-device copy, [1] baskets, [2] level 1 and the pruned baskets, [3] levels >= 2, [4] rules,
 * [5] ranking, [6] device-to-host copy and the host model, [7] total; [8] baskets before minBasketSize, [9]
 * transactions T, [10] levels >= 2 enumerated, [11] the level rejected by the candidate limit (0: none); [16 + k]
 * candidates counted for level k (2 <= k <= 32).  Used by tools/assoc_bench.py and tests/test_gpu_assoc.py. */
__attribute__((visibility("default"))) int pio_assoc_debug_timing(double out[64]) {
  if (!out) return PIO_ALS_ERR_ARG;
  const AssocTiming& t = g_assoc_timing;
  out[0] = t.h2d, out[1] = t.baskets, out[2] = t.level1, out[3] = t.levels, out[4] = t.rules, out[5] = t.rank;
  out[6] = t.d2h, out[7] = t.total;
  out[8] = (double)t.n_baskets, out[9] = (double)t.n_transactions, out[10] = (double)t.levels_run;
  out[11] = (double)t.rejected_level;
  for (int k = 12; k < 16; ++k) out[k] = 0;
  for (int k = 0; k <= ASSOC_MAX_LEN; ++k) out[16 + k] = (double)t.cand[k];
  for (int k = 16 + ASSOC_MAX_LEN + 1; k < 64; ++k) out[k] = 0;
  return PIO_ALS_OK;
}

}  // extern "C"

// ---- product ranking (pio_als_rank_lists) -------------------------------------------------------------------------------
namespace pio {

// what the last pio_als_rank_lists on this thread did (pio_rank_lists_debug_stats)
struct RankListsStats {
  long long parts = 0, tile_queries = 0, radix_queries = 0, entries = 0, max_part_entries = 0;
  double device_ms = 0.0;
};
static thread_local RankListsStats g_rl_stats;

// host arrays packed into one upload, each block on a 256-byte boundary
struct HostPack {
  std::vector<unsigned char> buf;
  template <class T>
  size_t put(const T* src, size_t n) {
    const size_t at = al256(buf.size());
    buf.resize(at + n * sizeof(T));
    if (n) memcpy(buf.data() + at, src, n * sizeof(T));
    return at;
  }
};

// One part of a call (rank_plan.h): its inputs up, the tile CTAs and the radix sorts on the handle's stream, its outputs
// down into the caller's arrays at the part's offsets.
static int rank_part(pio_als_handle* h, const RankPart& p, const int32_t* users, const int64_t* list_ptr,
                     const int32_t* items, int32_t* out_pos, double* out_scores, uint8_t* out_ranked) {
  cudaStream_t st = h->stream;
  const int nq = p.q1 - p.q0, nt = p.n_tiles(), nr = (int)p.radix.size();
  const long long ne = p.e1 - p.e0;
  std::vector<long long> lp((size_t)nq + 1), c((size_t)nr + 1, 0);
  for (int j = 0; j <= nq; ++j) lp[j] = list_ptr[p.q0 + j] - p.e0;
  std::vector<int> tq(p.tile_q), rq(p.radix);
  for (int& q : tq) q -= p.q0;
  for (int k = 0; k < nr; ++k) {
    rq[k] -= p.q0;
    c[k + 1] = c[k] + (lp[rq[k] + 1] - lp[rq[k]]);
  }
  HostPack pk;
  const size_t at_lp = pk.put(lp.data(), lp.size()), at_tq = pk.put(tq.data(), tq.size()),
               at_tp = pk.put(p.tile_ptr.data(), p.tile_ptr.size()), at_to = pk.put(p.tile_off.data(), p.tile_off.size()),
               at_tn = pk.put(p.tile_n.data(), p.tile_n.size()), at_rq = pk.put(rq.data(), rq.size()),
               at_c = pk.put(c.data(), c.size());
  Scratch tmp(st);
  unsigned char* d_pack = nullptr;
  int *d_users = nullptr, *d_items = nullptr, *d_pos = nullptr;
  double* d_score = nullptr;
  uint8_t* d_ranked = nullptr;
  CK(h, tmp.alloc(&d_pack, pk.buf.size()));
  CK(h, tmp.alloc(&d_users, (size_t)nq));
  CK(h, tmp.alloc(&d_items, (size_t)ne));
  CK(h, tmp.alloc(&d_pos, (size_t)ne));
  CK(h, tmp.alloc(&d_score, (size_t)ne));
  CK(h, tmp.alloc(&d_ranked, (size_t)nq));
  CK(h, cudaMemcpyAsync(d_pack, pk.buf.data(), pk.buf.size(), cudaMemcpyHostToDevice, st));
  CK(h, cudaMemcpyAsync(d_users, users + p.q0, sizeof(int) * (size_t)nq, cudaMemcpyHostToDevice, st));
  if (ne) CK(h, cudaMemcpyAsync(d_items, items + p.e0, sizeof(int) * (size_t)ne, cudaMemcpyHostToDevice, st));
  CK(h, cudaMemsetAsync(d_ranked, 0, (size_t)nq, st));   // an empty list is not ranked
  const RlSide U{h->U.F, h->U.perm, h->U.deg, h->U.n}, I{h->I.F, h->I.perm, h->I.deg, h->I.n};
  const RlPart dp{d_users, (const long long*)(d_pack + at_lp), d_items, d_pos, d_score, d_ranked};
  if (nt) {
    rl_tile_kernel<<<nt, RL_THREADS, 0, st>>>(U, I, h->KP, dp, (const int*)(d_pack + at_tq), (const int*)(d_pack + at_tp),
                                              (const int*)(d_pack + at_to), (const int*)(d_pack + at_tn));
    LAUNCHED(h);
    CK(h, cudaGetLastError());
  }
  if (nr) {
    const long long n = c[nr];
    const int* d_rq = (const int*)(d_pack + at_rq);
    const long long* d_c = (const long long*)(d_pack + at_c);
    SortBufs sb;
    double* d_rscore = nullptr;
    uint8_t* d_has = nullptr;
    for (int b = 0; b < 2; ++b) {
      CK(h, tmp.alloc(&sb.k[b], (size_t)n));
      CK(h, tmp.alloc(&sb.v[b], (size_t)n));
    }
    CK(h, tmp.alloc(&d_rscore, (size_t)n));
    CK(h, tmp.alloc(&d_has, (size_t)nr));
    CK(h, cudaMemsetAsync(d_has, 0, (size_t)nr, st));
    const unsigned grid = (unsigned)std::min<long long>(nblk(n, 256), (long long)std::max(h->sm_count, 1) * 16);
    rl_radix_score_kernel<<<grid, 256, 0, st>>>(U, I, h->KP, dp, d_rq, d_c, nr, n, sb.keys(), sb.vals(), d_rscore, d_has);
    LAUNCHED(h);
    CK(h, cudaGetLastError());
    CK(h, radix_sort_pairs(sb, (size_t)n, 64, st, &h->st.kernel_launches));
    if (nr > 1) {   // equal keys of a query stay in entry order: a stable sort by the query alone groups them
      rl_radix_query_keys_kernel<<<grid, 256, 0, st>>>(sb.vals(), d_c, nr, n, sb.spare_keys(), sb.spare_vals());
      LAUNCHED(h);
      CK(h, cudaGetLastError());
      sb.flip();
      CK(h, radix_sort_pairs(sb, (size_t)n, ceil_log2((uint64_t)nr), st, &h->st.kernel_launches));
    } else {
      CK(h, cudaMemsetAsync(sb.keys(), 0, sizeof(uint64_t) * (size_t)n, st));
    }
    rl_radix_out_kernel<<<grid, 256, 0, st>>>(dp, d_rq, d_c, sb.keys(), sb.vals(), d_rscore, d_has, n);
    LAUNCHED(h);
    CK(h, cudaGetLastError());
  }
  if (ne) {
    CK(h, cudaMemcpyAsync(out_pos + p.e0, d_pos, sizeof(int) * (size_t)ne, cudaMemcpyDeviceToHost, st));
    CK(h, cudaMemcpyAsync(out_scores + p.e0, d_score, sizeof(double) * (size_t)ne, cudaMemcpyDeviceToHost, st));
  }
  CK(h, cudaMemcpyAsync(out_ranked + p.q0, d_ranked, (size_t)nq, cudaMemcpyDeviceToHost, st));
  CK(h, cudaStreamSynchronize(st));
  return PIO_ALS_OK;
}

static int rank_lists(pio_als_handle* h, const int32_t* users, int32_t n_queries, const int64_t* list_ptr,
                      const int32_t* items, int32_t* out_pos, double* out_scores, uint8_t* out_ranked) {
  if (n_queries < 0) return fail(h, PIO_ALS_ERR_ARG, "n_queries must be >= 0");
  if (!list_ptr || !out_pos || !out_scores || !out_ranked || (n_queries > 0 && !users))
    return fail(h, PIO_ALS_ERR_ARG, "null argument");
  if (list_ptr[0] != 0) return fail(h, PIO_ALS_ERR_ARG, "list_ptr[0] must be 0, not %lld", (long long)list_ptr[0]);
  for (int q = 0; q < n_queries; ++q) {
    const long long len = list_ptr[q + 1] - list_ptr[q];
    if (len < 0) return fail(h, PIO_ALS_ERR_ARG, "list_ptr decreases at query %d", q);
    if (len >= (1ll << 31)) return fail(h, PIO_ALS_ERR_ARG, "query %d has %lld entries: a list holds fewer than 2^31", q, len);
  }
  if (list_ptr[n_queries] > 0 && !items) return fail(h, PIO_ALS_ERR_ARG, "null argument");
  if (n_queries == 0) return PIO_ALS_OK;
  if (!h->U.F || !h->I.F) return fail(h, PIO_ALS_ERR_STATE, "no model");
  // PIO_RANK_LISTS_BUDGET: entries per part; capped so that a part's entries are numbered in 32 bits
  const char* env_b = getenv("PIO_RANK_LISTS_BUDGET");
  const long long budget = std::min<long long>(env_b && atoll(env_b) > 0 ? atoll(env_b) : PIO_RANK_LISTS_BUDGET,
                                               (1ll << 31) - 1);
  const std::vector<RankPart> parts = plan_rank_lists(list_ptr, n_queries, budget);
  CK(h, cudaSetDevice(h->cfg.device));
  cudaEvent_t ev[2] = {nullptr, nullptr};
  CK(h, cudaEventCreate(&ev[0]));
  const cudaError_t e1 = cudaEventCreate(&ev[1]);
  if (e1 != cudaSuccess) {
    cudaEventDestroy(ev[0]);
    CK(h, e1);
  }
  struct Events {
    cudaEvent_t* e;
    ~Events() { cudaEventDestroy(e[0]), cudaEventDestroy(e[1]); }
  } own{ev};
  CK(h, cudaEventRecord(ev[0], h->stream));
  RankListsStats& s = g_rl_stats;
  for (const RankPart& p : parts) {
    s.parts += 1;
    s.tile_queries += (long long)p.tile_q.size();
    s.radix_queries += (long long)p.radix.size();
    s.entries += p.e1 - p.e0;
    s.max_part_entries = std::max(s.max_part_entries, p.e1 - p.e0);
    const int rc = rank_part(h, p, users, list_ptr, items, out_pos, out_scores, out_ranked);
    if (rc) return rc;
  }
  CK(h, cudaEventRecord(ev[1], h->stream));
  CK(h, cudaEventSynchronize(ev[1]));
  float ms = 0.f;
  CK(h, cudaEventElapsedTime(&ms, ev[0], ev[1]));
  s.device_ms = ms;
  return PIO_ALS_OK;
}

}  // namespace pio

extern "C" {

int pio_als_rank_lists(pio_als_handle* h, const int32_t* users, int32_t n_queries, const int64_t* list_ptr,
                       const int32_t* items, int32_t* out_pos, double* out_scores, uint8_t* out_ranked) {
  g_rl_stats = RankListsStats{};
  if (!h) return fail(nullptr, PIO_ALS_ERR_ARG, "null handle");
  std::lock_guard<std::mutex> lk(h->mu);
  try {   // bad_alloc must not cross the C boundary; Scratch releases device memory on the way out
    return rank_lists(h, users, n_queries, list_ptr, items, out_pos, out_scores, out_ranked);
  } catch (const std::bad_alloc&) {
    return fail(h, PIO_ALS_ERR_NOMEM, "pio_als_rank_lists: out of host memory");
  }
}

int pio_rank_lists_debug_stats(double out[6]) {
  if (!out) return PIO_ALS_ERR_ARG;
  const RankListsStats& s = g_rl_stats;
  out[0] = (double)s.parts, out[1] = (double)s.tile_queries, out[2] = (double)s.radix_queries;
  out[3] = (double)s.entries, out[4] = (double)s.max_part_entries, out[5] = s.device_ms;
  return PIO_ALS_OK;
}

}  // extern "C"

// ---- association rule predict (complementary purchase Algorithm.predict on batches, DESIGN.md 4.15.1) --------------------
namespace pio {
// the conds of a pio_assoc_predict call, in the contract's order (pio_als.h)
struct ApResult {
  std::vector<int64_t> q_cond_ptr, cond_ptr, rule_first;
  std::vector<int32_t> cond_items, rule_n;
};
}  // namespace pio

struct pio_assoc_index {
  int device = 0, n_items = 0, n_levels = 0;
  std::vector<int64_t> level_off;                  // [n_levels + 1]
  std::vector<uint8_t> frequent;                   // per item: it has a level-1 set (sizes a call's parts on the host)
  std::vector<int64_t> set_prefix, rule_cond;      // host copies until the first call uploads them
  std::vector<int32_t> set_item;
  int64_t n_sets = 0, n_rules = 0;
  cudaStream_t st = nullptr;
  bool uploaded = false;
  long long *d_prefix = nullptr, *d_rule_lo = nullptr, *d_rule_hi = nullptr;
  int *d_item = nullptr, *d_child_lo = nullptr, *d_child_hi = nullptr, *d_item_set = nullptr;
  std::mutex mu;                                   // serialises the calls
  bool has_result = false;                         // the last call's result, until pio_assoc_predict_get takes it
  pio::ApResult res;
};

namespace pio {

// what the last pio_assoc_predict on this thread did (pio_assoc_predict_debug_stats)
struct AssocPredictStats {
  long long parts = 0, max_part_queries = 0, budget = 0, conds = 0;
  double device_ms = 0.0;
  long long entries[33] = {};   // frontier entries (frequent sets found inside the queries) per level 1 .. 32
};
static thread_local AssocPredictStats g_ap_stats;

static void ap_free_device(pio_assoc_index* ix) {
  for (void* p : {(void*)ix->d_prefix, (void*)ix->d_rule_lo, (void*)ix->d_rule_hi, (void*)ix->d_item,
                  (void*)ix->d_child_lo, (void*)ix->d_child_hi, (void*)ix->d_item_set})
    if (p) cudaFree(p);
  ix->d_prefix = ix->d_rule_lo = ix->d_rule_hi = nullptr;
  ix->d_item = ix->d_child_lo = ix->d_child_hi = ix->d_item_set = nullptr;
}

// The device copy and the derived ranges, made on the index's stream by the first call; published only once they have
// all landed, so a failed upload leaves nothing half made and the next call starts over.
static int ap_upload(pio_assoc_index* ix, const FilterEnv& env) {
  if (ix->uploaded) return PIO_ALS_OK;
  if (!ix->st) CKF(env, cudaStreamCreateWithFlags(&ix->st, cudaStreamNonBlocking));
  const size_t ns = (size_t)std::max<int64_t>(ix->n_sets, 1), nr = (size_t)std::max<int64_t>(ix->n_rules, 1);
  cudaStream_t st = ix->st;
  cudaError_t e = cudaSuccess;
  auto step = [&e](cudaError_t r) {
    if (e == cudaSuccess) e = r;
  };
  long long* d_cond = nullptr;
  step(cudaMalloc((void**)&ix->d_prefix, 8 * ns));
  step(cudaMalloc((void**)&ix->d_item, 4 * ns));
  step(cudaMalloc((void**)&ix->d_child_lo, 4 * ns));
  step(cudaMalloc((void**)&ix->d_child_hi, 4 * ns));
  step(cudaMalloc((void**)&ix->d_rule_lo, 8 * ns));
  step(cudaMalloc((void**)&ix->d_rule_hi, 8 * ns));
  step(cudaMalloc((void**)&ix->d_item_set, 4 * (size_t)ix->n_items));
  step(cudaMalloc((void**)&d_cond, 8 * nr));
  if (e == cudaSuccess) {
    step(cudaMemsetAsync(ix->d_child_lo, 0, 4 * ns, st));
    step(cudaMemsetAsync(ix->d_child_hi, 0, 4 * ns, st));
    step(cudaMemsetAsync(ix->d_rule_lo, 0, 8 * ns, st));
    step(cudaMemsetAsync(ix->d_rule_hi, 0, 8 * ns, st));
    step(cudaMemsetAsync(ix->d_item_set, 0xff, 4 * (size_t)ix->n_items, st));   // -1: not frequent
  }
  if (e == cudaSuccess && ix->n_sets > 0) {
    step(cudaMemcpyAsync(ix->d_prefix, ix->set_prefix.data(), 8 * (size_t)ix->n_sets, cudaMemcpyHostToDevice, st));
    step(cudaMemcpyAsync(ix->d_item, ix->set_item.data(), 4 * (size_t)ix->n_sets, cudaMemcpyHostToDevice, st));
    const long long n1 = ix->level_off[1], s0 = n1;
    if (e == cudaSuccess) {
      ap_item_set_kernel<<<nblk(n1, 256), 256, 0, st>>>(ix->d_item, n1, ix->d_item_set);
      ++*env.launches;
      if (ix->n_sets > s0) {
        ap_children_kernel<<<nblk(ix->n_sets - s0, 256), 256, 0, st>>>(ix->d_prefix, s0, ix->n_sets, ix->d_child_lo,
                                                                        ix->d_child_hi);
        ++*env.launches;
      }
      step(cudaGetLastError());
    }
  }
  if (e == cudaSuccess && ix->n_rules > 0) {
    step(cudaMemcpyAsync(d_cond, ix->rule_cond.data(), 8 * (size_t)ix->n_rules, cudaMemcpyHostToDevice, st));
    if (e == cudaSuccess) {
      ap_rules_kernel<<<nblk(ix->n_rules, 256), 256, 0, st>>>(d_cond, ix->n_rules, ix->d_rule_lo, ix->d_rule_hi);
      ++*env.launches;
      step(cudaGetLastError());
    }
  }
  step(cudaStreamSynchronize(st));   // the host copies are read until here
  if (d_cond) cudaFree(d_cond);
  if (e != cudaSuccess) {
    cudaStreamSynchronize(st);
    ap_free_device(ix);
    return fail_to(env.err, PIO_ALS_ERR_CUDA, "uploading the association index: %s", cudaGetErrorString(e));
  }
  ix->uploaded = true;
  std::vector<int64_t>().swap(ix->set_prefix);
  std::vector<int64_t>().swap(ix->rule_cond);
  std::vector<int32_t>().swap(ix->set_item);
  return PIO_ALS_OK;
}

// exclusive scan of v[0, n) into pos and the total, read back (synchronises the stream)
static int ap_total(const FilterEnv& env, const uint32_t* v, uint32_t* pos, long long n, long long* total) {
  *total = 0;
  if (n == 0) return PIO_ALS_OK;
  CKF(env, scan_exclusive_u32(v, pos, (size_t)n, env.st, env.launches));
  uint32_t last[2] = {0, 0};
  CKF(env, cudaMemcpyAsync(&last[0], pos + n - 1, 4, cudaMemcpyDeviceToHost, env.st));
  CKF(env, cudaMemcpyAsync(&last[1], v + n - 1, 4, cudaMemcpyDeviceToHost, env.st));
  CKF(env, cudaStreamSynchronize(env.st));
  *total = (long long)last[0] + last[1];
  return PIO_ALS_OK;
}

// the conds of one level of one part, sorted by (query, positions), on the host
struct ApLevel {
  int k = 0;
  std::vector<int32_t> q, items, n;
  std::vector<int64_t> rule;
};

// the frontier of one level: (set, index into L) per entry, in its own device memory
struct ApFrontier {
  std::unique_ptr<Scratch> mem;
  int* set = nullptr;
  uint32_t* t = nullptr;
  long long n = 0;
};

// The queries [j0, j1) of a call: the walk over levels 1 .. K on the device, then each query's conds appended to res
// level by level.
static int ap_part(pio_assoc_index* ix, const FilterEnv& env, const int64_t* q_ptr, const int32_t* q_items,
                   const int32_t* num, int j0, int j1, int K, ApResult* res) {
  cudaStream_t st = env.st;
  const int nq = j1 - j0;
  const long long E = q_ptr[j1] - q_ptr[j0];
  std::vector<long long> rel((size_t)nq + 1);
  long long longest = 1;
  for (int j = 0; j <= nq; ++j) rel[j] = q_ptr[j0 + j] - q_ptr[j0];
  for (int j = 0; j < nq; ++j) longest = std::max(longest, rel[j + 1] - rel[j]);
  const int bits_q = ceil_log2((uint64_t)nq), bits_i = ceil_log2((uint64_t)ix->n_items),
            bits_p = ceil_log2((uint64_t)longest);
  Scratch tmp(st);
  long long* d_ptr = nullptr;
  int *d_items = nullptr, *d_num = nullptr;
  CKF(env, tmp.alloc(&d_ptr, (size_t)nq + 1));
  CKF(env, tmp.alloc(&d_items, (size_t)E));
  CKF(env, tmp.alloc(&d_num, (size_t)nq));
  CKF(env, cudaMemcpyAsync(d_ptr, rel.data(), 8 * rel.size(), cudaMemcpyHostToDevice, st));
  if (E) CKF(env, cudaMemcpyAsync(d_items, q_items + q_ptr[j0], 4 * (size_t)E, cudaMemcpyHostToDevice, st));
  CKF(env, cudaMemcpyAsync(d_num, num + j0, 4 * (size_t)nq, cudaMemcpyHostToDevice, st));
  // L: every query's distinct frequent items sorted by item, with the first position of each; the level-1 frontier
  int *L_q = nullptr, *L_item = nullptr;
  uint32_t *L_pos = nullptr, *L_start = nullptr, *L_end = nullptr;
  ApFrontier f;
  f.mem.reset(new Scratch(st));
  if (E > 0) {
    Scratch lv(st);
    uint32_t *flag = nullptr, *at = nullptr;
    long long U0 = 0;
    CKF(env, lv.alloc(&flag, (size_t)E));
    CKF(env, lv.alloc(&at, (size_t)E));
    int rc = env_launch(env, ap_known_kernel, E, (const int*)d_items, E, ix->n_items, (const int*)ix->d_item_set, flag);
    if (rc) return rc;
    EVF(ap_total(env, flag, at, E, &U0));
    if (U0 > 0) {
      SortBufs sb;
      for (int b = 0; b < 2; ++b) {
        CKF(env, lv.alloc(&sb.k[b], (size_t)U0));
        CKF(env, lv.alloc(&sb.v[b], (size_t)U0));
      }
      rc = env_launch(env, ap_entry_keys_kernel, E, (const int*)d_items, (const long long*)d_ptr, nq, E,
                      (const uint32_t*)flag, (const uint32_t*)at, bits_i, sb.keys(), sb.vals());
      if (rc) return rc;
      CKF(env, radix_sort_pairs(sb, (size_t)U0, bits_q + bits_i, st, env.launches));   // stable: first positions lead
      rc = env_launch(env, ap_first_kernel, U0, (const uint64_t*)sb.keys(), U0, flag);
      if (rc) return rc;
      EVF(ap_total(env, flag, at, U0, &f.n));
      CKF(env, tmp.alloc(&L_q, (size_t)f.n));
      CKF(env, tmp.alloc(&L_item, (size_t)f.n));
      CKF(env, tmp.alloc(&L_pos, (size_t)f.n));
      CKF(env, f.mem->alloc(&f.set, (size_t)f.n));
      CKF(env, f.mem->alloc(&f.t, (size_t)f.n));
      rc = env_launch(env, ap_list_kernel, U0, (const uint64_t*)sb.keys(), (const uint32_t*)sb.vals(), U0,
                      (const uint32_t*)flag, (const uint32_t*)at, bits_i, (const int*)ix->d_item_set, L_q, L_item, L_pos,
                      f.set, f.t);
      if (rc) return rc;
    }
  }
  CKF(env, tmp.alloc(&L_start, (size_t)nq));
  CKF(env, tmp.alloc(&L_end, (size_t)nq));
  CKF(env, cudaMemsetAsync(L_start, 0, 4 * (size_t)nq, st));
  CKF(env, cudaMemsetAsync(L_end, 0, 4 * (size_t)nq, st));
  if (f.n > 0) {
    const int rc = env_launch(env, ap_list_ranges_kernel, f.n, (const int*)L_q, f.n, L_start, L_end);
    if (rc) return rc;
  }
  AssocPredictStats& s = g_ap_stats;
  std::vector<ApLevel> levels;
  for (int k = 1; k <= K && f.n > 0; ++k) {
    s.entries[std::min(k, 32)] += f.n;
    Scratch lv(st);
    uint32_t *has = nullptr, *at = nullptr;
    CKF(env, lv.alloc(&has, (size_t)f.n));
    CKF(env, lv.alloc(&at, (size_t)f.n));
    int rc = env_launch(env, ap_has_rules_kernel, f.n, (const int*)f.set, f.n, (const long long*)ix->d_rule_lo,
                        (const long long*)ix->d_rule_hi, has);
    if (rc) return rc;
    long long R = 0;
    EVF(ap_total(env, has, at, f.n, &R));
    if (R > 0) {
      int *c_set = nullptr, *c_item = nullptr, *o_q = nullptr, *o_item = nullptr, *o_n = nullptr;
      uint32_t *c_t = nullptr, *c_pos = nullptr;
      long long* o_rule = nullptr;
      const size_t Rk = (size_t)R * k;
      CKF(env, lv.alloc(&c_set, (size_t)R));
      CKF(env, lv.alloc(&c_t, (size_t)R));
      CKF(env, lv.alloc(&c_pos, Rk));
      CKF(env, lv.alloc(&c_item, Rk));
      rc = env_launch(env, ap_cond_kernel, f.n, (const int*)f.set, (const uint32_t*)f.t, f.n, k, (const uint32_t*)has,
                      (const uint32_t*)at, (const long long*)ix->d_prefix, (const int*)ix->d_item, (const int*)L_q,
                      (const int*)L_item, (const uint32_t*)L_pos, (const uint32_t*)L_start, c_set, c_t, c_pos, c_item);
      if (rc) return rc;
      // stable LSD passes over the fields (query, position 1, ..., position k), least significant first, as many
      // fields per pass as fit 64 bits: exact for any query length and any k
      SortBufs sb;
      for (int b = 0; b < 2; ++b) {
        CKF(env, lv.alloc(&sb.k[b], (size_t)R));
        CKF(env, lv.alloc(&sb.v[b], (size_t)R));
      }
      rc = env_launch(env, ap_iota_kernel, R, sb.vals(), R);
      if (rc) return rc;
      for (int f1 = k; f1 >= 0;) {
        int f0 = f1, bits = f1 == 0 ? bits_q : bits_p;
        while (f0 > 0 && bits + (f0 - 1 == 0 ? bits_q : bits_p) <= 64) bits += (--f0 == 0 ? bits_q : bits_p);
        rc = env_launch(env, ap_key_kernel, R, (const uint32_t*)sb.vals(), R, k, f0, f1, bits_q, bits_p,
                        (const uint32_t*)c_t, (const int*)L_q, (const uint32_t*)c_pos, sb.keys());
        if (rc) return rc;
        CKF(env, radix_sort_pairs(sb, (size_t)R, bits, st, env.launches));
        f1 = f0 - 1;
      }
      CKF(env, lv.alloc(&o_q, (size_t)R));
      CKF(env, lv.alloc(&o_item, Rk));
      CKF(env, lv.alloc(&o_rule, (size_t)R));
      CKF(env, lv.alloc(&o_n, (size_t)R));
      rc = env_launch(env, ap_emit_kernel, R, (const uint32_t*)sb.vals(), R, k, (const int*)c_set, (const uint32_t*)c_t,
                      (const int*)c_item, (const int*)L_q, (const long long*)ix->d_rule_lo,
                      (const long long*)ix->d_rule_hi, (const int*)d_num, o_q, o_item, o_rule, o_n);
      if (rc) return rc;
      levels.emplace_back();
      ApLevel& l = levels.back();
      l.k = k;
      l.q.resize((size_t)R), l.items.resize(Rk), l.rule.resize((size_t)R), l.n.resize((size_t)R);
      CKF(env, cudaMemcpyAsync(l.q.data(), o_q, 4 * (size_t)R, cudaMemcpyDeviceToHost, st));
      CKF(env, cudaMemcpyAsync(l.items.data(), o_item, 4 * Rk, cudaMemcpyDeviceToHost, st));
      CKF(env, cudaMemcpyAsync(l.rule.data(), o_rule, 8 * (size_t)R, cudaMemcpyDeviceToHost, st));
      CKF(env, cudaMemcpyAsync(l.n.data(), o_n, 4 * (size_t)R, cudaMemcpyDeviceToHost, st));
      CKF(env, cudaStreamSynchronize(st));
    }
    if (k == K) break;
    // the next level: count each entry's extensions, scan, fill
    uint32_t* cnt = has;   // reused: the level's conds are built
    long long G = 0;
    rc = env_launch(env, ap_count_kernel, f.n, (const int*)f.set, (const uint32_t*)f.t, f.n, (const int*)L_q,
                    (const int*)L_item, (const uint32_t*)L_end, (const int*)ix->d_child_lo, (const int*)ix->d_child_hi,
                    (const int*)ix->d_item, cnt);
    if (rc) return rc;
    EVF(ap_total(env, cnt, at, f.n, &G));
    ApFrontier g;
    g.mem.reset(new Scratch(st));
    g.n = G;
    if (G > 0) {
      CKF(env, g.mem->alloc(&g.set, (size_t)G));
      CKF(env, g.mem->alloc(&g.t, (size_t)G));
      rc = env_launch(env, ap_fill_kernel, f.n, (const int*)f.set, (const uint32_t*)f.t, f.n, (const int*)L_q,
                      (const int*)L_item, (const uint32_t*)L_end, (const int*)ix->d_child_lo,
                      (const int*)ix->d_child_hi, (const int*)ix->d_item, (const uint32_t*)at, g.set, g.t);
      if (rc) return rc;
    }
    f = std::move(g);
  }
  // each query's conds: level by level, each level already in (query, positions) order
  std::vector<size_t> cur(levels.size(), 0);
  for (int q = 0; q < nq; ++q) {
    for (size_t li = 0; li < levels.size(); ++li) {
      const ApLevel& l = levels[li];
      for (size_t& c = cur[li]; c < l.q.size() && l.q[c] == q; ++c) {
        res->cond_items.insert(res->cond_items.end(), l.items.begin() + c * l.k, l.items.begin() + (c + 1) * l.k);
        res->cond_ptr.push_back((int64_t)res->cond_items.size());
        res->rule_first.push_back(l.rule[c]);
        res->rule_n.push_back(l.n[c]);
      }
    }
    res->q_cond_ptr[j0 + q + 1] = (int64_t)res->rule_first.size();
  }
  return PIO_ALS_OK;
}

// An upper bound of the frontier entries of a query with f listed frequent ids: sum over k <= K of min(C(f, k), the
// sets of level k).  C(f, k) is exact while it fits 64 bits; beyond that the level's size bounds it.
static unsigned long long ap_bound(const pio_assoc_index* ix, long long f, int K) {
  unsigned long long b = 0;
  unsigned __int128 c = 1;
  bool big = false;
  for (int k = 1; k <= K; ++k) {
    const unsigned long long lk = (unsigned long long)(ix->level_off[k] - ix->level_off[k - 1]);
    if (!big) {
      c = c * (unsigned __int128)(f - k + 1 > 0 ? f - k + 1 : 0) / (unsigned __int128)k;
      big = c > (unsigned __int128)~0ull;
    }
    b += big ? lk : std::min<unsigned long long>((unsigned long long)c, lk);
  }
  return b;
}

static int assoc_predict(pio_assoc_index* ix, int32_t max_cond_len, const int64_t* q_ptr, const int32_t* q_items,
                         int32_t n_queries, const int32_t* num, int64_t* n_conds, int64_t* n_cond_items) {
  ix->has_result = false;
  ix->res = ApResult();
  if (n_queries < 0 || max_cond_len < 0)
    return fail(nullptr, PIO_ALS_ERR_ARG, "n_queries and max_cond_len must be >= 0");
  if (!n_conds || !n_cond_items || (n_queries > 0 && (!q_ptr || !num)))
    return fail(nullptr, PIO_ALS_ERR_ARG, "null argument");
  if (n_queries > 0 && q_ptr[0] < 0) return fail(nullptr, PIO_ALS_ERR_ARG, "q_ptr must be non-decreasing offsets from 0");
  for (int j = 0; j < n_queries; ++j) {
    const long long len = q_ptr[j + 1] - q_ptr[j];
    if (len < 0) return fail(nullptr, PIO_ALS_ERR_ARG, "q_ptr decreases at query %d", j);
    if (len > 0 && !q_items) return fail(nullptr, PIO_ALS_ERR_ARG, "null q_items");
    if (len >= (1ll << 31)) return fail(nullptr, PIO_ALS_ERR_ARG, "query %d lists 2^31 or more ids", j);
  }
  const int K = std::min(max_cond_len, ix->n_levels);
  // PIO_ASSOC_PREDICT_BUDGET: entries per part (listed ids plus the bound of frontier entries); capped so that a part's
  // entries are numbered in 32 bits
  const char* env_b = getenv("PIO_ASSOC_PREDICT_BUDGET");
  const long long budget = std::min<long long>(env_b && atoll(env_b) > 0 ? atoll(env_b) : PIO_ASSOC_PREDICT_BUDGET,
                                               (1ll << 32) - 1);
  std::vector<int> first;
  long long acc = 0;
  for (int j = 0; j < n_queries; ++j) {
    long long freq = 0;
    for (int64_t e = q_ptr[j]; e < q_ptr[j + 1]; ++e) {
      const int32_t it = q_items[e];
      freq += it >= 0 && it < ix->n_items && ix->frequent[it];
    }
    const unsigned long long w = (unsigned long long)(q_ptr[j + 1] - q_ptr[j]) + ap_bound(ix, freq, K);
    if (w >= (1ull << 32))
      return fail(nullptr, PIO_ALS_ERR_ARG,
                  "query %d may find %llu frequent sets inside its %lld ids: at most 2^32 - 1 fit one part", j, w,
                  (long long)(q_ptr[j + 1] - q_ptr[j]));
    if (j == 0 || acc + (long long)w > budget) {
      first.push_back(j);
      acc = 0;
    }
    acc += (long long)w;
  }
  first.push_back(n_queries);
  AssocPredictStats& s = g_ap_stats;
  s.budget = budget;
  ApResult res;   // moved onto ix on success
  res.q_cond_ptr.assign((size_t)n_queries + 1, 0);
  if (n_queries > 0 && K > 0) {
    CK0(cudaSetDevice(ix->device));
    int64_t launches = 0;
    const FilterEnv env0{nullptr, ix->n_items, &launches, &g_create_error};
    EVF(ap_upload(ix, env0));
    FilterEnv env = env0;
    env.st = ix->st;
    cudaEvent_t ev[2] = {nullptr, nullptr};
    CK0(cudaEventCreate(&ev[0]));
    const cudaError_t e1 = cudaEventCreate(&ev[1]);
    if (e1 != cudaSuccess) {
      cudaEventDestroy(ev[0]);
      CK0(e1);
    }
    struct Events {
      cudaEvent_t* e;
      ~Events() { cudaEventDestroy(e[0]), cudaEventDestroy(e[1]); }
    } own{ev};
    CK0(cudaEventRecord(ev[0], ix->st));
    for (size_t p = 0; p + 1 < first.size(); ++p) {
      const int j0 = first[p], j1 = first[p + 1];
      s.parts += 1;
      s.max_part_queries = std::max<long long>(s.max_part_queries, j1 - j0);
      EVF(ap_part(ix, env, q_ptr, q_items, num, j0, j1, K, &res));
    }
    CK0(cudaEventRecord(ev[1], ix->st));
    CK0(cudaEventSynchronize(ev[1]));
    float ms = 0.f;
    CK0(cudaEventElapsedTime(&ms, ev[0], ev[1]));
    s.device_ms = ms;
  }
  res.cond_ptr.insert(res.cond_ptr.begin(), 0);
  s.conds = (long long)res.rule_first.size();
  *n_conds = (int64_t)res.rule_first.size();
  *n_cond_items = (int64_t)res.cond_items.size();
  ix->res = std::move(res);
  ix->has_result = true;
  return PIO_ALS_OK;
}

}  // namespace pio

extern "C" {

int pio_assoc_index_create(int device, int32_t n_items, int32_t n_levels, const int64_t* level_off,
                           const int64_t* set_prefix, const int32_t* set_item, int64_t n_rules,
                           const int64_t* rule_cond, pio_assoc_index** out) {
  if (!out || n_items < 1 || n_levels < 0 || !level_off || n_rules < 0 || (n_rules > 0 && !rule_cond))
    return fail(nullptr, PIO_ALS_ERR_ARG, "bad pio_assoc_index_create arguments");
  *out = nullptr;
  if (level_off[0] != 0) return fail(nullptr, PIO_ALS_ERR_ARG, "level_off[0] must be 0");
  for (int l = 0; l < n_levels; ++l)
    if (level_off[l + 1] < level_off[l]) return fail(nullptr, PIO_ALS_ERR_ARG, "level_off decreases at level %d", l + 1);
  const int64_t n_sets = level_off[n_levels];
  if (n_sets >= (1ll << 31)) return fail(nullptr, PIO_ALS_ERR_ARG, "%lld sets: at most 2^31 - 1", (long long)n_sets);
  if (n_sets > 0 && (!set_prefix || !set_item)) return fail(nullptr, PIO_ALS_ERR_ARG, "null set arrays");
  std::vector<uint8_t> frequent;
  try {
    frequent.assign((size_t)n_items, 0);
  } catch (const std::bad_alloc&) {
    return fail(nullptr, PIO_ALS_ERR_NOMEM, "pio_assoc_index_create: out of host memory");
  }
  for (int64_t s = 0; n_levels > 0 && s < level_off[1]; ++s)
    if (set_item[s] >= 0 && set_item[s] < n_items) frequent[set_item[s]] = 1;
  // the trie: level 1 holds distinct items ascending; a set of level l >= 2 extends a set of level l - 1 by a larger
  // frequent item, with prefixes non-decreasing and, under one prefix, items ascending
  for (int l = 1; l <= n_levels; ++l)
    for (int64_t s = level_off[l - 1]; s < level_off[l]; ++s) {
      const int64_t p = set_prefix[s];
      const int32_t it = set_item[s];
      if (it < 0 || it >= n_items || !frequent[it])
        return fail(nullptr, PIO_ALS_ERR_ARG, "set %lld: item %d is not a level-1 item in [0, %d)", (long long)s, it,
                    n_items);
      if (l == 1 ? p != -1 : (p < level_off[l - 2] || p >= level_off[l - 1]))
        return fail(nullptr, PIO_ALS_ERR_ARG, "set %lld: prefix %lld is not a set of level %d", (long long)s,
                    (long long)p, l - 1);
      const bool same = s > level_off[l - 1] && set_prefix[s - 1] == p;
      if ((s > level_off[l - 1] && set_prefix[s - 1] > p) || (same && set_item[s - 1] >= it))
        return fail(nullptr, PIO_ALS_ERR_ARG, "set %lld is out of lexicographic order", (long long)s);
      if (l > 1 && set_item[p] >= it)
        return fail(nullptr, PIO_ALS_ERR_ARG, "set %lld: item %d is not larger than its prefix's", (long long)s, it);
    }
  for (int64_t r = 0; r < n_rules; ++r)
    if (rule_cond[r] < 0 || rule_cond[r] >= n_sets || (r > 0 && rule_cond[r] < rule_cond[r - 1]))
      return fail(nullptr, PIO_ALS_ERR_ARG, "rule %lld: cond %lld is not a set index grouped in set order",
                  (long long)r, (long long)rule_cond[r]);
  std::unique_ptr<pio_assoc_index> ix;
  try {   // bad_alloc must not cross the C boundary
    ix.reset(new pio_assoc_index);
    ix->device = device, ix->n_items = n_items, ix->n_levels = n_levels, ix->n_sets = n_sets, ix->n_rules = n_rules;
    ix->level_off.assign(level_off, level_off + n_levels + 1);
    ix->set_prefix.assign(set_prefix, set_prefix + n_sets);
    ix->set_item.assign(set_item, set_item + n_sets);
    ix->rule_cond.assign(rule_cond, rule_cond + n_rules);
    ix->frequent.swap(frequent);
  } catch (const std::bad_alloc&) {
    return fail(nullptr, PIO_ALS_ERR_NOMEM, "pio_assoc_index_create: out of host memory");
  }
  *out = ix.release();
  return PIO_ALS_OK;
}

int pio_assoc_index_destroy(pio_assoc_index* ix) {
  if (!ix) return PIO_ALS_OK;
  if (ix->st) {
    cudaSetDevice(ix->device);
    cudaStreamSynchronize(ix->st);
    cudaStreamDestroy(ix->st);
  }
  ap_free_device(ix);
  delete ix;
  return PIO_ALS_OK;
}

int pio_assoc_predict(pio_assoc_index* ix, int32_t max_cond_len, const int64_t* q_ptr, const int32_t* q_items,
                      int32_t n_queries, const int32_t* num, int64_t* n_conds, int64_t* n_cond_items) {
  g_ap_stats = AssocPredictStats{};
  if (!ix) return fail(nullptr, PIO_ALS_ERR_ARG, "null association index");
  std::lock_guard<std::mutex> lk(ix->mu);
  try {   // bad_alloc must not cross the C boundary; Scratch releases a part's device memory on the way out
    return assoc_predict(ix, max_cond_len, q_ptr, q_items, n_queries, num, n_conds, n_cond_items);
  } catch (const std::bad_alloc&) {
    return fail(nullptr, PIO_ALS_ERR_NOMEM, "pio_assoc_predict: out of host memory");
  }
}

int pio_assoc_predict_get(pio_assoc_index* ix, int64_t* q_cond_ptr, int64_t* cond_ptr, int32_t* cond_items,
                          int64_t* rule_first, int32_t* rule_n) {
  if (!ix) return fail(nullptr, PIO_ALS_ERR_ARG, "null association index");
  std::lock_guard<std::mutex> lk(ix->mu);
  if (!ix->has_result) return fail(nullptr, PIO_ALS_ERR_STATE, "no pio_assoc_predict result to get");
  auto put = [](auto* dst, auto& v) {
    if (dst && !v.empty()) memcpy(dst, v.data(), v.size() * sizeof(v[0]));
    std::remove_reference_t<decltype(v)>().swap(v);
  };
  put(q_cond_ptr, ix->res.q_cond_ptr);
  put(cond_ptr, ix->res.cond_ptr);
  put(cond_items, ix->res.cond_items);
  put(rule_first, ix->res.rule_first);
  put(rule_n, ix->res.rule_n);
  ix->has_result = false;
  return PIO_ALS_OK;
}

int pio_assoc_predict_debug_stats(double out[40]) {
  if (!out) return PIO_ALS_ERR_ARG;
  const AssocPredictStats& s = g_ap_stats;
  out[0] = (double)s.parts, out[1] = (double)s.max_part_queries, out[2] = (double)s.budget, out[3] = (double)s.conds;
  out[4] = s.device_ms;
  for (int j = 5; j < 8; ++j) out[j] = 0;
  for (int k = 1; k <= 32; ++k) out[7 + k] = (double)s.entries[k];   // out[8 .. 39]
  return PIO_ALS_OK;
}

}  // extern "C"

// ---- text classification (pio_text_*) -----------------------------------------------------------------------------------
struct pio_text_model {
  int device = 0, n_gram = 1, num_features = 1, n_stop = 0, n_class = 0;
  unsigned stop_mask = 0;
  cudaStream_t st = nullptr;
  int* d_slot = nullptr;
  uint8_t* d_stop = nullptr;
  long long* d_stop_off = nullptr;
  double *d_idf = nullptr, *d_pi = nullptr, *d_theta = nullptr;
  int* d_nonfinite = nullptr;
  std::mutex mu;                                   // serialises the calls
  bool has_features = false;                       // the last pio_text_features result, until _get takes it
  std::vector<int64_t> f_ptr;
  std::vector<int32_t> f_idx;
  std::vector<double> f_val;
};

namespace pio {

// what the last pio_text_* call on this thread did (pio_text_debug_stats)
struct TextStats {
  long long parts = 0, docs = 0, windows = 0, entries = 0, max_part_bytes = 0, budget = 0;
  double device_ms = 0.0;
};
static thread_local TextStats g_tx_stats;

// One part's (document, index, count) entries, in (document, index) order; documents local to the part.
struct TxEntries {
  uint32_t *doc = nullptr, *idx = nullptr, *cnt = nullptr;
  long long n = 0;
};

static int tx_check_tokens(const uint8_t* tok_bytes, const int64_t* tok_off, int32_t n) {
  if (n < 0) return fail(nullptr, PIO_ALS_ERR_ARG, "n_docs must be >= 0");
  if (!tok_off || (n > 0 && !tok_bytes)) return fail(nullptr, PIO_ALS_ERR_ARG, "null token argument");
  if (tok_off[0] < 0) return fail(nullptr, PIO_ALS_ERR_ARG, "tok_off[0] must be >= 0");
  for (int d = 0; d < n; ++d) {
    const long long len = tok_off[d + 1] - tok_off[d];
    if (len < 0) return fail(nullptr, PIO_ALS_ERR_ARG, "tok_off decreases at document %d", d);
    if (len >= (1ll << 31)) return fail(nullptr, PIO_ALS_ERR_ARG, "document %d: a token holds fewer than 2^31 bytes", d);
    if (len < 2 || tok_bytes[tok_off[d]] != '"' || tok_bytes[tok_off[d + 1] - 1] != '"')
      return fail(nullptr, PIO_ALS_ERR_ARG, "document %d is not a JSON string token", d);
  }
  return PIO_ALS_OK;
}

static std::vector<TextPart> tx_plan(const int64_t* tok_off, int32_t n) {
  // PIO_TEXT_BUDGET: raw token bytes per part; capped so that a part's bytes are numbered in 31 bits
  const char* env_b = getenv("PIO_TEXT_BUDGET");
  const long long budget = std::min<long long>(env_b && atoll(env_b) > 0 ? atoll(env_b) : PIO_TEXT_BUDGET,
                                               (1ll << 31) - 1);
  g_tx_stats.budget = budget;
  return plan_text(tok_off, n, budget);
}

// The entries of part p: decode, split, stop words, n-gram hashes, the sort and its runs.  The entries go into `keep`
// (they outlive the part); everything else is released when the part returns.
static int tx_part(pio_text_model* m, Scratch& keep, const uint8_t* tok_bytes, const int64_t* tok_off,
                   const TextPart& p, TxEntries* out) {
  cudaStream_t st = m->st;
  const int nd = p.d1 - p.d0;
  const long long nb = p.b1 - p.b0;
  TextStats& s = g_tx_stats;
  s.parts += 1, s.docs += nd, s.max_part_bytes = std::max(s.max_part_bytes, nb);
  std::vector<long long> off((size_t)nd + 1);
  for (int j = 0; j <= nd; ++j) off[j] = tok_off[p.d0 + j] - p.b0;
  Scratch tmp(st);
  uint8_t *d_raw = nullptr, *d_dec = nullptr;
  long long* d_off = nullptr;
  uint32_t *d_tb = nullptr, *d_tn = nullptr, *d_ntok = nullptr, *d_nwin = nullptr, *d_woff = nullptr;
  CK0(tmp.alloc(&d_raw, (size_t)nb));
  CK0(tmp.alloc(&d_dec, (size_t)nb));
  CK0(tmp.alloc(&d_off, (size_t)nd + 1));
  CK0(tmp.alloc(&d_tb, (size_t)nb));
  CK0(tmp.alloc(&d_tn, (size_t)nb));
  CK0(tmp.alloc(&d_ntok, (size_t)nd));
  CK0(tmp.alloc(&d_nwin, (size_t)nd));
  CK0(tmp.alloc(&d_woff, (size_t)nd));
  CK0(cudaMemcpyAsync(d_raw, tok_bytes + p.b0, (size_t)nb, cudaMemcpyHostToDevice, st));
  CK0(cudaMemcpyAsync(d_off, off.data(), sizeof(long long) * off.size(), cudaMemcpyHostToDevice, st));
  const TxStop stop{m->d_slot, m->d_stop, m->d_stop_off, m->stop_mask, m->n_stop};
  tx_split_kernel<<<nblk(nd, 256), 256, 0, st>>>(d_raw, d_off, nd, stop, m->n_gram, d_dec, d_tb, d_tn, d_ntok, d_nwin);
  CK0(cudaGetLastError());
  CK0(scan_exclusive_u32(d_nwin, d_woff, (size_t)nd, st, nullptr));
  uint32_t last[2] = {0, 0};
  CK0(cudaMemcpyAsync(&last[0], d_woff + nd - 1, 4, cudaMemcpyDeviceToHost, st));
  CK0(cudaMemcpyAsync(&last[1], d_nwin + nd - 1, 4, cudaMemcpyDeviceToHost, st));
  CK0(cudaStreamSynchronize(st));
  const long long W = (long long)last[0] + last[1];
  s.windows += W;
  out->n = 0;
  if (W == 0) return PIO_ALS_OK;
  SortBufs sb;
  for (int b = 0; b < 2; ++b) {
    CK0(tmp.alloc(&sb.k[b], (size_t)W));
    CK0(tmp.alloc(&sb.v[b], (size_t)W));
  }
  const int fbits = ceil_log2((uint64_t)m->num_features), dbits = ceil_log2((uint64_t)nd);
  tx_hash_kernel<<<nblk(W, 256), 256, 0, st>>>(d_dec, d_off, d_tb, d_tn, d_ntok, d_woff, nd, W, m->n_gram,
                                               m->num_features, fbits, sb.keys(), sb.vals());
  CK0(cudaGetLastError());
  CK0(radix_sort_pairs(sb, (size_t)W, fbits + dbits, st, nullptr));
  uint32_t *d_flag = nullptr, *d_rid = nullptr;
  CK0(tmp.alloc(&d_flag, (size_t)W));
  CK0(tmp.alloc(&d_rid, (size_t)W));
  tx_head_flag_kernel<<<nblk(W, 256), 256, 0, st>>>(sb.keys(), W, d_flag);
  CK0(cudaGetLastError());
  CK0(scan_exclusive_u32(d_flag, d_rid, (size_t)W, st, nullptr));
  CK0(cudaMemcpyAsync(&last[0], d_rid + W - 1, 4, cudaMemcpyDeviceToHost, st));
  CK0(cudaMemcpyAsync(&last[1], d_flag + W - 1, 4, cudaMemcpyDeviceToHost, st));
  CK0(cudaStreamSynchronize(st));
  const long long nu = (long long)last[0] + last[1];
  uint32_t* d_start = nullptr;
  CK0(tmp.alloc(&d_start, (size_t)nu));
  CK0(keep.alloc(&out->doc, (size_t)nu));
  CK0(keep.alloc(&out->idx, (size_t)nu));
  CK0(keep.alloc(&out->cnt, (size_t)nu));
  tx_head_kernel<<<nblk(W, 256), 256, 0, st>>>(sb.keys(), d_flag, d_rid, W, d_start);
  tx_entry_kernel<<<nblk(nu, 256), 256, 0, st>>>(sb.keys(), d_start, nu, W, fbits, out->doc, out->idx, out->cnt);
  CK0(cudaGetLastError());
  out->n = nu;
  s.entries += nu;
  return PIO_ALS_OK;
}

// device time of a call: one event pair on the model's stream
struct TxTimer {
  cudaEvent_t ev[2] = {nullptr, nullptr};
  ~TxTimer() {
    if (ev[0]) cudaEventDestroy(ev[0]);
    if (ev[1]) cudaEventDestroy(ev[1]);
  }
  int start(cudaStream_t st) {
    CK0(cudaEventCreate(&ev[0]));
    CK0(cudaEventCreate(&ev[1]));
    CK0(cudaEventRecord(ev[0], st));
    return PIO_ALS_OK;
  }
  int stop(cudaStream_t st) {
    CK0(cudaEventRecord(ev[1], st));
    CK0(cudaEventSynchronize(ev[1]));
    float ms = 0.f;
    CK0(cudaEventElapsedTime(&ms, ev[0], ev[1]));
    g_tx_stats.device_ms = ms;
    return PIO_ALS_OK;
  }
};

// One list of training entries: feature index, term count and class per entry (any order).
struct TxTrainList {
  const uint32_t *idx = nullptr, *cnt = nullptr;
  const int* cls = nullptr;
  long long n = 0;
};

// IDF.fit with minDocFreq 0 over m documents: log((m + 1) / (df + 1)), the division first
static void tx_idf(long long m, const int64_t* df, long long D, double* idf) {
  for (long long j = 0; j < D; ++j) idf[j] = log(((double)m + 1.0) / ((double)df[j] + 1.0));
}

// multinomial NaiveBayes from the rounded class sums s (in theta, overwritten) of m documents, n_c of class c:
// pi_c = log(n_c + l) - log(m + C l); theta_cj = log(s_cj + l) - log(sum_j s_cj + D l), the sum in j order
static void tx_nb_logs(long long m, const std::vector<long long>& n_c, double lambda, long long D, double* pi,
                       double* theta) {
  const int n_class = (int)n_c.size();
  const double logden = log((double)m + n_class * lambda);
  for (int c = 0; c < n_class; ++c) {
    pi[c] = log((double)n_c[c] + lambda) - logden;
    double* row = theta + (long long)c * D;
    double tot = 0.0;
    for (long long j = 0; j < D; ++j) tot += row[j];
    const double lt = log(tot + (double)D * lambda);
    for (long long j = 0; j < D; ++j) row[j] = log(row[j] + lambda) - lt;
  }
}

// per class: the entries of theta [C x D] that are not finite (tx_score_kernel's NaN rule)
static std::vector<int> tx_nonfinite(const double* theta, int n_class, long long D) {
  std::vector<int> nonfinite((size_t)n_class, 0);
  for (long long t = 0; t < (long long)n_class * D; ++t) nonfinite[t / D] += !std::isfinite(theta[t]);
  return nonfinite;
}

// IDF.fit and NaiveBayes.train over the entries of m training documents (n_c per class), with the timer started by the
// caller: df on the device, idf on the host, the exact class sums on the device, the logarithms on the host.
static int tx_fit(cudaStream_t st, Scratch& keep, TxTimer& timer, const std::vector<TxTrainList>& lists, long long m,
                  const std::vector<long long>& n_c, double lambda, long long D, int64_t* out_df, double* out_idf,
                  double* out_pi, double* out_theta) {
  const long long CD = (long long)n_c.size() * D;
  unsigned long long* d_df = nullptr;
  CK0(keep.alloc(&d_df, (size_t)D));
  CK0(cudaMemsetAsync(d_df, 0, sizeof(unsigned long long) * (size_t)D, st));
  long long total = 0;
  for (const TxTrainList& l : lists) {
    if (l.n) tx_df_kernel<<<nblk(l.n, 256), 256, 0, st>>>(l.idx, l.n, d_df);
    CK0(cudaGetLastError());
    total += l.n;
  }
  if (total >= (1ll << 33))
    return fail(nullptr, PIO_ALS_ERR_NUMERIC, "%lld (document, feature) entries: the exact class sums hold fewer "
                "than 2^33", total);
  CK0(cudaMemcpyAsync(out_df, d_df, sizeof(int64_t) * (size_t)D, cudaMemcpyDeviceToHost, st));
  CK0(cudaStreamSynchronize(st));
  tx_idf(m, out_df, D, out_idf);
  double* d_idf = nullptr;
  unsigned long long* d_acc = nullptr;
  double* d_s = nullptr;
  int* d_bad = nullptr;
  CK0(keep.alloc(&d_idf, (size_t)D));
  CK0(keep.alloc(&d_acc, (size_t)CD * 3));
  CK0(keep.alloc(&d_s, (size_t)CD));
  CK0(keep.alloc(&d_bad, 1));
  CK0(cudaMemcpyAsync(d_idf, out_idf, sizeof(double) * (size_t)D, cudaMemcpyHostToDevice, st));
  CK0(cudaMemsetAsync(d_acc, 0, sizeof(unsigned long long) * 3 * (size_t)CD, st));
  CK0(cudaMemsetAsync(d_bad, 0, sizeof(int), st));
  for (const TxTrainList& l : lists) {
    if (l.n) tx_sum_kernel<<<nblk(l.n, 256), 256, 0, st>>>(l.idx, l.cnt, l.cls, d_idf, l.n, D, d_acc, d_bad);
    CK0(cudaGetLastError());
  }
  tx_round_kernel<<<nblk(CD, 256), 256, 0, st>>>(d_acc, CD, d_s);
  CK0(cudaGetLastError());
  int bad = 0;
  CK0(cudaMemcpyAsync(&bad, d_bad, sizeof(int), cudaMemcpyDeviceToHost, st));
  CK0(cudaMemcpyAsync(out_theta, d_s, sizeof(double) * (size_t)CD, cudaMemcpyDeviceToHost, st));
  EVF(timer.stop(st));
  if (bad)
    return fail(nullptr, PIO_ALS_ERR_NUMERIC, "a TF-IDF value is outside [2^-44, 2^63): the exact class sums cannot "
                "hold it");
  tx_nb_logs(m, n_c, lambda, D, out_pi, out_theta);
  return PIO_ALS_OK;
}

static int tx_check_fit(int32_t n_class, double lambda) {
  if (n_class < 1) return fail(nullptr, PIO_ALS_ERR_ARG, "n_class must be >= 1");
  if (!(lambda >= 0.0)) return fail(nullptr, PIO_ALS_ERR_ARG, "lambda must be >= 0 (got %g)", lambda);
  return PIO_ALS_OK;
}

static int text_train(pio_text_model* m, const uint8_t* tok_bytes, const int64_t* tok_off, int32_t n,
                      const int32_t* label, int32_t n_class, double lambda, int64_t* out_df, double* out_idf,
                      double* out_pi, double* out_theta) {
  EVF(tx_check_tokens(tok_bytes, tok_off, n));
  if (n < 1) return fail(nullptr, PIO_ALS_ERR_ARG, "training needs at least one document");
  EVF(tx_check_fit(n_class, lambda));
  if (!label || !out_df || !out_idf || !out_pi || !out_theta) return fail(nullptr, PIO_ALS_ERR_ARG, "null argument");
  std::vector<long long> n_c((size_t)n_class, 0);
  for (int d = 0; d < n; ++d) {
    if (label[d] < 0 || label[d] >= n_class)
      return fail(nullptr, PIO_ALS_ERR_ARG, "label %d of document %d is not in [0, %d)", label[d], d, n_class);
    ++n_c[label[d]];
  }
  const std::vector<TextPart> parts = tx_plan(tok_off, n);
  CK0(cudaSetDevice(m->device));
  cudaStream_t st = m->st;
  TxTimer timer;
  EVF(timer.start(st));
  Scratch keep(st);
  std::vector<TxTrainList> lists(parts.size());
  for (size_t k = 0; k < parts.size(); ++k) {
    const TextPart& p = parts[k];
    TxEntries e;
    int* lab = nullptr;
    EVF(tx_part(m, keep, tok_bytes, tok_off, p, &e));
    CK0(keep.alloc(&lab, (size_t)(p.d1 - p.d0)));
    CK0(cudaMemcpyAsync(lab, label + p.d0, sizeof(int) * (size_t)(p.d1 - p.d0), cudaMemcpyHostToDevice, st));
    // the class of each entry, from its document's label, in place of its document
    if (e.n) tx_label_kernel<<<nblk(e.n, 256), 256, 0, st>>>(e.doc, lab, e.n, (int*)e.doc);
    CK0(cudaGetLastError());
    lists[k] = TxTrainList{e.idx, e.cnt, (const int*)e.doc, e.n};
  }
  return tx_fit(st, keep, timer, lists, n, n_c, lambda, m->num_features, out_df, out_idf, out_pi, out_theta);
}

// the entries of every part of a batch, with their values (tf, or tf * idf), handed to `each` part by part
template <class Each>
static int tx_batch(pio_text_model* m, const uint8_t* tok_bytes, const int64_t* tok_off, int32_t n, bool use_idf,
                    Each each) {
  const std::vector<TextPart> parts = tx_plan(tok_off, n);
  cudaStream_t st = m->st;
  TxTimer timer;
  EVF(timer.start(st));
  for (const TextPart& p : parts) {
    Scratch keep(st);
    TxEntries e;
    EVF(tx_part(m, keep, tok_bytes, tok_off, p, &e));
    double* d_val = nullptr;
    CK0(keep.alloc(&d_val, (size_t)e.n));
    if (e.n) tx_value_kernel<<<nblk(e.n, 256), 256, 0, st>>>(e.idx, e.cnt, use_idf ? m->d_idf : nullptr, e.n, d_val);
    CK0(cudaGetLastError());
    EVF(each(p, e, d_val, keep));
  }
  return timer.stop(st);
}

static int text_features(pio_text_model* m, const uint8_t* tok_bytes, const int64_t* tok_off, int32_t n,
                         int32_t use_idf, int64_t* out_nnz) {
  m->has_features = false;
  std::vector<int64_t>().swap(m->f_ptr);
  std::vector<int32_t>().swap(m->f_idx);
  std::vector<double>().swap(m->f_val);
  EVF(tx_check_tokens(tok_bytes, tok_off, n));
  if (!out_nnz) return fail(nullptr, PIO_ALS_ERR_ARG, "null argument");
  if (use_idf && !m->d_idf) return fail(nullptr, PIO_ALS_ERR_STATE, "no idf: the model has not been set");
  std::vector<int64_t> ptr((size_t)n + 1, 0);
  std::vector<int32_t> idx;
  std::vector<double> val;
  if (n > 0) {
    CK0(cudaSetDevice(m->device));
    std::vector<uint32_t> doc;
    EVF(tx_batch(m, tok_bytes, tok_off, n, use_idf != 0, [&](const TextPart& p, const TxEntries& e, double* d_val,
                                                              Scratch&) -> int {
      const size_t at = idx.size();
      doc.resize((size_t)e.n);
      idx.resize(at + (size_t)e.n);
      val.resize(at + (size_t)e.n);
      if (e.n) {
        CK0(cudaMemcpyAsync(doc.data(), e.doc, 4 * (size_t)e.n, cudaMemcpyDeviceToHost, m->st));
        CK0(cudaMemcpyAsync(idx.data() + at, e.idx, 4 * (size_t)e.n, cudaMemcpyDeviceToHost, m->st));
        CK0(cudaMemcpyAsync(val.data() + at, d_val, 8 * (size_t)e.n, cudaMemcpyDeviceToHost, m->st));
      }
      CK0(cudaStreamSynchronize(m->st));
      for (long long u = 0; u < e.n; ++u) ++ptr[(size_t)p.d0 + doc[u] + 1];
      return PIO_ALS_OK;
    }));
    for (int d = 0; d < n; ++d) ptr[d + 1] += ptr[d];
  }
  *out_nnz = (int64_t)idx.size();
  m->f_ptr.swap(ptr), m->f_idx.swap(idx), m->f_val.swap(val);
  m->has_features = true;
  return PIO_ALS_OK;
}

static int text_scores(pio_text_model* m, const uint8_t* tok_bytes, const int64_t* tok_off, int32_t n,
                       double* out_scores) {
  EVF(tx_check_tokens(tok_bytes, tok_off, n));
  if (!out_scores && n > 0) return fail(nullptr, PIO_ALS_ERR_ARG, "null argument");
  if (!m->d_theta) return fail(nullptr, PIO_ALS_ERR_STATE, "no model: pio_text_model_set has not been called");
  if (n == 0) return PIO_ALS_OK;
  CK0(cudaSetDevice(m->device));
  const int C = m->n_class;
  return tx_batch(m, tok_bytes, tok_off, n, true, [&](const TextPart& p, const TxEntries& e, double* d_val,
                                                      Scratch& keep) -> int {
    const int nq = p.d1 - p.d0;
    double* d_out = nullptr;
    CK0(keep.alloc(&d_out, (size_t)nq * C));
    tx_score_kernel<<<nblk((long long)nq * C, 256), 256, 0, m->st>>>(e.doc, e.idx, d_val, e.n, nq, C,
                                                                     m->num_features, m->d_theta, m->d_pi,
                                                                     m->d_nonfinite, d_out);
    CK0(cudaGetLastError());
    CK0(cudaMemcpyAsync(out_scores + (long long)p.d0 * C, d_out, sizeof(double) * (size_t)nq * C,
                        cudaMemcpyDeviceToHost, m->st));
    CK0(cudaStreamSynchronize(m->st));
    return PIO_ALS_OK;
  });
}

static void tx_free_model(pio_text_model* m) {
  for (void* p : {(void*)m->d_idf, (void*)m->d_pi, (void*)m->d_theta, (void*)m->d_nonfinite})
    if (p) cudaFree(p);
  m->d_idf = m->d_pi = m->d_theta = nullptr;
  m->d_nonfinite = nullptr;
  m->n_class = 0;
}

}  // namespace pio

extern "C" {

int pio_text_model_create(int device, const uint8_t* stop_bytes, const int64_t* stop_off, int32_t n_stop,
                          int32_t n_gram, int32_t num_features, pio_text_model** out) {
  if (!out) return fail(nullptr, PIO_ALS_ERR_ARG, "null argument");
  *out = nullptr;
  if (n_gram < 1) return fail(nullptr, PIO_ALS_ERR_ARG, "nGram must be >= 1 (got %d)", n_gram);
  if (num_features < 1) return fail(nullptr, PIO_ALS_ERR_ARG, "numFeatures must be >= 1 (got %d)", num_features);
  if (n_stop < 0 || (n_stop > 0 && (!stop_off || !stop_bytes)))
    return fail(nullptr, PIO_ALS_ERR_ARG, "bad stop words");
  for (int w = 0; w < n_stop; ++w)
    if (stop_off[w + 1] < stop_off[w] || stop_off[w] < 0)
      return fail(nullptr, PIO_ALS_ERR_ARG, "stop_off decreases at word %d", w);
  std::unique_ptr<pio_text_model> m;
  try {   // bad_alloc must not cross the C boundary
    m.reset(new pio_text_model);
    m->device = device, m->n_gram = n_gram, m->num_features = num_features;
    // the stop words, de-duplicated, in an open-addressing set at most half full
    std::vector<long long> off{0};
    std::vector<uint8_t> bytes;
    size_t slots = 2;
    while (slots < 2 * (size_t)n_stop) slots <<= 1;
    std::vector<int> slot(slots, -1);
    const unsigned mask = (unsigned)(slots - 1);
    for (int w = 0; w < n_stop; ++w) {
      const uint8_t* p = stop_bytes + stop_off[w];
      const long long len = stop_off[w + 1] - stop_off[w];
      unsigned i = (unsigned)tx_hash(p, len) & mask;
      bool dup = false;
      for (; slot[i] >= 0; i = (i + 1) & mask) {
        const int v = slot[i];
        if (off[v + 1] - off[v] == len && !memcmp(bytes.data() + off[v], p, (size_t)len)) {
          dup = true;
          break;
        }
      }
      if (dup) continue;
      slot[i] = (int)off.size() - 1;
      bytes.insert(bytes.end(), p, p + len);
      off.push_back((long long)bytes.size());
    }
    m->n_stop = (int)off.size() - 1, m->stop_mask = mask;
    CK0(cudaSetDevice(device));
    CK0(cudaStreamCreateWithFlags(&m->st, cudaStreamNonBlocking));
    std::unique_ptr<pio_text_model, int (*)(pio_text_model*)> guard(m.release(), pio_text_model_destroy);
    pio_text_model* g = guard.get();
    CK0(cudaMalloc((void**)&g->d_slot, sizeof(int) * slots));
    CK0(cudaMalloc((void**)&g->d_stop, std::max<size_t>(bytes.size(), 1)));
    CK0(cudaMalloc((void**)&g->d_stop_off, sizeof(long long) * off.size()));
    CK0(cudaMemcpy(g->d_slot, slot.data(), sizeof(int) * slots, cudaMemcpyHostToDevice));
    if (!bytes.empty()) CK0(cudaMemcpy(g->d_stop, bytes.data(), bytes.size(), cudaMemcpyHostToDevice));
    CK0(cudaMemcpy(g->d_stop_off, off.data(), sizeof(long long) * off.size(), cudaMemcpyHostToDevice));
    *out = guard.release();
  } catch (const std::bad_alloc&) {
    return fail(nullptr, PIO_ALS_ERR_NOMEM, "pio_text_model_create: out of host memory");
  }
  return PIO_ALS_OK;
}

int pio_text_model_destroy(pio_text_model* m) {
  if (!m) return PIO_ALS_OK;
  cudaSetDevice(m->device);
  if (m->st) {
    cudaStreamSynchronize(m->st);
    cudaStreamDestroy(m->st);
  }
  for (void* p : {(void*)m->d_slot, (void*)m->d_stop, (void*)m->d_stop_off})
    if (p) cudaFree(p);
  tx_free_model(m);
  delete m;
  return PIO_ALS_OK;
}

int pio_text_model_set(pio_text_model* m, int32_t n_class, const double* idf, const double* pi, const double* theta) {
  if (!m) return fail(nullptr, PIO_ALS_ERR_ARG, "null text model");
  if (n_class < 1 || !idf || !pi || !theta) return fail(nullptr, PIO_ALS_ERR_ARG, "bad pio_text_model_set arguments");
  std::lock_guard<std::mutex> lk(m->mu);
  try {
    const long long D = m->num_features, CD = (long long)n_class * D;
    const std::vector<int> nonfinite = tx_nonfinite(theta, n_class, D);
    CK0(cudaSetDevice(m->device));
    tx_free_model(m);
    CK0(cudaMalloc((void**)&m->d_idf, sizeof(double) * (size_t)D));
    CK0(cudaMalloc((void**)&m->d_pi, sizeof(double) * (size_t)n_class));
    CK0(cudaMalloc((void**)&m->d_theta, sizeof(double) * (size_t)CD));
    CK0(cudaMalloc((void**)&m->d_nonfinite, sizeof(int) * (size_t)n_class));
    CK0(cudaMemcpy(m->d_idf, idf, sizeof(double) * (size_t)D, cudaMemcpyHostToDevice));
    CK0(cudaMemcpy(m->d_pi, pi, sizeof(double) * (size_t)n_class, cudaMemcpyHostToDevice));
    CK0(cudaMemcpy(m->d_theta, theta, sizeof(double) * (size_t)CD, cudaMemcpyHostToDevice));
    CK0(cudaMemcpy(m->d_nonfinite, nonfinite.data(), sizeof(int) * (size_t)n_class, cudaMemcpyHostToDevice));
    m->n_class = n_class;
  } catch (const std::bad_alloc&) {
    return fail(nullptr, PIO_ALS_ERR_NOMEM, "pio_text_model_set: out of host memory");
  }
  return PIO_ALS_OK;
}

int pio_text_train_nb(pio_text_model* m, const uint8_t* tok_bytes, const int64_t* tok_off, int32_t n_docs,
                      const int32_t* label, int32_t n_class, double lambda, int64_t* out_df, double* out_idf,
                      double* out_pi, double* out_theta) {
  g_tx_stats = TextStats{};
  if (!m) return fail(nullptr, PIO_ALS_ERR_ARG, "null text model");
  std::lock_guard<std::mutex> lk(m->mu);
  try {   // Scratch releases device memory on the way out
    return text_train(m, tok_bytes, tok_off, n_docs, label, n_class, lambda, out_df, out_idf, out_pi, out_theta);
  } catch (const std::bad_alloc&) {
    return fail(nullptr, PIO_ALS_ERR_NOMEM, "pio_text_train_nb: out of host memory");
  }
}

int pio_text_features(pio_text_model* m, const uint8_t* tok_bytes, const int64_t* tok_off, int32_t n_docs,
                      int32_t use_idf, int64_t* out_nnz) {
  g_tx_stats = TextStats{};
  if (!m) return fail(nullptr, PIO_ALS_ERR_ARG, "null text model");
  std::lock_guard<std::mutex> lk(m->mu);
  try {
    return text_features(m, tok_bytes, tok_off, n_docs, use_idf, out_nnz);
  } catch (const std::bad_alloc&) {
    return fail(nullptr, PIO_ALS_ERR_NOMEM, "pio_text_features: out of host memory");
  }
}

int pio_text_features_get(pio_text_model* m, int64_t* doc_ptr, int32_t* index, double* value) {
  if (!m) return fail(nullptr, PIO_ALS_ERR_ARG, "null text model");
  std::lock_guard<std::mutex> lk(m->mu);
  if (!m->has_features) return fail(nullptr, PIO_ALS_ERR_STATE, "no pio_text_features result to get");
  auto put = [](auto* dst, auto& v) {
    if (dst && !v.empty()) memcpy(dst, v.data(), v.size() * sizeof(v[0]));
    std::remove_reference_t<decltype(v)>().swap(v);
  };
  put(doc_ptr, m->f_ptr);
  put(index, m->f_idx);
  put(value, m->f_val);
  m->has_features = false;
  return PIO_ALS_OK;
}

int pio_text_scores(pio_text_model* m, const uint8_t* tok_bytes, const int64_t* tok_off, int32_t n_docs,
                    double* out_scores) {
  g_tx_stats = TextStats{};
  if (!m) return fail(nullptr, PIO_ALS_ERR_ARG, "null text model");
  std::lock_guard<std::mutex> lk(m->mu);
  try {
    return text_scores(m, tok_bytes, tok_off, n_docs, out_scores);
  } catch (const std::bad_alloc&) {
    return fail(nullptr, PIO_ALS_ERR_NOMEM, "pio_text_scores: out of host memory");
  }
}

int pio_text_debug_stats(double out[7]) {
  if (!out) return PIO_ALS_ERR_ARG;
  const TextStats& s = g_tx_stats;
  out[0] = (double)s.parts, out[1] = (double)s.docs, out[2] = (double)s.windows, out[3] = (double)s.entries;
  out[4] = (double)s.max_part_bytes, out[5] = (double)s.budget, out[6] = s.device_ms;
  return PIO_ALS_OK;
}

}  // extern "C"

// ---- k-fold evaluation of the text classification template (pio_text_folds_*; DESIGN.md 4.18.1) ------------------------
struct pio_text_folds {
  int k = 1;
  int32_t n = 0;                                   // documents; document d tests in fold d % k
  std::vector<uint8_t> tok_bytes;                  // the documents' raw tokens, offsets from 0
  std::vector<int64_t> tok_off;
  pio_text_model* fz = nullptr;                    // the stop words, the stream and the featurizer's parameters
  // the current featurization: every entry (global document, index, count) in (document, index) order
  std::unique_ptr<pio::Scratch> ents;
  uint32_t *doc = nullptr, *idx = nullptr, *cnt = nullptr;
  long long nu = 0;
  int n_gram = 0, num_features = 0;                // 0: nothing featurized
  long long featurizations = 0, parts = 0;
  double featurize_ms = 0.0, train_ms = 0.0, scores_ms = 0.0;
};

namespace pio {

static long long tf_n_test(const pio_text_folds* t, int f) { return ((long long)t->n + t->k - 1 - f) / t->k; }

static int tf_fold(const pio_text_folds* t, int32_t fold, const char* what) {
  if (!t) return fail(nullptr, PIO_ALS_ERR_ARG, "%s: null object", what);
  if (fold < 0 || fold >= t->k)
    return fail(nullptr, PIO_ALS_ERR_ARG, "%s: fold %d outside 0..%d", what, fold, t->k - 1);
  if (!t->n_gram) return fail(nullptr, PIO_ALS_ERR_STATE, "%s: pio_text_folds_featurize has not been called", what);
  return PIO_ALS_OK;
}

static int tf_featurize(pio_text_folds* t, int32_t n_gram, int32_t num_features) {
  if (n_gram < 1) return fail(nullptr, PIO_ALS_ERR_ARG, "nGram must be >= 1 (got %d)", n_gram);
  if (num_features < 1) return fail(nullptr, PIO_ALS_ERR_ARG, "numFeatures must be >= 1 (got %d)", num_features);
  if (t->n_gram == n_gram && t->num_features == num_features) return PIO_ALS_OK;
  pio_text_model* m = t->fz;
  t->ents.reset();
  t->doc = t->idx = t->cnt = nullptr;
  t->nu = 0, t->n_gram = 0, t->num_features = 0;
  m->n_gram = n_gram, m->num_features = num_features;
  const std::vector<TextPart> parts = tx_plan(t->tok_off.data(), t->n);
  CK0(cudaSetDevice(m->device));
  cudaStream_t st = m->st;
  TxTimer timer;
  EVF(timer.start(st));
  std::unique_ptr<Scratch> keep(new Scratch(st));
  {
    Scratch part_mem(st);   // the parts' own entries, released once they are copied into one list
    std::vector<TxEntries> pe(parts.size());
    long long total = 0;
    for (size_t q = 0; q < parts.size(); ++q) {
      EVF(tx_part(m, part_mem, t->tok_bytes.data(), t->tok_off.data(), parts[q], &pe[q]));
      total += pe[q].n;
    }
    if (total >= (1ll << 32))
      return fail(nullptr, PIO_ALS_ERR_NUMERIC, "%lld (document, feature) entries: the fold lists hold fewer than "
                  "2^32", total);
    CK0(keep->alloc(&t->doc, (size_t)total));
    CK0(keep->alloc(&t->idx, (size_t)total));
    CK0(keep->alloc(&t->cnt, (size_t)total));
    long long at = 0;
    for (size_t q = 0; q < parts.size(); ++q) {
      const TxEntries& e = pe[q];
      if (!e.n) continue;
      tx_doc_base_kernel<<<nblk(e.n, 256), 256, 0, st>>>(e.doc, e.n, (uint32_t)parts[q].d0, t->doc + at);
      CK0(cudaGetLastError());
      CK0(cudaMemcpyAsync(t->idx + at, e.idx, 4 * (size_t)e.n, cudaMemcpyDeviceToDevice, st));
      CK0(cudaMemcpyAsync(t->cnt + at, e.cnt, 4 * (size_t)e.n, cudaMemcpyDeviceToDevice, st));
      at += e.n;
    }
    t->nu = total;
  }
  EVF(timer.stop(st));
  t->ents = std::move(keep);
  t->n_gram = n_gram, t->num_features = num_features;
  t->featurizations += 1, t->parts = (long long)parts.size(), t->featurize_ms += g_tx_stats.device_ms;
  return PIO_ALS_OK;
}

// fold f's training (test = false) or test list, cut from the resident entries into `tmp`: key (the document's class
// cls_doc[d], or the test position (d - f) / k), index and count per entry, in (document, index) order
static int tf_list(pio_text_folds* t, Scratch& tmp, int f, bool test, const int* d_cls_doc, uint32_t** key,
                   uint32_t** idx, uint32_t** cnt, long long* n_out) {
  cudaStream_t st = t->fz->st;
  const long long nu = t->nu;
  uint32_t *flag = nullptr, *pos = nullptr;
  long long n = 0;
  if (nu) {
    CK0(tmp.alloc(&flag, (size_t)nu));
    CK0(tmp.alloc(&pos, (size_t)nu));
    tx_fold_flag_kernel<<<nblk(nu, 256), 256, 0, st>>>(t->doc, nu, t->k, f, test, flag);
    CK0(cudaGetLastError());
    CK0(scan_exclusive_u32(flag, pos, (size_t)nu, st, nullptr));
    uint32_t last[2] = {0, 0};
    CK0(cudaMemcpyAsync(&last[0], pos + nu - 1, 4, cudaMemcpyDeviceToHost, st));
    CK0(cudaMemcpyAsync(&last[1], flag + nu - 1, 4, cudaMemcpyDeviceToHost, st));
    CK0(cudaStreamSynchronize(st));
    n = (long long)last[0] + last[1];
  }
  CK0(tmp.alloc(key, (size_t)n));
  CK0(tmp.alloc(idx, (size_t)n));
  CK0(tmp.alloc(cnt, (size_t)n));
  if (n) {
    tx_fold_gather_kernel<<<nblk(nu, 256), 256, 0, st>>>(t->doc, t->idx, t->cnt, pos, nu, t->k, f, test, d_cls_doc,
                                                         *key, *idx, *cnt);
    CK0(cudaGetLastError());
  }
  *n_out = n;
  return PIO_ALS_OK;
}

static int tf_train(pio_text_folds* t, int f, const int32_t* cls_doc, int32_t n_class, double lambda, int64_t* out_df,
                    double* out_idf, double* out_pi, double* out_theta) {
  EVF(tx_check_fit(n_class, lambda));
  if (!cls_doc || !out_df || !out_idf || !out_pi || !out_theta) return fail(nullptr, PIO_ALS_ERR_ARG, "null argument");
  const long long m = t->n - tf_n_test(t, f);
  if (m < 1) return fail(nullptr, PIO_ALS_ERR_ARG, "training needs at least one document");
  std::vector<long long> n_c((size_t)n_class, 0);
  for (int d = 0; d < t->n; ++d) {
    if (d % t->k == f) continue;
    if (cls_doc[d] < 0 || cls_doc[d] >= n_class)
      return fail(nullptr, PIO_ALS_ERR_ARG, "class %d of document %d is not in [0, %d)", cls_doc[d], d, n_class);
    ++n_c[cls_doc[d]];
  }
  CK0(cudaSetDevice(t->fz->device));
  cudaStream_t st = t->fz->st;
  TxTimer timer;
  EVF(timer.start(st));
  Scratch tmp(st);
  int* d_cls_doc = nullptr;
  CK0(tmp.alloc(&d_cls_doc, (size_t)t->n));
  CK0(cudaMemcpyAsync(d_cls_doc, cls_doc, sizeof(int) * (size_t)t->n, cudaMemcpyHostToDevice, st));
  TxTrainList l;
  uint32_t *key = nullptr, *idx = nullptr, *cnt = nullptr;
  EVF(tf_list(t, tmp, f, false, d_cls_doc, &key, &idx, &cnt, &l.n));
  l.idx = idx, l.cnt = cnt, l.cls = (const int*)key;
  g_tx_stats.entries = l.n;
  const int rc = tx_fit(st, tmp, timer, {l}, m, n_c, lambda, t->num_features, out_df, out_idf, out_pi, out_theta);
  t->train_ms += g_tx_stats.device_ms;
  return rc;
}

static int tf_scores(pio_text_folds* t, int f, int32_t n_class, const double* idf, const double* pi,
                     const double* theta, double* out) {
  if (n_class < 1 || !idf || !pi || !theta) return fail(nullptr, PIO_ALS_ERR_ARG, "bad pio_text_folds_scores arguments");
  const long long nq = tf_n_test(t, f), D = t->num_features, CD = (long long)n_class * D;
  if (nq == 0) return PIO_ALS_OK;
  if (!out) return fail(nullptr, PIO_ALS_ERR_ARG, "null argument");
  const std::vector<int> nonfinite = tx_nonfinite(theta, n_class, D);
  CK0(cudaSetDevice(t->fz->device));
  cudaStream_t st = t->fz->st;
  TxTimer timer;
  EVF(timer.start(st));
  Scratch tmp(st);
  double *d_idf = nullptr, *d_pi = nullptr, *d_theta = nullptr, *d_val = nullptr, *d_out = nullptr;
  int* d_nonfinite = nullptr;
  CK0(tmp.alloc(&d_idf, (size_t)D));
  CK0(tmp.alloc(&d_pi, (size_t)n_class));
  CK0(tmp.alloc(&d_theta, (size_t)CD));
  CK0(tmp.alloc(&d_nonfinite, (size_t)n_class));
  CK0(tmp.alloc(&d_out, (size_t)(nq * n_class)));
  CK0(cudaMemcpyAsync(d_idf, idf, sizeof(double) * (size_t)D, cudaMemcpyHostToDevice, st));
  CK0(cudaMemcpyAsync(d_pi, pi, sizeof(double) * (size_t)n_class, cudaMemcpyHostToDevice, st));
  CK0(cudaMemcpyAsync(d_theta, theta, sizeof(double) * (size_t)CD, cudaMemcpyHostToDevice, st));
  CK0(cudaMemcpyAsync(d_nonfinite, nonfinite.data(), sizeof(int) * (size_t)n_class, cudaMemcpyHostToDevice, st));
  uint32_t *q = nullptr, *idx = nullptr, *cnt = nullptr;
  long long ne = 0;
  EVF(tf_list(t, tmp, f, true, nullptr, &q, &idx, &cnt, &ne));
  g_tx_stats.entries = ne;
  CK0(tmp.alloc(&d_val, (size_t)ne));
  if (ne) tx_value_kernel<<<nblk(ne, 256), 256, 0, st>>>(idx, cnt, d_idf, ne, d_val);
  CK0(cudaGetLastError());
  tx_score_kernel<<<nblk(nq * n_class, 256), 256, 0, st>>>(q, idx, d_val, ne, (int)nq, n_class, D, d_theta, d_pi,
                                                           d_nonfinite, d_out);
  CK0(cudaGetLastError());
  CK0(cudaMemcpyAsync(out, d_out, sizeof(double) * (size_t)(nq * n_class), cudaMemcpyDeviceToHost, st));
  EVF(timer.stop(st));
  t->scores_ms += g_tx_stats.device_ms;
  return PIO_ALS_OK;
}

}  // namespace pio

extern "C" {

int pio_text_folds_create(int device, const uint8_t* stop_bytes, const int64_t* stop_off, int32_t n_stop,
                          const uint8_t* tok_bytes, const int64_t* tok_off, int32_t n_docs, int32_t k_fold,
                          pio_text_folds** out) {
  g_tx_stats = TextStats{};
  if (!out) return fail(nullptr, PIO_ALS_ERR_ARG, "null argument");
  *out = nullptr;
  EVF(tx_check_tokens(tok_bytes, tok_off, n_docs));
  if (n_docs < 1 || k_fold < 1)
    return fail(nullptr, PIO_ALS_ERR_ARG, "bad pio_text_folds_create arguments (n_docs >= 1 and k_fold >= 1)");
  try {
    std::unique_ptr<pio_text_folds> t(new pio_text_folds);
    t->k = k_fold, t->n = n_docs;
    t->tok_bytes.assign(tok_bytes + tok_off[0], tok_bytes + tok_off[n_docs]);
    t->tok_off.resize((size_t)n_docs + 1);
    for (int d = 0; d <= n_docs; ++d) t->tok_off[d] = tok_off[d] - tok_off[0];
    EVF(pio_text_model_create(device, stop_bytes, stop_off, n_stop, 1, 1, &t->fz));
    *out = t.release();
  } catch (const std::bad_alloc&) {
    return fail(nullptr, PIO_ALS_ERR_NOMEM, "pio_text_folds_create: out of host memory");
  }
  return PIO_ALS_OK;
}

int pio_text_folds_destroy(pio_text_folds* t) {
  if (!t) return PIO_ALS_OK;
  if (t->fz) {
    cudaSetDevice(t->fz->device);
    t->ents.reset();   // frees on the featurizer's stream, which pio_text_model_destroy drains
    pio_text_model_destroy(t->fz);
  }
  delete t;
  return PIO_ALS_OK;
}

int pio_text_folds_featurize(pio_text_folds* t, int32_t n_gram, int32_t num_features) {
  g_tx_stats = TextStats{};
  if (!t) return fail(nullptr, PIO_ALS_ERR_ARG, "null text folds");
  std::lock_guard<std::mutex> lk(t->fz->mu);
  try {
    return tf_featurize(t, n_gram, num_features);
  } catch (const std::bad_alloc&) {
    return fail(nullptr, PIO_ALS_ERR_NOMEM, "pio_text_folds_featurize: out of host memory");
  }
}

int pio_text_folds_sizes(const pio_text_folds* t, int32_t fold, int64_t out[2]) {
  if (!t) return fail(nullptr, PIO_ALS_ERR_ARG, "pio_text_folds_sizes: null object");
  if (fold < 0 || fold >= t->k)
    return fail(nullptr, PIO_ALS_ERR_ARG, "pio_text_folds_sizes: fold %d outside 0..%d", fold, t->k - 1);
  if (!out) return fail(nullptr, PIO_ALS_ERR_ARG, "pio_text_folds_sizes: null out");
  const long long m = tf_n_test(t, fold);
  out[0] = t->n - m, out[1] = m;
  return PIO_ALS_OK;
}

int pio_text_folds_train_nb(pio_text_folds* t, int32_t fold, const int32_t* cls_doc, int32_t n_class, double lambda,
                            int64_t* out_df, double* out_idf, double* out_pi, double* out_theta) {
  g_tx_stats = TextStats{};
  if (!t) return fail(nullptr, PIO_ALS_ERR_ARG, "null text folds");
  std::lock_guard<std::mutex> lk(t->fz->mu);
  EVF(tf_fold(t, fold, "pio_text_folds_train_nb"));
  try {
    return tf_train(t, fold, cls_doc, n_class, lambda, out_df, out_idf, out_pi, out_theta);
  } catch (const std::bad_alloc&) {
    return fail(nullptr, PIO_ALS_ERR_NOMEM, "pio_text_folds_train_nb: out of host memory");
  }
}

int pio_text_folds_scores(pio_text_folds* t, int32_t fold, int32_t n_class, const double* idf, const double* pi,
                          const double* theta, double* out_scores) {
  g_tx_stats = TextStats{};
  if (!t) return fail(nullptr, PIO_ALS_ERR_ARG, "null text folds");
  std::lock_guard<std::mutex> lk(t->fz->mu);
  EVF(tf_fold(t, fold, "pio_text_folds_scores"));
  try {
    return tf_scores(t, fold, n_class, idf, pi, theta, out_scores);
  } catch (const std::bad_alloc&) {
    return fail(nullptr, PIO_ALS_ERR_NOMEM, "pio_text_folds_scores: out of host memory");
  }
}

int pio_text_folds_debug_stats(const pio_text_folds* t, double out[6]) {
  if (!t || !out) return PIO_ALS_ERR_ARG;
  out[0] = (double)t->featurizations, out[1] = (double)t->nu, out[2] = (double)t->parts;
  out[3] = t->featurize_ms, out[4] = t->train_ms, out[5] = t->scores_ms;
  return PIO_ALS_OK;
}

}  // extern "C"

// ---- dimensionality-reduction classification (pio_fr_*; DESIGN.md 4.19) ---------------------------------------------
struct pio_fr_data {
  int device = 0;
  cudaStream_t st = nullptr;
  std::mutex mu;                                   // serialises the calls
  long long n = 0;                                 // rows parsed
  int p = 0, k = 0, n_class = 0;
  bool rows_ok = false;                            // every row parsed and of length p
  double *d_x = nullptr;                           // n x p row-major
  double *d_y = nullptr, *d_yt = nullptr;          // the projected rows: n x k row-major, and k x n
  double* d_sigma = nullptr;                       // [k], after pio_fr_lr_prepare
  int* d_cls = nullptr;                            // [n]
  long long parts = 0, host_rows = 0, lr_evals = 0;
  int slices = 0;
  double parse_ms = 0, gram_ms = 0, project_ms = 0, sigma_ms = 0, lr_ms = 0;
};

struct pio_fr_model {
  int device = 0, p = 0, k = 0, n_label = 0;
  cudaStream_t st = nullptr;
  std::mutex mu;
  double *d_mean = nullptr, *d_a = nullptr, *d_coef = nullptr, *d_b = nullptr;
  long long parts = 0, rows = 0, host_rows = 0;
  double device_ms = 0;
};

namespace pio {

// Double.parseDouble's grammar on one piece [a, b): after String.trim, an optional sign, then NaN, Infinity, a decimal
// significand (digits with an optional point, at least one digit) with an optional exponent, or a hex significand
// (0x / 0X, hex digits with an optional point) with its required binary exponent; then an optional f, F, d or D.  The
// value is strtod's of the piece without its suffix, which is correctly rounded as Java's is.  False: not a double.
static bool fr_java_double(const uint8_t* s, int a, int b, double* v) {
  while (a < b && s[a] <= ' ') ++a;
  while (b > a && s[b - 1] <= ' ') --b;
  if (a >= b) return false;
  const std::string t((const char*)s + a, (size_t)(b - a));
  size_t i = 0;
  const bool neg = t[0] == '-';
  if (t[0] == '+' || t[0] == '-') i = 1;
  const std::string rest = t.substr(i);
  if (rest == "NaN") return *v = std::numeric_limits<double>::quiet_NaN(), true;
  if (rest == "Infinity") return *v = neg ? -HUGE_VAL : HUGE_VAL, true;
  const bool hex = rest.size() >= 2 && rest[0] == '0' && (rest[1] == 'x' || rest[1] == 'X');
  auto digit = [hex](char c) { return hex ? isxdigit((unsigned char)c) != 0 : (c >= '0' && c <= '9'); };
  size_t j = hex ? 2 : 0;
  int digits = 0;
  for (; j < rest.size() && digit(rest[j]); ++j) ++digits;
  if (j < rest.size() && rest[j] == '.')
    for (++j; j < rest.size() && digit(rest[j]); ++j) ++digits;
  if (!digits) return false;
  const bool has_exp = j < rest.size() && (hex ? (rest[j] == 'p' || rest[j] == 'P') : (rest[j] == 'e' || rest[j] == 'E'));
  if (hex && !has_exp) return false;
  if (has_exp) {
    ++j;
    if (j < rest.size() && (rest[j] == '+' || rest[j] == '-')) ++j;
    int ed = 0;
    for (; j < rest.size() && rest[j] >= '0' && rest[j] <= '9'; ++j) ++ed;
    if (!ed) return false;
  }
  const size_t end = j;
  if (j < rest.size() && strchr("fFdD", rest[j])) ++j;
  if (j != rest.size()) return false;
  const std::string num = t.substr(0, i) + rest.substr(0, end);
  *v = strtod(num.c_str(), nullptr);
  return true;
}

// The host's parse of one row (a raw JSON string token of len bytes): its values, and FR_OK, FR_BAD (the first piece
// that is not a double, as map(_.toDouble) throws there), FR_NONFINITE or, when p >= 0, FR_LEN.
static int fr_host_row(const uint8_t* tok, long long len, int p, std::vector<uint8_t>& dec, std::vector<double>& vals) {
  dec.resize((size_t)std::max<long long>(len, 1));
  const int L = ev::decode_string_lenient(tok, 0, (int)len, dec.data());
  const uint8_t* s = dec.data();
  vals.clear();
  if (L == 0) return FR_BAD;                         // "".split(", ") is [""]
  std::vector<std::pair<int, int>> pieces;
  for (int i = 0, start = 0;;) {
    const bool end = i >= L;
    if (end || (s[i] == ',' && i + 1 < L && s[i + 1] == ' ')) {
      pieces.emplace_back(start, i);
      if (end) break;
      i += 2;
      start = i;
    } else {
      ++i;
    }
  }
  while (!pieces.empty() && pieces.back().first == pieces.back().second) pieces.pop_back();   // trailing "" dropped
  bool finite = true;
  for (const auto& pc : pieces) {
    double v;
    if (!fr_java_double(s, pc.first, pc.second, &v)) return FR_BAD;
    finite &= std::isfinite(v) != 0;
    vals.push_back(v);
  }
  if (!finite) return FR_NONFINITE;
  if (p >= 0 && (int)vals.size() != p) return FR_LEN;
  return FR_OK;
}

static int fr_check_tokens(const uint8_t* tok_bytes, const int64_t* tok_off, int32_t n) {
  if (n < 0) return fail(nullptr, PIO_ALS_ERR_ARG, "n_rows must be >= 0");
  if (!tok_off || (n > 0 && !tok_bytes)) return fail(nullptr, PIO_ALS_ERR_ARG, "null token argument");
  if (tok_off[0] < 0) return fail(nullptr, PIO_ALS_ERR_ARG, "tok_off[0] must be >= 0");
  for (int r = 0; r < n; ++r) {
    const long long len = tok_off[r + 1] - tok_off[r];
    if (len < 0) return fail(nullptr, PIO_ALS_ERR_ARG, "tok_off decreases at row %d", r);
    if (len >= (1ll << 31)) return fail(nullptr, PIO_ALS_ERR_ARG, "row %d: a token holds fewer than 2^31 bytes", r);
    if (len < 2 || tok_bytes[tok_off[r]] != '"' || tok_bytes[tok_off[r + 1] - 1] != '"')
      return fail(nullptr, PIO_ALS_ERR_ARG, "row %d is not a JSON string token", r);
  }
  return PIO_ALS_OK;
}

// device milliseconds between two events on a stream
struct FrTimer {
  cudaEvent_t ev[2] = {nullptr, nullptr};
  ~FrTimer() {
    if (ev[0]) cudaEventDestroy(ev[0]);
    if (ev[1]) cudaEventDestroy(ev[1]);
  }
  int start(cudaStream_t st) {
    CK0(cudaEventCreate(&ev[0]));
    CK0(cudaEventCreate(&ev[1]));
    CK0(cudaEventRecord(ev[0], st));
    return PIO_ALS_OK;
  }
  int stop(cudaStream_t st, double* ms_out) {
    CK0(cudaEventRecord(ev[1], st));
    CK0(cudaEventSynchronize(ev[1]));
    float ms = 0.f;
    CK0(cudaEventElapsedTime(&ms, ev[0], ev[1]));
    *ms_out = ms;
    return PIO_ALS_OK;
  }
};

// Parses rows [0, n) into d_x (n x p) part by part: the device's fast path, then the host's parse of the rows it hands
// back.  Status per row into status; *parts and *host_rows counted.
static int fr_parse_rows(cudaStream_t st, const uint8_t* tok_bytes, const int64_t* tok_off, int32_t n, int p,
                         double* d_x, int32_t* status, long long* parts_out, long long* host_out) {
  const char* env_b = getenv("PIO_FR_BUDGET");
  const long long budget = std::min<long long>(env_b && atoll(env_b) > 0 ? atoll(env_b) : (256ll << 20),
                                               (1ll << 31) - 1);
  const std::vector<TextPart> parts = plan_text(tok_off, n, budget);
  std::vector<uint8_t> dec;
  std::vector<double> vals, host_vals;
  for (const TextPart& pt : parts) {
    const int nr = pt.d1 - pt.d0;
    const long long nb = pt.b1 - pt.b0;
    std::vector<long long> off((size_t)nr + 1);
    for (int j = 0; j <= nr; ++j) off[j] = tok_off[pt.d0 + j] - pt.b0;
    Scratch tmp(st);
    uint8_t *d_raw = nullptr, *d_dec = nullptr;
    long long* d_off = nullptr;
    int* d_status = nullptr;
    CK0(tmp.alloc(&d_raw, (size_t)nb));
    CK0(tmp.alloc(&d_dec, (size_t)nb));
    CK0(tmp.alloc(&d_off, (size_t)nr + 1));
    CK0(tmp.alloc(&d_status, (size_t)nr));
    CK0(cudaMemcpyAsync(d_raw, tok_bytes + pt.b0, (size_t)nb, cudaMemcpyHostToDevice, st));
    CK0(cudaMemcpyAsync(d_off, off.data(), sizeof(long long) * off.size(), cudaMemcpyHostToDevice, st));
    double* xp = d_x + (long long)pt.d0 * p;
    fr_parse_kernel<<<nblk(nr, 128), 128, 0, st>>>(d_raw, d_off, nr, p, d_dec, xp, d_status);
    CK0(cudaGetLastError());
    CK0(cudaMemcpyAsync(status + pt.d0, d_status, sizeof(int) * (size_t)nr, cudaMemcpyDeviceToHost, st));
    CK0(cudaStreamSynchronize(st));
    std::vector<int> rows;
    host_vals.clear();
    for (int r = pt.d0; r < pt.d1; ++r) {
      if (status[r] != FR_HOST) continue;
      const int rc = fr_host_row(tok_bytes + tok_off[r], tok_off[r + 1] - tok_off[r], p, dec, vals);
      if (rc != FR_OK) {
        status[r] = rc;
        continue;
      }
      ++*host_out;
      rows.push_back(r);
      host_vals.insert(host_vals.end(), vals.begin(), vals.end());
    }
    for (size_t q = 0; q < rows.size(); ++q)
      CK0(cudaMemcpyAsync(d_x + (long long)rows[q] * p, host_vals.data() + q * p, sizeof(double) * p,
                          cudaMemcpyHostToDevice, st));
    CK0(cudaStreamSynchronize(st));
    ++*parts_out;
  }
  return PIO_ALS_OK;
}

static void fr_free_rows(pio_fr_data* d) {
  for (void* q : {(void*)d->d_x, (void*)d->d_y, (void*)d->d_yt, (void*)d->d_sigma, (void*)d->d_cls})
    if (q) cudaFree(q);
  d->d_x = d->d_y = d->d_yt = d->d_sigma = nullptr;
  d->d_cls = nullptr;
  d->n = 0, d->p = 0, d->k = 0, d->n_class = 0, d->rows_ok = false;
}

static int fr_parse(pio_fr_data* d, const uint8_t* tok_bytes, const int64_t* tok_off, int32_t n, int32_t* status,
                    int32_t* out_p) {
  EVF(fr_check_tokens(tok_bytes, tok_off, n));
  if (n < 1) return fail(nullptr, PIO_ALS_ERR_ARG, "pio_fr_parse needs at least one row");
  if (!status || !out_p) return fail(nullptr, PIO_ALS_ERR_ARG, "null argument");
  CK0(cudaSetDevice(d->device));
  fr_free_rows(d);
  d->parts = d->host_rows = d->lr_evals = 0;
  d->parse_ms = d->gram_ms = d->project_ms = d->sigma_ms = d->lr_ms = 0;
  *out_p = 0;
  for (int r = 0; r < n; ++r) status[r] = FR_OK;
  std::vector<uint8_t> dec;
  std::vector<double> vals;
  const int rc0 = fr_host_row(tok_bytes + tok_off[0], tok_off[1] - tok_off[0], -1, dec, vals);
  if (rc0 != FR_OK) {
    status[0] = rc0;
    return PIO_ALS_OK;
  }
  const long long p = (long long)vals.size();
  if (p < 1 || p > 65535)
    return fail(nullptr, PIO_ALS_ERR_ARG, "row 0 holds %lld values: between 1 and 65535 are supported", p);
  CK0(cudaMalloc((void**)&d->d_x, sizeof(double) * (size_t)n * (size_t)p));
  FrTimer timer;
  EVF(timer.start(d->st));
  EVF(fr_parse_rows(d->st, tok_bytes, tok_off, n, (int)p, d->d_x, status, &d->parts, &d->host_rows));
  EVF(timer.stop(d->st, &d->parse_ms));
  d->n = n, d->p = (int)p, *out_p = (int)p;
  bool ok = true;
  for (int r = 0; r < n; ++r) ok &= status[r] == FR_OK || status[r] == FR_HOST;
  d->rows_ok = ok;
  return PIO_ALS_OK;
}

static int fr_gramian(pio_fr_data* d, double* out_mean, double* out_gram) {
  if (!out_mean || !out_gram) return fail(nullptr, PIO_ALS_ERR_ARG, "null argument");
  if (!d->rows_ok) return fail(nullptr, PIO_ALS_ERR_STATE, "no parsed rows: pio_fr_parse has not succeeded");
  if (d->n < 2) return fail(nullptr, PIO_ALS_ERR_ARG, "the Gramian's mean and covariance need at least 2 rows");
  CK0(cudaSetDevice(d->device));
  cudaStream_t st = d->st;
  const long long n = d->n, p = d->p;
  const FrSlices sl = fr_slices(n, p);
  d->slices = sl.count;
  Scratch tmp(st);
  double *d_part = nullptr, *d_cs = nullptr, *d_g = nullptr;
  CK0(tmp.alloc(&d_part, (size_t)sl.count * p * p));
  CK0(tmp.alloc(&d_cs, (size_t)sl.count * p));
  CK0(tmp.alloc(&d_g, (size_t)p * p));
  FrTimer timer;
  EVF(timer.start(st));
  fr_colsum_kernel<<<dim3(nblk(p, 128), sl.count), 128, 0, st>>>(d->d_x, n, (int)p, sl.rows, d_cs);
  const unsigned T = nblk(p, FR_TILE);
  fr_gram_kernel<<<dim3(T, T, sl.count), 256, 0, st>>>(d->d_x, n, (int)p, sl.rows, d_part);
  fr_gram_fold_kernel<<<nblk(p * p, 256), 256, 0, st>>>(d_part, sl.count, (int)p, d_g);
  CK0(cudaGetLastError());
  std::vector<double> cs((size_t)sl.count * p);
  CK0(cudaMemcpyAsync(cs.data(), d_cs, sizeof(double) * cs.size(), cudaMemcpyDeviceToHost, st));
  CK0(cudaMemcpyAsync(out_gram, d_g, sizeof(double) * (size_t)p * p, cudaMemcpyDeviceToHost, st));
  EVF(timer.stop(st, &d->gram_ms));
  for (long long j = 0; j < p; ++j) {
    double acc = 0.0;
    for (int s = 0; s < sl.count; ++s) acc += cs[(size_t)s * p + j];
    out_mean[j] = acc / (double)n;
  }
  return PIO_ALS_OK;
}

// a = pc^T: k x p row-major from pc p x k row-major
static std::vector<double> fr_components(const double* pc, long long p, long long k) {
  std::vector<double> a((size_t)(p * k));
  for (long long j = 0; j < p; ++j)
    for (long long o = 0; o < k; ++o) a[(size_t)(o * p + j)] = pc[j * k + o];
  return a;
}

static int fr_project(pio_fr_data* d, int32_t k, const double* mean, const double* pc, double* out_y) {
  if (!mean || !pc) return fail(nullptr, PIO_ALS_ERR_ARG, "null argument");
  if (!d->rows_ok) return fail(nullptr, PIO_ALS_ERR_STATE, "no parsed rows: pio_fr_parse has not succeeded");
  if (k < 1 || k > d->p) return fail(nullptr, PIO_ALS_ERR_ARG, "k = %d out of range (0, p = %d]", k, d->p);
  CK0(cudaSetDevice(d->device));
  cudaStream_t st = d->st;
  const long long n = d->n, p = d->p;
  for (double* q : {d->d_y, d->d_yt, d->d_sigma})
    if (q) cudaFree(q);
  d->d_y = d->d_yt = d->d_sigma = nullptr;
  d->k = 0, d->n_class = 0;
  const std::vector<double> a = fr_components(pc, p, k);
  Scratch tmp(st);
  double *d_mean = nullptr, *d_a = nullptr;
  CK0(tmp.alloc(&d_mean, (size_t)p));
  CK0(tmp.alloc(&d_a, a.size()));
  CK0(cudaMalloc((void**)&d->d_y, sizeof(double) * (size_t)(n * k)));
  CK0(cudaMalloc((void**)&d->d_yt, sizeof(double) * (size_t)(n * k)));
  FrTimer timer;
  EVF(timer.start(st));
  CK0(cudaMemcpyAsync(d_mean, mean, sizeof(double) * (size_t)p, cudaMemcpyHostToDevice, st));
  CK0(cudaMemcpyAsync(d_a, a.data(), sizeof(double) * a.size(), cudaMemcpyHostToDevice, st));
  fr_fold_kernel<<<dim3(nblk(n, FR_TILE), nblk(k, FR_TILE)), 256, 0, st>>>(d->d_x, n, (int)p, d_a, k, d_mean, nullptr,
                                                                           d->d_y, k, 1, d->d_yt, 1, n);
  CK0(cudaGetLastError());
  if (out_y) CK0(cudaMemcpyAsync(out_y, d->d_y, sizeof(double) * (size_t)(n * k), cudaMemcpyDeviceToHost, st));
  EVF(timer.stop(st, &d->project_ms));
  d->k = k;
  return PIO_ALS_OK;
}

static int fr_lr_prepare(pio_fr_data* d, const int32_t* cls, int32_t n_class, double* out_sigma) {
  if (!cls || !out_sigma) return fail(nullptr, PIO_ALS_ERR_ARG, "null argument");
  if (!d->k) return fail(nullptr, PIO_ALS_ERR_STATE, "no projected rows: pio_fr_project has not been called");
  if (n_class < 1) return fail(nullptr, PIO_ALS_ERR_ARG, "n_class must be >= 1");
  const long long n = d->n, k = d->k;
  for (long long i = 0; i < n; ++i)
    if (cls[i] < 0 || cls[i] >= n_class)
      return fail(nullptr, PIO_ALS_ERR_ARG, "class %d of row %lld is not in [0, %d)", cls[i], i, n_class);
  CK0(cudaSetDevice(d->device));
  cudaStream_t st = d->st;
  if (d->d_cls) cudaFree(d->d_cls);
  if (d->d_sigma) cudaFree(d->d_sigma);
  d->d_cls = nullptr, d->d_sigma = nullptr, d->n_class = 0;
  CK0(cudaMalloc((void**)&d->d_cls, sizeof(int) * (size_t)n));
  CK0(cudaMalloc((void**)&d->d_sigma, sizeof(double) * (size_t)k));
  const int nb = (int)nblk(n, FR_LR_BLOCK);
  Scratch tmp(st);
  double *d_part = nullptr, *d_sum = nullptr;
  CK0(tmp.alloc(&d_part, (size_t)nb * k));
  CK0(tmp.alloc(&d_sum, (size_t)k));
  FrTimer timer;
  EVF(timer.start(st));
  CK0(cudaMemcpyAsync(d->d_cls, cls, sizeof(int) * (size_t)n, cudaMemcpyHostToDevice, st));
  std::vector<double> s((size_t)k);
  for (int pass = 0; pass < 2; ++pass) {
    fr_lr_colsum_kernel<<<dim3(nb, nblk(k, 128)), 128, 0, st>>>(d->d_y, n, (int)k, pass ? d->d_sigma : nullptr,
                                                                  d_part);
    fr_lr_fold_kernel<<<dim3(nblk(k, 128), 1), 128, 0, st>>>(d_part, nb, (int)k, d_sum);
    CK0(cudaGetLastError());
    CK0(cudaMemcpyAsync(s.data(), d_sum, sizeof(double) * (size_t)k, cudaMemcpyDeviceToHost, st));
    CK0(cudaStreamSynchronize(st));
    for (long long j = 0; j < k; ++j) s[j] = pass ? sqrt(s[j] / (double)(n - 1)) : s[j] / (double)n;
    // the first pass leaves the column means in d_sigma as the centres of the second
    CK0(cudaMemcpyAsync(d->d_sigma, s.data(), sizeof(double) * (size_t)k, cudaMemcpyHostToDevice, st));
    CK0(cudaStreamSynchronize(st));
  }
  EVF(timer.stop(st, &d->sigma_ms));
  memcpy(out_sigma, s.data(), sizeof(double) * (size_t)k);
  d->n_class = n_class;
  return PIO_ALS_OK;
}

static int fr_lr_eval(pio_fr_data* d, int32_t na, const int32_t* labels, const double* wb, double reg, double* out_f,
                      double* out_g) {
  if (!labels || !wb || !out_f || !out_g) return fail(nullptr, PIO_ALS_ERR_ARG, "null argument");
  if (!d->n_class) return fail(nullptr, PIO_ALS_ERR_STATE, "pio_fr_lr_prepare has not been called");
  if (na < 1 || na > 65535) return fail(nullptr, PIO_ALS_ERR_ARG, "n_active must be in [1, 65535] (got %d)", na);
  if (!(reg >= 0.0)) return fail(nullptr, PIO_ALS_ERR_ARG, "reg_param must be >= 0 (got %g)", reg);
  for (int a = 0; a < na; ++a)
    if (labels[a] < 0 || labels[a] >= d->n_class)
      return fail(nullptr, PIO_ALS_ERR_ARG, "label %d of slot %d is not in [0, %d)", labels[a], a, d->n_class);
  CK0(cudaSetDevice(d->device));
  cudaStream_t st = d->st;
  const long long n = d->n, k = d->k, w = k + 2;
  const int nb = (int)nblk(n, FR_LR_BLOCK);
  Scratch tmp(st);
  double *d_wb = nullptr, *d_mult = nullptr, *d_loss = nullptr, *d_part = nullptr, *d_out = nullptr;
  int* d_lab = nullptr;
  CK0(tmp.alloc(&d_wb, (size_t)na * (k + 1)));
  CK0(tmp.alloc(&d_lab, (size_t)na));
  CK0(tmp.alloc(&d_mult, (size_t)na * n));
  CK0(tmp.alloc(&d_loss, (size_t)na * n));
  CK0(tmp.alloc(&d_part, (size_t)na * nb * w));
  CK0(tmp.alloc(&d_out, (size_t)na * w));
  FrTimer timer;
  EVF(timer.start(st));
  CK0(cudaMemcpyAsync(d_wb, wb, sizeof(double) * (size_t)na * (k + 1), cudaMemcpyHostToDevice, st));
  CK0(cudaMemcpyAsync(d_lab, labels, sizeof(int) * (size_t)na, cudaMemcpyHostToDevice, st));
  fr_lr_margin_kernel<<<dim3(nblk(n, 256), na), 256, 0, st>>>(d->d_yt, n, (int)k, d->d_sigma, d->d_cls, d_wb, d_lab,
                                                              d_mult, d_loss);
  fr_lr_grad_kernel<<<dim3(nb, nblk(w, 128), na), 128, 0, st>>>(d->d_y, n, (int)k, d->d_sigma, d_mult, d_loss, nb,
                                                                d_part);
  fr_lr_fold_kernel<<<dim3(nblk(w, 128), na), 128, 0, st>>>(d_part, nb, (int)w, d_out);
  CK0(cudaGetLastError());
  std::vector<double> sums((size_t)na * w);
  CK0(cudaMemcpyAsync(sums.data(), d_out, sizeof(double) * sums.size(), cudaMemcpyDeviceToHost, st));
  double ms = 0;
  EVF(timer.stop(st, &ms));
  d->lr_ms += ms;
  ++d->lr_evals;
  // loss = lossSum / n + 0.5 reg sum_j w_j^2; gradient = sum / n + reg w_j, the intercept's unregularized
  for (int a = 0; a < na; ++a) {
    const double* sa = sums.data() + (size_t)a * w;
    const double* wa = wb + (size_t)a * (k + 1);
    double* ga = out_g + (size_t)a * (k + 1);
    double sq = 0.0;
    for (long long j = 0; j < k; ++j) {
      sq += wa[j] * wa[j];
      ga[j] = sa[j] / (double)n + reg * wa[j];
    }
    ga[k] = sa[k] / (double)n;
    out_f[a] = sa[k + 1] / (double)n + 0.5 * reg * sq;
  }
  return PIO_ALS_OK;
}

static int fr_model_scores(pio_fr_model* m, const uint8_t* tok_bytes, const int64_t* tok_off, int32_t n,
                           int32_t* status, double* out) {
  EVF(fr_check_tokens(tok_bytes, tok_off, n));
  if (n > 0 && (!status || !out)) return fail(nullptr, PIO_ALS_ERR_ARG, "null argument");
  m->parts = m->rows = m->host_rows = 0;
  m->device_ms = 0;
  if (n == 0) return PIO_ALS_OK;
  CK0(cudaSetDevice(m->device));
  cudaStream_t st = m->st;
  const long long p = m->p, k = m->k, L = m->n_label;
  Scratch tmp(st);
  double *d_x = nullptr, *d_y = nullptr, *d_s = nullptr;
  CK0(tmp.alloc(&d_x, (size_t)n * p));
  CK0(tmp.alloc(&d_y, (size_t)n * k));
  CK0(tmp.alloc(&d_s, (size_t)n * L));
  FrTimer timer;
  EVF(timer.start(st));
  EVF(fr_parse_rows(st, tok_bytes, tok_off, n, (int)p, d_x, status, &m->parts, &m->host_rows));
  fr_fold_kernel<<<dim3(nblk(n, FR_TILE), nblk(k, FR_TILE)), 256, 0, st>>>(d_x, n, (int)p, m->d_a, (int)k, m->d_mean,
                                                                           nullptr, d_y, k, 1, nullptr, 0, 0);
  fr_fold_kernel<<<dim3(nblk(n, FR_TILE), nblk(L, FR_TILE)), 256, 0, st>>>(d_y, n, (int)k, m->d_coef, (int)L,
                                                                           nullptr, m->d_b, d_s, L, 1, nullptr, 0, 0);
  CK0(cudaGetLastError());
  CK0(cudaMemcpyAsync(out, d_s, sizeof(double) * (size_t)n * L, cudaMemcpyDeviceToHost, st));
  EVF(timer.stop(st, &m->device_ms));
  m->rows = n;
  return PIO_ALS_OK;
}

}  // namespace pio

extern "C" {

int pio_fr_data_create(int device, pio_fr_data** out) {
  if (!out) return fail(nullptr, PIO_ALS_ERR_ARG, "null argument");
  *out = nullptr;
  try {
    std::unique_ptr<pio_fr_data> d(new pio_fr_data);
    d->device = device;
    CK0(cudaSetDevice(device));
    CK0(cudaStreamCreateWithFlags(&d->st, cudaStreamNonBlocking));
    *out = d.release();
  } catch (const std::bad_alloc&) {
    return fail(nullptr, PIO_ALS_ERR_NOMEM, "pio_fr_data_create: out of host memory");
  }
  return PIO_ALS_OK;
}

int pio_fr_data_destroy(pio_fr_data* d) {
  if (!d) return PIO_ALS_OK;
  cudaSetDevice(d->device);
  if (d->st) cudaStreamSynchronize(d->st);
  fr_free_rows(d);
  if (d->st) cudaStreamDestroy(d->st);
  delete d;
  return PIO_ALS_OK;
}

#define FR_CALL(obj, what, body)                                                      \
  do {                                                                                \
    if (!(obj)) return fail(nullptr, PIO_ALS_ERR_ARG, "%s: null object", what);       \
    std::lock_guard<std::mutex> lk((obj)->mu);                                        \
    try {                                                                             \
      return body;                                                                    \
    } catch (const std::bad_alloc&) {                                                 \
      return fail(nullptr, PIO_ALS_ERR_NOMEM, "%s: out of host memory", what);        \
    }                                                                                 \
  } while (0)

int pio_fr_parse(pio_fr_data* d, const uint8_t* tok_bytes, const int64_t* tok_off, int32_t n_rows,
                 int32_t* out_status, int32_t* out_p) {
  FR_CALL(d, "pio_fr_parse", fr_parse(d, tok_bytes, tok_off, n_rows, out_status, out_p));
}

int pio_fr_gramian(pio_fr_data* d, double* out_mean, double* out_gram) {
  FR_CALL(d, "pio_fr_gramian", fr_gramian(d, out_mean, out_gram));
}

int pio_fr_project(pio_fr_data* d, int32_t k, const double* mean, const double* pc, double* out_y) {
  FR_CALL(d, "pio_fr_project", fr_project(d, k, mean, pc, out_y));
}

int pio_fr_lr_prepare(pio_fr_data* d, const int32_t* cls, int32_t n_class, double* out_sigma) {
  FR_CALL(d, "pio_fr_lr_prepare", fr_lr_prepare(d, cls, n_class, out_sigma));
}

int pio_fr_lr_eval(pio_fr_data* d, int32_t n_active, const int32_t* labels, const double* wb, double reg_param,
                   double* out_f, double* out_g) {
  FR_CALL(d, "pio_fr_lr_eval", fr_lr_eval(d, n_active, labels, wb, reg_param, out_f, out_g));
}

int pio_fr_data_debug_stats(const pio_fr_data* d, double out[10]) {
  if (!d || !out) return PIO_ALS_ERR_ARG;
  out[0] = (double)d->parts, out[1] = (double)d->n, out[2] = (double)d->host_rows, out[3] = d->parse_ms;
  out[4] = d->gram_ms, out[5] = d->project_ms, out[6] = d->sigma_ms, out[7] = d->lr_ms, out[8] = (double)d->lr_evals;
  out[9] = (double)d->slices;
  return PIO_ALS_OK;
}

int pio_fr_model_create(int device, int32_t p, int32_t k, int32_t n_label, const double* mean, const double* pc,
                        const double* coef, const double* b, pio_fr_model** out) {
  if (!out) return fail(nullptr, PIO_ALS_ERR_ARG, "null argument");
  *out = nullptr;
  if (p < 1 || p > 65535 || k < 1 || k > p || n_label < 1 || n_label > 65535)
    return fail(nullptr, PIO_ALS_ERR_ARG, "bad model shape: p = %d, k = %d, n_label = %d (1 <= k <= p <= 65535, "
                "n_label >= 1)", p, k, n_label);
  if (!mean || !pc || !coef || !b) return fail(nullptr, PIO_ALS_ERR_ARG, "null argument");
  try {
    const std::vector<double> a = fr_components(pc, p, k);
    std::unique_ptr<pio_fr_model> m(new pio_fr_model);
    m->device = device, m->p = p, m->k = k, m->n_label = n_label;
    CK0(cudaSetDevice(device));
    CK0(cudaStreamCreateWithFlags(&m->st, cudaStreamNonBlocking));
    std::unique_ptr<pio_fr_model, int (*)(pio_fr_model*)> g(m.release(), pio_fr_model_destroy);
    CK0(cudaMalloc((void**)&g->d_mean, sizeof(double) * (size_t)p));
    CK0(cudaMalloc((void**)&g->d_a, sizeof(double) * a.size()));
    CK0(cudaMalloc((void**)&g->d_coef, sizeof(double) * (size_t)n_label * k));
    CK0(cudaMalloc((void**)&g->d_b, sizeof(double) * (size_t)n_label));
    CK0(cudaMemcpy(g->d_mean, mean, sizeof(double) * (size_t)p, cudaMemcpyHostToDevice));
    CK0(cudaMemcpy(g->d_a, a.data(), sizeof(double) * a.size(), cudaMemcpyHostToDevice));
    CK0(cudaMemcpy(g->d_coef, coef, sizeof(double) * (size_t)n_label * k, cudaMemcpyHostToDevice));
    CK0(cudaMemcpy(g->d_b, b, sizeof(double) * (size_t)n_label, cudaMemcpyHostToDevice));
    *out = g.release();
  } catch (const std::bad_alloc&) {
    return fail(nullptr, PIO_ALS_ERR_NOMEM, "pio_fr_model_create: out of host memory");
  }
  return PIO_ALS_OK;
}

int pio_fr_model_destroy(pio_fr_model* m) {
  if (!m) return PIO_ALS_OK;
  cudaSetDevice(m->device);
  if (m->st) cudaStreamSynchronize(m->st);
  for (void* q : {(void*)m->d_mean, (void*)m->d_a, (void*)m->d_coef, (void*)m->d_b})
    if (q) cudaFree(q);
  if (m->st) cudaStreamDestroy(m->st);
  delete m;
  return PIO_ALS_OK;
}

int pio_fr_model_scores(pio_fr_model* m, const uint8_t* tok_bytes, const int64_t* tok_off, int32_t n,
                        int32_t* out_status, double* out_scores) {
  FR_CALL(m, "pio_fr_model_scores", fr_model_scores(m, tok_bytes, tok_off, n, out_status, out_scores));
}

int pio_fr_model_debug_stats(const pio_fr_model* m, double out[4]) {
  if (!m || !out) return PIO_ALS_ERR_ARG;
  out[0] = (double)m->parts, out[1] = (double)m->rows, out[2] = (double)m->host_rows, out[3] = m->device_ms;
  return PIO_ALS_OK;
}

}  // extern "C"
