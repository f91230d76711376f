// sort_scan.cuh -- device primitives for the ratings ingest (COO -> dedup -> CSR):
// a multi-block exclusive scan and a stable LSD radix sort of (uint64 key, uint32 payload)
// pairs.  Hand-written (no CUB/Thrust).  All work is HBM-bound integer traffic; the sort is
// stable so equal (row, col) keys keep event order, which the keep-last dedup rule of the
// ecommerce template relies on (ECommAlgorithm.scala:189-197).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

namespace pio {

// ------------------------------------------------------------------------------------------
// exclusive scan, uint32 (sums must fit in 32 bits: callers guarantee n_total < 2^32)
// ------------------------------------------------------------------------------------------
constexpr int SCAN_THREADS = 256;
constexpr int SCAN_ITEMS = 8;
constexpr int SCAN_TILE = SCAN_THREADS * SCAN_ITEMS;

__device__ __forceinline__ uint32_t warp_incl_scan(uint32_t v) {
  const int lane = threadIdx.x & 31;
#pragma unroll
  for (int d = 1; d < 32; d <<= 1) {
    uint32_t t = __shfl_up_sync(0xffffffffu, v, d);
    if (lane >= d) v += t;
  }
  return v;
}

__global__ void __launch_bounds__(SCAN_THREADS)
scan_tile_kernel(const uint32_t* __restrict__ in, uint32_t* __restrict__ out,
                 uint32_t* __restrict__ tile_sums, size_t n) {
  __shared__ uint32_t warp_tot[SCAN_THREADS / 32];
  const size_t base = (size_t)blockIdx.x * SCAN_TILE + (size_t)threadIdx.x * SCAN_ITEMS;
  uint32_t v[SCAN_ITEMS];
  uint32_t sum = 0;
#pragma unroll
  for (int i = 0; i < SCAN_ITEMS; ++i) {
    v[i] = (base + i < n) ? in[base + i] : 0u;
    sum += v[i];
  }
  const uint32_t incl = warp_incl_scan(sum);
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
  if (lane == 31) warp_tot[w] = incl;
  __syncthreads();
  if (w == 0) {
    uint32_t t = lane < SCAN_THREADS / 32 ? warp_tot[lane] : 0u;
    uint32_t ti = warp_incl_scan(t);
    if (lane < SCAN_THREADS / 32) warp_tot[lane] = ti - t;  // exclusive warp offsets
    if (lane == SCAN_THREADS / 32 - 1 && tile_sums) tile_sums[blockIdx.x] = ti;
  }
  __syncthreads();
  uint32_t run = warp_tot[w] + incl - sum;
#pragma unroll
  for (int i = 0; i < SCAN_ITEMS; ++i) {
    if (base + i < n) out[base + i] = run;
    run += v[i];
  }
}

__global__ void __launch_bounds__(SCAN_THREADS)
scan_add_kernel(uint32_t* __restrict__ out, const uint32_t* __restrict__ tile_offs, size_t n) {
  const uint32_t add = tile_offs[blockIdx.x];
  const size_t base = (size_t)blockIdx.x * SCAN_TILE + (size_t)threadIdx.x * SCAN_ITEMS;
#pragma unroll
  for (int i = 0; i < SCAN_ITEMS; ++i)
    if (base + i < n) out[base + i] += add;
}

// in may alias out. Returns cudaError; *launches counts kernels launched.
inline cudaError_t scan_exclusive_u32(const uint32_t* in, uint32_t* out, size_t n, cudaStream_t st,
                                      int64_t* launches) {
  if (n == 0) return cudaSuccess;
  const size_t nt = (n + SCAN_TILE - 1) / SCAN_TILE;
  uint32_t* sums = nullptr;
  cudaError_t e = cudaSuccess;
  if (nt > 1) {
    e = cudaMallocAsync((void**)&sums, nt * sizeof(uint32_t), st);
    if (e != cudaSuccess) return e;
  }
  scan_tile_kernel<<<(unsigned)nt, SCAN_THREADS, 0, st>>>(in, out, sums, n);
  if (launches) ++*launches;
  if (nt > 1) {
    e = scan_exclusive_u32(sums, sums, nt, st, launches);
    if (e != cudaSuccess) return e;
    scan_add_kernel<<<(unsigned)nt, SCAN_THREADS, 0, st>>>(out, sums, n);
    if (launches) ++*launches;
    e = cudaFreeAsync(sums, st);
    if (e != cudaSuccess) return e;
  }
  return cudaGetLastError();
}

// ------------------------------------------------------------------------------------------
// stable LSD radix sort, 8-bit digits, (uint64 key, uint32 payload)
// ------------------------------------------------------------------------------------------
constexpr int RS_THREADS = 256;
constexpr int RS_WARPS = RS_THREADS / 32;
constexpr int RS_ROUNDS = 16;                        // items per lane
constexpr int RS_WARP_ITEMS = 32 * RS_ROUNDS;        // 512
constexpr int RS_TILE = RS_THREADS * RS_ROUNDS;      // 4096

__global__ void __launch_bounds__(RS_THREADS)
rs_hist_kernel(const uint64_t* __restrict__ keys, size_t n, int shift, unsigned dmask, uint32_t* __restrict__ hist,
               unsigned nblocks) {
  __shared__ uint32_t sh[256];
  sh[threadIdx.x] = 0;
  __syncthreads();
  const size_t base = (size_t)blockIdx.x * RS_TILE;
#pragma unroll 4
  for (int i = 0; i < RS_ROUNDS; ++i) {
    const size_t idx = base + (size_t)i * RS_THREADS + threadIdx.x;
    if (idx < n) atomicAdd(&sh[(unsigned)(keys[idx] >> shift) & dmask], 1u);
  }
  __syncthreads();
  hist[(size_t)threadIdx.x * nblocks + blockIdx.x] = sh[threadIdx.x];
}

__global__ void __launch_bounds__(RS_THREADS)
rs_scatter_kernel(const uint64_t* __restrict__ kin, const uint32_t* __restrict__ vin,
                  uint64_t* __restrict__ kout, uint32_t* __restrict__ vout, size_t n, int shift, unsigned dmask,
                  const uint32_t* __restrict__ offs, unsigned nblocks) {
  __shared__ uint32_t wcnt[RS_WARPS][256];
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
  for (int i = threadIdx.x; i < RS_WARPS * 256; i += RS_THREADS) (&wcnt[0][0])[i] = 0;
  __syncthreads();
  const size_t wbase = (size_t)blockIdx.x * RS_TILE + (size_t)w * RS_WARP_ITEMS;
  uint64_t key[RS_ROUNDS];
  uint32_t val[RS_ROUNDS];
  uint32_t rnk[RS_ROUNDS];
  const uint32_t lt = (1u << lane) - 1u;
#pragma unroll
  for (int r = 0; r < RS_ROUNDS; ++r) {
    const size_t idx = wbase + (size_t)r * 32 + lane;
    const bool valid = idx < n;
    key[r] = valid ? kin[idx] : 0ull;
    val[r] = valid ? vin[idx] : 0u;
    const unsigned d = valid ? ((unsigned)(key[r] >> shift) & dmask) : 256u;
    const uint32_t peers = __match_any_sync(0xffffffffu, d);
    uint32_t prev = 0;
    if (valid) prev = wcnt[w][d];
    __syncwarp();
    if (valid && (peers & lt) == 0) wcnt[w][d] = prev + __popc(peers);
    __syncwarp();
    rnk[r] = prev + __popc(peers & lt);
  }
  __syncthreads();
  // per digit: exclusive prefix over the warps (position inside the digit's run of this tile), the tile-local start of
  // the run (exclusive scan over the digits) and the global start of the run
  __shared__ uint32_t lstart[256];
  __shared__ uint32_t goff[256];
  __shared__ uint32_t wtot[RS_WARPS];
  {
    const unsigned d = threadIdx.x;
    uint32_t run = 0;
#pragma unroll
    for (int ww = 0; ww < RS_WARPS; ++ww) {
      const uint32_t t = wcnt[ww][d];
      wcnt[ww][d] = run;
      run += t;
    }
    goff[d] = offs[(size_t)d * nblocks + blockIdx.x];
    const uint32_t incl = warp_incl_scan(run);
    if (lane == 31) wtot[w] = incl;
    __syncthreads();
    uint32_t pre = 0;
#pragma unroll
    for (int ww = 0; ww < RS_WARPS; ++ww)
      if (ww < w) pre += wtot[ww];
    lstart[d] = pre + incl - run;
  }
  __syncthreads();
  // tile-local sort into shared memory ...
  extern __shared__ __align__(16) unsigned char rs_smem[];
  uint64_t* skey = reinterpret_cast<uint64_t*>(rs_smem);            // [RS_TILE]
  uint32_t* sval = reinterpret_cast<uint32_t*>(skey + RS_TILE);     // [RS_TILE]
#pragma unroll
  for (int r = 0; r < RS_ROUNDS; ++r) {
    const size_t idx = wbase + (size_t)r * 32 + lane;
    if (idx < n) {
      const unsigned d = (unsigned)(key[r] >> shift) & dmask;
      const uint32_t lp = lstart[d] + wcnt[w][d] + rnk[r];
      skey[lp] = key[r];
      sval[lp] = val[r];
    }
  }
  __syncthreads();
  // ... then out in tile order: consecutive threads write consecutive elements of a digit's run (coalesced), instead
  // of every lane scattering 12 bytes to its own address
  const size_t tbase = (size_t)blockIdx.x * RS_TILE;
  const uint32_t cnt = (uint32_t)(n - tbase < (size_t)RS_TILE ? n - tbase : (size_t)RS_TILE);
#pragma unroll
  for (int r = 0; r < RS_ROUNDS; ++r) {
    const uint32_t pidx = (uint32_t)r * RS_THREADS + threadIdx.x;
    if (pidx < cnt) {
      const uint64_t kk = skey[pidx];
      const unsigned d = (unsigned)(kk >> shift) & dmask;
      const size_t pos = (size_t)goff[d] + (pidx - lstart[d]);
      kout[pos] = kk;
      vout[pos] = sval[pidx];
    }
  }
}

constexpr size_t RS_SCATTER_SMEM = (size_t)RS_TILE * (sizeof(uint64_t) + sizeof(uint32_t));   // 48 KB

// The two halves of a sort's ping-pong, each a key buffer with its payload buffer. The caller allocates both halves
// (all four buffers hold n elements) and fills the live one; radix_sort_pairs sorts the live half and leaves `live`
// naming the half that holds the result. The other half is spare: free for the caller to reuse.
struct SortBufs {
  uint64_t* k[2] = {nullptr, nullptr};
  uint32_t* v[2] = {nullptr, nullptr};
  int live = 0;
  uint64_t* keys() const { return k[live]; }
  uint32_t* vals() const { return v[live]; }
  uint64_t* spare_keys() const { return k[live ^ 1]; }
  uint32_t* spare_vals() const { return v[live ^ 1]; }
  void flip() { live ^= 1; }   // the spare half becomes live: for data the caller writes there
};

// Stable sort of the live half by key bits [0, nbits); the spare half is clobbered.  Bits at and above nbits do not
// order the keys: the last pass masks its digit to the bits below nbits.
inline cudaError_t radix_sort_pairs(SortBufs& b, size_t n, int nbits, cudaStream_t st, int64_t* launches) {
  if (n == 0) return cudaSuccess;
  const unsigned nblocks = (unsigned)((n + RS_TILE - 1) / RS_TILE);
  uint32_t* hist = nullptr;
  cudaError_t e = cudaMallocAsync((void**)&hist, (size_t)256 * nblocks * sizeof(uint32_t), st);
  if (e != cudaSuccess) return e;
  e = cudaFuncSetAttribute(rs_scatter_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)RS_SCATTER_SMEM);
  for (int shift = 0; e == cudaSuccess && shift < nbits; shift += 8) {
    const unsigned dmask = nbits - shift >= 8 ? 255u : (1u << (nbits - shift)) - 1u;
    rs_hist_kernel<<<nblocks, RS_THREADS, 0, st>>>(b.keys(), n, shift, dmask, hist, nblocks);
    if (launches) ++*launches;
    e = scan_exclusive_u32(hist, hist, (size_t)256 * nblocks, st, launches);
    if (e != cudaSuccess) break;
    rs_scatter_kernel<<<nblocks, RS_THREADS, RS_SCATTER_SMEM, st>>>(b.keys(), b.vals(), b.spare_keys(), b.spare_vals(),
                                                                    n, shift, dmask, hist, nblocks);
    if (launches) ++*launches;
    b.flip();
  }
  const cudaError_t ef = cudaFreeAsync(hist, st);
  if (e != cudaSuccess) return e;
  if (ef != cudaSuccess) return ef;
  return cudaGetLastError();
}

}  // namespace pio
