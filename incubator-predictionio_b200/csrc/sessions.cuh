// sessions.cuh -- the lead scoring template's sessions (pio_lead_sessions; rules: tests/leadscoring_ref.py, DESIGN 4.16)
//   landing_time_kernel   per session, the earliest view time (atomicMin on an order-preserving key of the milliseconds)
//   landing_pick_kernel   per session, the last view in event order among the views at that time (atomicMax)
//   buy_flag_kernel       per session, whether some buy is strictly after the landing view
// Minimum and maximum do not depend on the order of the atomics, so the sessions are the same on every run.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

namespace pio {
namespace lead {

__device__ __forceinline__ unsigned long long time_key(long long t) { return (unsigned long long)t ^ (1ull << 63); }

__global__ void landing_time_kernel(const int* __restrict__ sess, const uint8_t* __restrict__ is_buy,
                                    const long long* __restrict__ t, int64_t n, unsigned long long* __restrict__ tmin) {
  const int64_t r = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (r < n && !is_buy[r]) atomicMin(&tmin[sess[r]], time_key(t[r]));
}
__global__ void landing_pick_kernel(const int* __restrict__ sess, const uint8_t* __restrict__ is_buy,
                                    const long long* __restrict__ t, int64_t n,
                                    const unsigned long long* __restrict__ tmin, long long* __restrict__ landing) {
  const int64_t r = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (r < n && !is_buy[r] && time_key(t[r]) == tmin[sess[r]]) atomicMax(&landing[sess[r]], (long long)r);
}
__global__ void buy_flag_kernel(const int* __restrict__ sess, const uint8_t* __restrict__ is_buy,
                                const long long* __restrict__ t, int64_t n, const unsigned long long* __restrict__ tmin,
                                const long long* __restrict__ landing, uint8_t* __restrict__ buy) {
  const int64_t r = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (r >= n || !is_buy[r]) return;
  const int s = sess[r];
  if (landing[s] >= 0 && time_key(t[r]) > tmin[s]) buy[s] = 1;
}

}  // namespace lead
}  // namespace pio
