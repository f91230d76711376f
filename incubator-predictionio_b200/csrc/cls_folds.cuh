// cls_folds.cuh -- the k-fold split of the classification template's evaluation on the device
// (examples/scala-parallel-classification/add-algorithm/src/main/scala/DataSource.scala readEval: row i of the labeled
// points goes to the test set of fold i % evalK and to the training set of every other fold), the input checks of
// NaiveBayes / RandomForest over a fold's training rows, and the counts behind Accuracy and Precision
// (Evaluation.scala, PrecisionEvaluation.scala) over a fold's predicted labels.  DESIGN.md 4.12.
//
// Rows are cut without a scan: training row e of fold f (e % k != f) is row e - ceil((e - f) / k) of the fold's training
// set (eval_folds.cuh's train_coo_kernel uses the same formula), test row t is row f + t * k.  Labels are encoded once:
// distinct labels ascending (rf::key_of order), and per row its index among them.  Fold f trains on class c unless every
// row of c is in fold f, i.e. unless c's smallest and largest fold are both f.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include "forest.cuh"

namespace pio {
namespace clf {

constexpr int THREADS = 256;
constexpr int CHECK_NEG_F32 = 0;     // first_bad_kernel: a feature negative after rounding to float32 (NaiveBayes)
constexpr int CHECK_FINITE = 1;      // a non-finite label or feature (RandomForest)
constexpr int CHECK_LABEL = 2;       // a label outside [0, num_classes) (RandomForest)

__device__ __forceinline__ long long train_pos(long long e, int k, int f) { return e - (e + k - 1 - f) / k; }

// order-preserving keys of the labels, payload = row
__global__ void label_keys_kernel(const double* __restrict__ label, long long n, uint64_t* __restrict__ key,
                                  uint32_t* __restrict__ val) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  key[i] = rf::key_of(label[i]);
  val[i] = (uint32_t)i;
}

// sorted keys, run heads and their exclusive scan -> cls[row] = index of its label among the distinct labels, ukey[c] =
// the key of distinct label c
__global__ void class_index_kernel(const uint64_t* __restrict__ key, const uint32_t* __restrict__ val,
                                   const uint32_t* __restrict__ head, const uint32_t* __restrict__ pos, long long n,
                                   int* __restrict__ cls, uint64_t* __restrict__ ukey) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const int c = (int)(pos[i] + head[i]) - 1;
  cls[val[i]] = c;
  if (head[i]) ukey[c] = key[i];
}

// per class: smallest and largest fold that holds one of its rows (fmin preset to k, fmax to -1).  Most rows find their
// class's range already covering their fold and issue no atomic.
__global__ void class_folds_kernel(const int* __restrict__ cls, long long n, int k, int* fmin, int* fmax) {
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
    const int c = cls[i], f = (int)(i % k);
    if (f < *(volatile int*)&fmin[c]) atomicMin(&fmin[c], f);
    if (f > *(volatile int*)&fmax[c]) atomicMax(&fmax[c], f);
  }
}

// the first training row of fold f (smallest row e, so also smallest training position) that fails check `mode`;
// *out preset to n
__global__ void first_bad_kernel(const double* __restrict__ label, const double* __restrict__ x, long long n, int F,
                                 int k, int f, int mode, int num_classes, unsigned long long* out) {
  for (long long e = (long long)blockIdx.x * blockDim.x + threadIdx.x; e < n; e += (long long)gridDim.x * blockDim.x) {
    if ((int)(e % k) == f) continue;
    bool bad = false;
    if (mode == CHECK_LABEL) {
      bad = label[e] >= (double)num_classes || label[e] < 0.0;
    } else if (mode == CHECK_FINITE) {
      bad = !isfinite(label[e]);
      for (int j = 0; j < F; ++j) bad |= !isfinite(x[e * F + j]);
    } else {
      for (int j = 0; j < F; ++j) bad |= __double2float_rn(x[e * F + j]) < 0.0f;
    }
    if (bad) atomicMin(out, (unsigned long long)e);
  }
}

// NaiveBayes input of fold f: float32 features (round to nearest, as numpy's astype(float32)) and the fold-local class
// (lmap: class -> index among the fold's training classes)
__global__ void nb_gather_kernel(const int* __restrict__ cls, const double* __restrict__ x, long long n, int F, int k,
                                 int f, const int* __restrict__ lmap, int* __restrict__ ocls, float* __restrict__ ox) {
  for (long long e = (long long)blockIdx.x * blockDim.x + threadIdx.x; e < n; e += (long long)gridDim.x * blockDim.x) {
    if ((int)(e % k) == f) continue;
    const long long p = train_pos(e, k, f);
    ocls[p] = lmap[cls[e]];
    for (int j = 0; j < F; ++j) ox[p * F + j] = __double2float_rn(x[e * F + j]);
  }
}

// RandomForest input of fold f: the fp64 rows and trunc(label) as the class byte (pio_rf_train's hcls)
__global__ void rf_gather_kernel(const double* __restrict__ label, const double* __restrict__ x, long long n, int F,
                                 int k, int f, uint8_t* __restrict__ ocls, double* __restrict__ ox) {
  for (long long e = (long long)blockIdx.x * blockDim.x + threadIdx.x; e < n; e += (long long)gridDim.x * blockDim.x) {
    if ((int)(e % k) == f) continue;
    const long long p = train_pos(e, k, f);
    ocls[p] = (uint8_t)(int)trunc(label[e]);
    for (int j = 0; j < F; ++j) ox[p * F + j] = x[e * F + j];
  }
}

__device__ __forceinline__ void put(float* o, double v) { *o = __double2float_rn(v); }
__device__ __forceinline__ void put(double* o, double v) { *o = v; }

// the m test rows of fold f (row f + t * k), as float32 (NaiveBayes) or fp64 (RandomForest) features
template <typename T>
__global__ void test_gather_kernel(const double* __restrict__ x, int F, int k, int f, long long m, T* __restrict__ ox) {
  const long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= m) return;
  const long long e = (long long)f + t * k;
  for (int j = 0; j < F; ++j) put(ox + t * F + j, x[e * F + j]);
}

// predicted label of test row t: class_label[class index]
__global__ void pred_label_kernel(const int* __restrict__ idx, long long m, const double* __restrict__ class_label,
                                  double* __restrict__ pred) {
  const long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (t < m) pred[t] = class_label[idx[t]];
}

// over the m test rows of fold f: out[0] rows with predicted == actual, out[1] with predicted == L, out[2] both (fp64
// ==, as Python compares floats); out preset to 0
__global__ void __launch_bounds__(THREADS) counts_kernel(const double* __restrict__ pred, const double* __restrict__ label,
                                                         long long m, int k, int f, double L,
                                                         unsigned long long* __restrict__ out) {
  unsigned long long c[3] = {0, 0, 0};
  for (long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x; t < m; t += (long long)gridDim.x * blockDim.x) {
    const double p = pred[t];
    const bool ok = p == label[(long long)f + t * k], hit = p == L;
    c[0] += ok, c[1] += hit, c[2] += ok && hit;
  }
  __shared__ unsigned long long s[3][THREADS / 32];
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
#pragma unroll
  for (int j = 0; j < 3; ++j) {
    for (int d = 16; d > 0; d >>= 1) c[j] += __shfl_down_sync(0xffffffffu, c[j], d);
    if (lane == 0) s[j][w] = c[j];
  }
  __syncthreads();
  if (threadIdx.x < 3) {
    unsigned long long v = 0;
    for (int q = 0; q < THREADS / 32; ++q) v += s[threadIdx.x][q];
    if (v) atomicAdd(&out[threadIdx.x], v);
  }
}

}  // namespace clf
}  // namespace pio
