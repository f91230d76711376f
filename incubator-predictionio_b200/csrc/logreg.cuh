// logreg.cuh -- binary logistic regression's loss and gradient over the resident projected rows (pio_fr_lr_*;
// DESIGN.md 4.19), for every class still training, each at its own point (w, b).
//
// Rows are summed in a fixed order: consecutive blocks of FR_LR_BLOCK rows, each folded left from 0.0 in row order,
// then the block sums folded left from 0.0 in block order.  A class's sums read only its own point and labels, so its
// loss and gradient do not depend on which other classes share the call.
//
//   fr_lr_colsum_kernel   per (block, column): sum of y_ij, or of (y_ij - c_j)^2 -- the two passes of sigma
//   fr_lr_margin_kernel   per (row, class): margin = -(fold_j (w_j * y_ij) / sigma_j + b) over the columns with
//                         sigma_j != 0 and y_ij != 0, multiplier = 1 / (1 + exp(margin)) - label, and the loss term
//                         log1pExp(margin), minus margin when the label is 0
//   fr_lr_grad_kernel     per (block, column, class): the block's sum of multiplier * y_ij / sigma_j (same skips);
//                         column k sums the multipliers (intercept), column k + 1 the loss terms
//   fr_lr_fold_kernel     per (class or column, entry): the block sums folded left
#pragma once
#include <stdint.h>

namespace pio {

constexpr int FR_LR_BLOCK = 256;

// y: n x k row-major.  part[blk * k + j]
__global__ void fr_lr_colsum_kernel(const double* __restrict__ y, long long n, int k, const double* __restrict__ center,
                                    double* __restrict__ part) {
  const int j = blockIdx.y * blockDim.x + threadIdx.x;
  if (j >= k) return;
  const long long r0 = (long long)blockIdx.x * FR_LR_BLOCK, r1 = min(n, r0 + FR_LR_BLOCK);
  double acc = 0.0;
  if (center) {
    const double c = center[j];
    for (long long r = r0; r < r1; ++r) {
      const double d = __dsub_rn(y[r * k + j], c);
      acc = __dadd_rn(acc, __dmul_rn(d, d));
    }
  } else {
    for (long long r = r0; r < r1; ++r) acc = __dadd_rn(acc, y[r * k + j]);
  }
  part[(long long)blockIdx.x * k + j] = acc;
}

// Spark's MLUtils.log1pExp
__device__ __forceinline__ double fr_log1p_exp(double x) {
  return x > 0.0 ? __dadd_rn(x, log1p(exp(-x))) : log1p(exp(x));
}

// yt: k x n column-major copy of the rows.  wb: [na][k + 1] (w, then b); lab: the class index of each slot; cls: each
// row's class.  mult, loss: [na][n].
__global__ void fr_lr_margin_kernel(const double* __restrict__ yt, long long n, int k, const double* __restrict__ sigma,
                                    const int* __restrict__ cls, const double* __restrict__ wb,
                                    const int* __restrict__ lab, double* __restrict__ mult, double* __restrict__ loss) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  const int c = blockIdx.y;
  if (i >= n) return;
  const double* w = wb + (long long)c * (k + 1);
  double s = 0.0;
  for (int j = 0; j < k; ++j) {
    const double v = yt[(long long)j * n + i], sd = sigma[j];
    if (sd != 0.0 && v != 0.0) s = __dadd_rn(s, __ddiv_rn(__dmul_rn(w[j], v), sd));
  }
  const double margin = -__dadd_rn(s, w[k]);
  const double label = cls[i] == lab[c] ? 1.0 : 0.0;
  mult[(long long)c * n + i] = __dsub_rn(__ddiv_rn(1.0, __dadd_rn(1.0, exp(margin))), label);
  const double l = fr_log1p_exp(margin);
  loss[(long long)c * n + i] = label > 0.0 ? l : __dsub_rn(l, margin);
}

// part[(c * nb + blk) * (k + 2) + j]
__global__ void fr_lr_grad_kernel(const double* __restrict__ y, long long n, int k, const double* __restrict__ sigma,
                                  const double* __restrict__ mult, const double* __restrict__ loss, int nb,
                                  double* __restrict__ part) {
  const int j = blockIdx.y * blockDim.x + threadIdx.x;
  const int c = blockIdx.z;
  if (j > k + 1) return;
  const long long r0 = (long long)blockIdx.x * FR_LR_BLOCK, r1 = min(n, r0 + FR_LR_BLOCK);
  const double* mc = mult + (long long)c * n;
  double acc = 0.0;
  if (j < k) {
    const double sd = sigma[j];
    if (sd != 0.0)
      for (long long r = r0; r < r1; ++r) {
        const double v = y[r * k + j];
        if (v != 0.0) acc = __dadd_rn(acc, __ddiv_rn(__dmul_rn(mc[r], v), sd));
      }
  } else {
    const double* src = j == k ? mc : loss + (long long)c * n;
    for (long long r = r0; r < r1; ++r) acc = __dadd_rn(acc, src[r]);
  }
  part[((long long)c * nb + blockIdx.x) * (k + 2) + j] = acc;
}

// out[c * w + j] = fold over blk < nb of part[(c * nb + blk) * w + j], for c < blockIdx.y's range
__global__ void fr_lr_fold_kernel(const double* __restrict__ part, int nb, int w, double* __restrict__ out) {
  const int j = blockIdx.x * blockDim.x + threadIdx.x;
  const int c = blockIdx.y;
  if (j >= w) return;
  double acc = 0.0;
  for (int b = 0; b < nb; ++b) acc = __dadd_rn(acc, part[((long long)c * nb + b) * w + j]);
  out[(long long)c * w + j] = acc;
}

}  // namespace pio
