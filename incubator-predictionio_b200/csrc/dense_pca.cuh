// dense_pca.cuh -- the dimensionality-reduction template's dense path (pio_fr_*; DESIGN.md 4.19): feature strings
// parsed into a resident row-major fp64 matrix, its column means and Gramian, and the fixed-order folds that project
// rows onto the principal components and score them.
//
//   fr_parse_kernel      one thread per row: decode the raw JSON string token (decode_string_lenient), split it with
//                        Java's String.split(", ") rules and parse each piece on Clinger's exact fast path (decimal
//                        significand < 2^53, |exponent| <= 22: one IEEE multiply or divide by an exact power of ten).
//                        A row holding any other piece is marked FR_HOST and parsed by the host's restatement of
//                        Double.parseDouble; a row of fast pieces whose count differs from p is marked FR_LEN.
//   fr_colsum_kernel     per (slice, column): the column's sum over the slice's rows, in row order
//   fr_gram_kernel       per (slice, 64 x 64 tile on or above the diagonal): fma over the slice's rows in row order
//   fr_gram_fold_kernel  per entry i <= j: the slices' partial sums added left to right from 0.0, mirrored to (j, i)
//   fr_fold_kernel       per (row, output): y = 0.0; y = y + A_oj * (x_j - shift_j) for j ascending, each operation
//                        rounded on its own (no FMA), then y + add_o.  Serves transform and the prediction scores.
//
// The slices are a function of (n, p) alone (fr_slices), so the mean and the Gramian do not depend on the parse budget
// or on the launch geometry, and no floating-point atomics are used.
#pragma once
#include <stdint.h>

#include "event_line.h"

namespace pio {

enum { FR_OK = 0, FR_HOST = 1, FR_BAD = -1, FR_NONFINITE = -2, FR_LEN = -3 };

constexpr int FR_TILE = 64;          // Gramian and fold tiles: 64 x 64 outputs per 256-thread block, 4 x 4 per thread
constexpr int FR_KC = 16;            // rows (Gramian) or inputs (fold) staged in shared memory per step
constexpr long long FR_SLICE_MIN = 4096;
constexpr int FR_SLICE_MAX = 64;
constexpr long long FR_PART_DOUBLES = 1ll << 27;   // the slices' partial Gramians hold at most 1 GiB

// rows of one slice (a multiple of FR_KC) and the slice count for n rows of p columns
struct FrSlices {
  long long rows = 0;
  int count = 0;
};
inline FrSlices fr_slices(long long n, long long p) {
  long long s = (n + FR_SLICE_MIN - 1) / FR_SLICE_MIN;
  s = s < FR_SLICE_MAX ? s : FR_SLICE_MAX;
  const long long cap = FR_PART_DOUBLES / (p * p);
  s = s < cap ? s : cap;
  if (s < 1) s = 1;
  long long rows = (n + s - 1) / s;
  rows = (rows + FR_KC - 1) / FR_KC * FR_KC;
  FrSlices out;
  out.rows = rows;
  out.count = (int)((n + rows - 1) / rows);
  if (out.count < 1) out.count = 1;
  return out;
}

__constant__ double c_fr_pow10[23] = {1e0,  1e1,  1e2,  1e3,  1e4,  1e5,  1e6,  1e7,  1e8,  1e9,  1e10, 1e11,
                                      1e12, 1e13, 1e14, 1e15, 1e16, 1e17, 1e18, 1e19, 1e20, 1e21, 1e22};

// One piece [a, b) on the fast path: true and *v, or false (the host parses the row).
__device__ __forceinline__ bool fr_fast_piece(const uint8_t* s, int a, int b, double* v) {
  while (a < b && s[a] <= ' ') ++a;       // String.trim: every char <= U+0020
  while (b > a && s[b - 1] <= ' ') --b;
  if (a >= b) return false;
  bool neg = false;
  if (s[a] == '+' || s[a] == '-') neg = s[a++] == '-';
  unsigned long long m = 0;
  int e10 = 0, digits = 0;
  bool point = false;
  for (; a < b; ++a) {
    const uint8_t c = s[a];
    if (c == '.' && !point) {
      point = true;
      continue;
    }
    if (c < '0' || c > '9') break;
    ++digits;
    if (m > (((1ull << 53) - 1) - (c - '0')) / 10) return false;   // the significand would reach 2^53
    m = m * 10 + (c - '0');
    if (point) --e10;
  }
  if (!digits) return false;
  if (a < b && (s[a] == 'e' || s[a] == 'E')) {
    ++a;
    bool eneg = false;
    if (a < b && (s[a] == '+' || s[a] == '-')) eneg = s[a++] == '-';
    int ex = 0, ed = 0;
    for (; a < b && s[a] >= '0' && s[a] <= '9'; ++a, ++ed) ex = ex < 100000 ? ex * 10 + (s[a] - '0') : ex;
    if (!ed) return false;
    e10 += eneg ? -ex : ex;
  }
  if (a != b) return false;                // a suffix, hex, NaN, Infinity or anything else
  double x;
  if (m == 0) {
    x = 0.0;
  } else {
    if (e10 > 22 || e10 < -22) return false;
    const double dm = (double)m;           // exact: m < 2^53
    x = e10 >= 0 ? __dmul_rn(dm, c_fr_pow10[e10]) : __ddiv_rn(dm, c_fr_pow10[-e10]);
  }
  *v = neg ? -x : x;
  return true;
}

// One part of rows: raw tokens raw[off[r] .. off[r + 1]) (offsets local to the part), decoded into dec (same offsets);
// values of row r go to x + r * p.
__global__ void fr_parse_kernel(const uint8_t* __restrict__ raw, const long long* __restrict__ off, int nr, int p,
                                uint8_t* __restrict__ dec, double* __restrict__ x, int* __restrict__ status) {
  const int r = blockIdx.x * blockDim.x + threadIdx.x;
  if (r >= nr) return;
  const long long b = off[r];
  uint8_t* s = dec + b;
  const int len = ev::decode_string_lenient(raw + b, 0, (int)(off[r + 1] - b), s);
  double* row = x + (long long)r * p;
  if (len == 0) {                          // "".split(", ") is [""], which does not parse
    status[r] = FR_HOST;
    return;
  }
  int j = 0, empty = 0, start = 0;
  for (int i = 0;; ) {
    const bool end = i >= len;
    if (end || (s[i] == ',' && i + 1 < len && s[i + 1] == ' ')) {
      if (i == start) {
        ++empty;                           // dropped if only empty pieces follow
      } else {
        double v;
        if (empty || !fr_fast_piece(s, start, i, &v)) {
          status[r] = FR_HOST;
          return;
        }
        if (j < p) row[j] = v;
        ++j;
      }
      if (end) break;
      i += 2;
      start = i;
    } else {
      ++i;
    }
  }
  status[r] = j == p ? FR_OK : FR_LEN;
}

// cs[s * p + j] = sum of x[r][j] over the rows r of slice s, in row order from 0.0
__global__ void fr_colsum_kernel(const double* __restrict__ x, long long n, int p, long long slice_rows,
                                 double* __restrict__ cs) {
  const int j = blockIdx.x * blockDim.x + threadIdx.x;
  const int s = blockIdx.y;
  if (j >= p) return;
  const long long r0 = (long long)s * slice_rows, r1 = min(n, r0 + slice_rows);
  double acc = 0.0;
  for (long long r = r0; r < r1; ++r) acc = __dadd_rn(acc, x[r * p + j]);
  cs[(long long)s * p + j] = acc;
}

// Partial Gramian of slice blockIdx.z over tile (blockIdx.y, blockIdx.x) with tile row <= tile column; entries into
// part + s * p * p.  Thread (ty, tx) owns rows I0 + ty + 16a and columns J0 + tx + 16b.
__global__ void __launch_bounds__(256) fr_gram_kernel(const double* __restrict__ x, long long n, int p,
                                                      long long slice_rows, double* __restrict__ part) {
  const int ti = blockIdx.y, tj = blockIdx.x;
  if (ti > tj) return;
  __shared__ double xa[FR_KC][FR_TILE];
  __shared__ double xb[FR_KC][FR_TILE];
  const int tx = threadIdx.x & 15, ty = threadIdx.x >> 4;
  const int I0 = ti * FR_TILE, J0 = tj * FR_TILE;
  const long long r0 = (long long)blockIdx.z * slice_rows, r1 = min(n, r0 + slice_rows);
  double acc[4][4];
#pragma unroll
  for (int a = 0; a < 4; ++a)
#pragma unroll
    for (int c = 0; c < 4; ++c) acc[a][c] = 0.0;
  for (long long rb = r0; rb < r1; rb += FR_KC) {
    const int kc = (int)min((long long)FR_KC, r1 - rb);
#pragma unroll
    for (int q = 0; q < 4; ++q) {
      const int e = threadIdx.x + q * 256, rr = e >> 6, cc = e & 63;
      const bool in = rr < kc;
      xa[rr][cc] = in && I0 + cc < p ? x[(rb + rr) * p + I0 + cc] : 0.0;
      xb[rr][cc] = in && J0 + cc < p ? x[(rb + rr) * p + J0 + cc] : 0.0;
    }
    __syncthreads();
    for (int k = 0; k < kc; ++k) {
      double va[4], vb[4];
#pragma unroll
      for (int a = 0; a < 4; ++a) va[a] = xa[k][ty + 16 * a];
#pragma unroll
      for (int c = 0; c < 4; ++c) vb[c] = xb[k][tx + 16 * c];
#pragma unroll
      for (int a = 0; a < 4; ++a)
#pragma unroll
        for (int c = 0; c < 4; ++c) acc[a][c] = __fma_rn(va[a], vb[c], acc[a][c]);
    }
    __syncthreads();
  }
  double* out = part + (long long)blockIdx.z * p * p;
#pragma unroll
  for (int a = 0; a < 4; ++a)
#pragma unroll
    for (int c = 0; c < 4; ++c) {
      const int i = I0 + ty + 16 * a, j = J0 + tx + 16 * c;
      if (i < p && j < p) out[(long long)i * p + j] = acc[a][c];
    }
}

// G[i][j] = G[j][i] = 0.0 + part_0[i][j] + part_1[i][j] + ... for i <= j
__global__ void fr_gram_fold_kernel(const double* __restrict__ part, int slices, int p, double* __restrict__ g) {
  const long long e = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (e >= (long long)p * p) return;
  const int i = (int)(e / p), j = (int)(e % p);
  if (i > j) return;
  double acc = 0.0;
  for (int s = 0; s < slices; ++s) acc = __dadd_rn(acc, part[(long long)s * p * p + e]);
  g[e] = acc;
  g[(long long)j * p + i] = acc;
}

// out[r * out_rs + o * out_os] (and out2's, when not null) = fold_j(a[o * m + j] * (x[r * m + j] - shift[j])) + add[o] over rows r < n, outputs
// o < no, inputs j < m (shift and add may be null: no subtraction, no addend).  Thread (ty, tx) of the 64 x 64 tile
// owns rows R0 + ty + 16a and outputs O0 + tx + 16b; each output's fold runs over j in index order.
__global__ void __launch_bounds__(256) fr_fold_kernel(const double* __restrict__ x, long long n, int m,
                                                      const double* __restrict__ a, int no,
                                                      const double* __restrict__ shift, const double* __restrict__ add,
                                                      double* __restrict__ out, long long out_rs, long long out_os,
                                                      double* __restrict__ out2, long long out2_rs,
                                                      long long out2_os) {
  __shared__ double xs[FR_TILE][FR_KC + 1];
  __shared__ double as[FR_TILE][FR_KC + 1];
  const int tx = threadIdx.x & 15, ty = threadIdx.x >> 4;
  const long long R0 = (long long)blockIdx.x * FR_TILE;
  const int O0 = blockIdx.y * FR_TILE;
  double acc[4][4];
#pragma unroll
  for (int u = 0; u < 4; ++u)
#pragma unroll
    for (int c = 0; c < 4; ++c) acc[u][c] = 0.0;
  for (int j0 = 0; j0 < m; j0 += FR_KC) {
    const int kc = min(FR_KC, m - j0);
#pragma unroll
    for (int q = 0; q < 4; ++q) {
      const int e = threadIdx.x + q * 256, rr = e >> 4, jj = e & 15;
      double v = 0.0, w = 0.0;
      if (jj < kc) {
        if (R0 + rr < n) {
          v = x[(R0 + rr) * m + j0 + jj];
          if (shift) v = __dsub_rn(v, shift[j0 + jj]);
        }
        if (O0 + rr < no) w = a[(long long)(O0 + rr) * m + j0 + jj];
      }
      xs[rr][jj] = v;
      as[rr][jj] = w;
    }
    __syncthreads();
    for (int k = 0; k < kc; ++k) {
      double vx[4], va[4];
#pragma unroll
      for (int u = 0; u < 4; ++u) vx[u] = xs[ty + 16 * u][k];
#pragma unroll
      for (int c = 0; c < 4; ++c) va[c] = as[tx + 16 * c][k];
#pragma unroll
      for (int u = 0; u < 4; ++u)
#pragma unroll
        for (int c = 0; c < 4; ++c) acc[u][c] = __dadd_rn(acc[u][c], __dmul_rn(va[c], vx[u]));
    }
    __syncthreads();
  }
#pragma unroll
  for (int u = 0; u < 4; ++u)
#pragma unroll
    for (int c = 0; c < 4; ++c) {
      const long long r = R0 + ty + 16 * u;
      const int o = O0 + tx + 16 * c;
      if (r < n && o < no) {
        const double v = add ? __dadd_rn(acc[u][c], add[o]) : acc[u][c];
        out[r * out_rs + (long long)o * out_os] = v;
        if (out2) out2[r * out2_rs + (long long)o * out2_os] = v;
      }
    }
}

}  // namespace pio
