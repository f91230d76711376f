// forest_splits.h -- the host-side rules of the RandomForest classifier (pio_rf_train, csrc/forest.cuh): argument and
// featureSubsetStrategy parsing, the per-feature thresholds of MLlib's findSplitsForContinuousFeature, the Poisson(1)
// table of the bootstrap, the keyed counter hash every random draw comes from, and the tree-group plan.
//
// Plain C++ with no CUDA header, so that tests/test_forest_ref.py compiles it alone with g++ and checks it against the
// NumPy restatement tests/forest_ref.py bit for bit.  The hash and the bag weight are also compiled for the device
// (RF_HD), so the kernels and the host draw the same bits.
#pragma once
#include <math.h>
#include <stdint.h>
#include <stdlib.h>
#include <string.h>

#include <algorithm>
#include <utility>
#include <vector>

#ifdef __CUDACC__
#define RF_HD __host__ __device__ __forceinline__
#else
#define RF_HD inline
#endif

namespace pio {

// limits of this implementation (pio_als.h): classes are a 64-bit mask away, bin codes are uint16, rows are int32
constexpr int RF_MAX_CLASSES = 64;
constexpr int RF_MAX_BINS = 65536;
constexpr int RF_MAX_DEPTH = 30;
constexpr int RF_POISSON_N = 16;        // weights are capped at 16: the table holds P(X <= k) for k = 0 .. 15
constexpr int RF_GINI = 0, RF_ENTROPY = 1, RF_VARIANCE = 2;
constexpr int RF_LABEL_BITS = 44;       // the regressor's quantised labels: |yq| <= 2^44 (tests/forest_reg_ref.py)
constexpr int RF_LABEL_EXP_MAX = 256;   // its labels: |y| < 2^256, and max |y| >= 2^-256 unless every label is 0

// stream tags of the counter hash
constexpr uint64_t RF_TAG_SAMPLE = 1, RF_TAG_BAG = 2, RF_TAG_SUBSET = 3;

RF_HD uint64_t rf_mix(uint64_t x) {   // the splitmix64 finaliser of the ALS counter-hash initialisation
  x += 0x9E3779B97F4A7C15ull;
  uint64_t z = x;
  z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9ull;
  z = (z ^ (z >> 27)) * 0x94D049BB133111EBull;
  return z ^ (z >> 31);
}
// the base of stream `tag` of tree t (the split sample uses tree 0); a draw is rf_draw(base, index)
RF_HD uint64_t rf_stream(int64_t seed, uint64_t tag, uint64_t t) { return rf_mix(rf_mix((uint64_t)seed ^ (tag << 56)) ^ t); }
RF_HD uint64_t rf_draw(uint64_t base, uint64_t index) { return rf_mix(base ^ index); }
RF_HD double rf_u53(uint64_t h) { return (double)(h >> 11) * (1.0 / 9007199254740992.0); }

// bootstrap weight of row `row` of a tree whose bag stream is `base`: the Poisson(1) inverse CDF over cdf[0 .. 15]
RF_HD int rf_bag_weight(const double* cdf, uint64_t base, uint64_t row) {
  const double u = rf_u53(rf_draw(base, row));
  int w = 0;
  for (int k = 0; k < RF_POISSON_N; ++k) w += cdf[k] <= u ? 1 : 0;
  return w;
}

// P(X <= k), X ~ Poisson(1), k = 0 .. 15: pmf(0) = e^-1 (the correctly rounded double, written out so that no libm
// is involved), pmf(k) = pmf(k - 1) / k, summed in order
inline void rf_poisson_table(double cdf[RF_POISSON_N]) {
  double p = 0x1.78b56362cef38p-2, c = 0.0;
  for (int k = 0; k < RF_POISSON_N; ++k) {
    if (k > 0) p = p / (double)k;
    c = c + p;
    cdf[k] = c;
  }
}

// featureSubsetStrategy -> features per node (RandomForest.run), or 0 for a string MLlib rejects.  The spellings:
// auto|all|sqrt|log2|onethird, an integer k > 0 (min(k, F)), or a fraction r in (0, 1] (ceil(r F)).  The integer and
// decimal grammars are this project's: [+-]?[0-9]+ within int32, and [+-]?(digits[.digits*] | .digits)([eE][+-]?digits)?
inline bool rf_is_int(const char* s, long long* v) {
  const char* p = s;
  if (*p == '+' || *p == '-') ++p;
  if (!*p) return false;
  for (const char* q = p; *q; ++q)
    if (*q < '0' || *q > '9') return false;
  if (strlen(p) > 10) return false;
  *v = strtoll(s, nullptr, 10);
  return *v >= -2147483648ll && *v <= 2147483647ll;
}
inline bool rf_is_decimal(const char* s, double* v) {
  const char* p = s;
  if (*p == '+' || *p == '-') ++p;
  int digits = 0;
  while (*p >= '0' && *p <= '9') ++p, ++digits;
  if (*p == '.') {
    ++p;
    while (*p >= '0' && *p <= '9') ++p, ++digits;
  }
  if (digits == 0) return false;
  if (*p == 'e' || *p == 'E') {
    ++p;
    if (*p == '+' || *p == '-') ++p;
    if (!(*p >= '0' && *p <= '9')) return false;
    while (*p >= '0' && *p <= '9') ++p;
  }
  if (*p) return false;
  *v = strtod(s, nullptr);
  return true;
}
inline int rf_ceil_log2(long long v) {
  int b = 0;
  while ((1ll << b) < v) ++b;
  return b;
}
inline int rf_subset_size(const char* s, int n_feat, int num_trees) {
  if (!s) return 0;
  const long long F = n_feat;
  if (!strcmp(s, "auto")) s = num_trees == 1 ? "all" : "sqrt";
  if (!strcmp(s, "all")) return (int)F;
  if (!strcmp(s, "sqrt")) return (int)ceil(sqrt((double)F));
  if (!strcmp(s, "log2")) return std::max(1, rf_ceil_log2(F));
  if (!strcmp(s, "onethird")) return (int)ceil((double)F / 3.0);
  long long k = 0;
  if (rf_is_int(s, &k)) return k > 0 ? (int)std::min(k, F) : 0;
  double r = 0;
  if (rf_is_decimal(s, &r) && r > 0.0 && r <= 1.0) return (int)ceil(r * (double)F);
  return 0;
}

// The split sample (findSplits): every row, or, when n > max(maxBins^2, 10000), the rows whose draw of stream
// RF_TAG_SAMPLE is below max(maxBins^2, 10000) / n.  Returns that fraction (1.0: every row).
inline double rf_sample_fraction(int64_t n, int max_bins) {
  const double req = std::max((double)max_bins * (double)max_bins, 10000.0);
  return (double)n > req ? req / (double)n : 1.0;
}
RF_HD bool rf_sampled(uint64_t base, uint64_t row, double fraction) {
  return fraction >= 1.0 || rf_u53(rf_draw(base, row)) < fraction;
}

// findSplitsForContinuousFeature over the sampled values of one feature, given as their distinct values in ascending
// order (-0.0 counted as 0.0) with their counts.  num_bins = min(maxBins, n).  A row goes left of threshold t iff x <= t.
inline void rf_thresholds(const double* v, const int64_t* cnt, int64_t m, int64_t num_bins, std::vector<double>& out) {
  out.clear();
  if (m <= 1) return;                                          // constant feature (or nothing sampled)
  const int64_t num_splits = num_bins - 1;
  if (m - 1 <= num_splits) {                                   // every midpoint
    for (int64_t i = 1; i < m; ++i) out.push_back((v[i - 1] + v[i]) / 2.0);
    return;
  }
  int64_t num_samples = 0;
  for (int64_t i = 0; i < m; ++i) num_samples += cnt[i];
  const double stride = (double)num_samples / (double)(num_splits + 1);
  int64_t cur = cnt[0];
  double target = stride;
  for (int64_t i = 1; i < m; ++i) {                            // the greedy stride walk
    const int64_t prev = cur;
    cur += cnt[i];
    if (fabs((double)prev - target) < fabs((double)cur - target)) {
      out.push_back((v[i - 1] + v[i]) / 2.0);
      target += stride;
    }
  }
}

// The k features of node `node` (heap index) of the tree whose subset stream is `base`: those with the smallest keys
// rf_draw(rf_draw(base, node), f), ties to the smaller feature; in ascending feature order.  k == F: all, no draw.
inline void rf_node_subset(uint64_t base, int64_t node, int n_feat, int k, int* out) {
  if (k >= n_feat) {
    for (int f = 0; f < n_feat; ++f) out[f] = f;
    return;
  }
  const uint64_t nb = rf_draw(base, (uint64_t)node);
  std::vector<std::pair<uint64_t, int>> key((size_t)n_feat);
  for (int f = 0; f < n_feat; ++f) key[f] = {rf_draw(nb, (uint64_t)f), f};
  std::partial_sort(key.begin(), key.begin() + k, key.end());
  for (int i = 0; i < k; ++i) out[i] = key[i].second;
  std::sort(out, out + k);
}

// Impurity of weighted class counts (MLlib's Gini / Entropy .calculate), class by class; 0 for an empty node.
inline double rf_impurity(const int64_t* c, int n_class, int kind) {
  int64_t tot = 0;
  for (int k = 0; k < n_class; ++k) tot += c[k];
  if (tot == 0) return 0.0;
  const double n = (double)tot;
  double imp = kind == RF_GINI ? 1.0 : 0.0;
  for (int k = 0; k < n_class; ++k) {
    const double f = (double)c[k] / n;
    if (kind == RF_GINI) {
      const double ff = f * f;
      imp = imp - ff;
    } else if (c[k] != 0) {
      const double l = log(f) / 0x1.62e42fefa39efp-1;          // log(2), correctly rounded
      const double fl = f * l;
      imp = imp - fl;
    }
  }
  return imp;
}
// Variance.calculate on fp64 statistics: (Q - S * S / W) / W, 0 for an empty node
inline double rf_variance(double W, double S, double Q) {
  if (W == 0.0) return 0.0;
  const double ss = S * S;
  const double m = ss / W;
  const double d = Q - m;
  return d / W;
}
// the regressor's featureSubsetStrategy: "auto" is all features for one tree and onethird for more
inline int rf_subset_size_reg(const char* s, int n_feat, int num_trees) {
  if (s && !strcmp(s, "auto")) s = num_trees == 1 ? "all" : "onethird";
  return rf_subset_size(s, n_feat, num_trees);
}
// the regressor's label shift: s puts max |y| in [2^43, 2^44); 0 when every label is 0
inline int rf_label_shift(double max_abs) {
  if (max_abs == 0.0) return 0;
  int e = 0;
  frexp(max_abs, &e);
  return RF_LABEL_BITS - e;
}

// the class with the largest count, ties to the smaller class
inline int rf_argmax(const int64_t* c, int n_class) {
  int b = 0;
  for (int k = 1; k < n_class; ++k)
    if (c[k] > c[b]) b = k;
  return b;
}

// Trees are trained in groups: a group holds one int32 node id per (tree, row).  The group size is what fits in
// node_budget bytes (at least one tree), or `per_pass` when it is > 0 (PIO_RF_TREES_PER_PASS).
inline std::vector<std::pair<int, int>> rf_plan_groups(int num_trees, int64_t n, int64_t node_budget, int per_pass) {
  int64_t g = per_pass > 0 ? per_pass : node_budget / std::max<int64_t>(1, 4 * n);
  g = std::max<int64_t>(1, std::min<int64_t>(g, num_trees));
  std::vector<std::pair<int, int>> out;
  for (int t = 0; t < num_trees; t += (int)g) out.push_back({t, (int)std::min<int64_t>(num_trees, t + g)});
  return out;
}

}  // namespace pio
