"""CPU: the RandomForest restatement (tests/forest_ref.py) on hand-computed trees and rules, and csrc/forest_splits.h
(compiled alone with g++) against it bit for bit: thresholds, subset sizes, the Poisson table, bag weights, the split
sample and node subsets."""
import math
import shutil
import subprocess
from pathlib import Path

import numpy as np
import pytest

from tests import forest_ref as fr

CSRC = Path(__file__).resolve().parents[1] / "incubator-predictionio_b200" / "csrc"


def _train(y, x, **kw):
    args = dict(num_classes=2, num_trees=1, strategy="auto", impurity="gini", max_depth=4, max_bins=32)
    args.update(kw)
    return fr.train(np.asarray(y, float), np.asarray(x, float).reshape(len(y), -1), args.pop("num_classes"),
                    args.pop("num_trees"), args.pop("strategy"), args.pop("impurity"), args.pop("max_depth"),
                    args.pop("max_bins"), **args)


# ---- hand-computed trees -----------------------------------------------------------------------------------------
def test_one_split_gini():
    f = _train([0, 0, 1, 1], [1, 2, 3, 4])
    assert list(f["feature"]) == [0, -1, -1] and f["threshold"][0] == 2.5
    assert list(f["left"]) == [1, -1, -1] and list(f["right"]) == [2, -1, -1]
    assert list(f["prediction"]) == [0, 0, 1] and list(f["count"]) == [4, 2, 2]
    assert f["impurity"][0] == 0.5 and f["gain"][0] == 0.5 and list(f["impurity"][1:]) == [0.0, 0.0]


def test_one_split_entropy():
    f = _train([0, 0, 1, 1], [1, 2, 3, 4], impurity="entropy")
    assert f["impurity"][0] == 1.0 and f["gain"][0] == 1.0 and f["threshold"][0] == 2.5


def test_gini_gain_by_hand():
    # x: 1 2 3 4 5, y: 0 0 1 0 1.  parent gini = 1 - .36 - .16 = .48; best split x <= 2.5: left {0,0} pure,
    # right {1,0,1}: gini 1 - 1/9 - 4/9 = 4/9; gain = .48 - 3/5 * 4/9
    f = _train([0, 0, 1, 0, 1], [1, 2, 3, 4, 5], max_depth=1)
    p = 1.0 - 0.6 * 0.6 - 0.4 * 0.4
    r = (1.0 - (1 / 3) * (1 / 3)) - (2 / 3) * (2 / 3)
    assert f["threshold"][0] == 2.5 and f["gain"][0] == (p - (2 / 5) * 0.0) - (3 / 5) * r
    assert list(f["prediction"]) == [0, 0, 1]


def test_tie_between_features_goes_to_the_smaller_feature():
    x = np.array([[1, 1], [2, 2], [3, 3], [4, 4]], float)       # both features split the labels equally well
    f = _train([0, 0, 1, 1], x)
    assert f["feature"][0] == 0
    f = _train([0, 0, 1, 1], x[:, ::-1].copy())
    assert f["feature"][0] == 0


def test_tie_between_classes_goes_to_the_smaller_class():
    f = _train([1, 0], [5, 5], num_classes=3)                   # constant feature: one leaf with counts 1, 1, 0
    assert list(f["feature"]) == [-1] and f["prediction"][0] == 0
    assert fr.predict(f, np.array([[5.0]]))[0] == 0.0


def test_constant_feature_is_never_split():
    x = np.array([[7, 1], [7, 2], [7, 3], [7, 4]], float)
    f = _train([0, 0, 1, 1], x)
    assert f["feature"][0] == 1


def test_max_depth_zero_is_one_leaf():
    f = _train([0, 1, 1], [1, 2, 3], max_depth=0)
    assert list(f["feature"]) == [-1] and f["prediction"][0] == 1 and f["count"][0] == 3 and f["gain"][0] == 0.0


def test_children_with_impurity_zero_are_leaves():
    f = _train([0, 0, 1, 1, 1, 0], [1, 2, 3, 4, 5, 6], max_depth=5)
    assert f["feature"][0] == 0
    assert all(f["impurity"][i] == 0.0 for i in range(len(f["feature"])) if f["feature"][i] < 0)


def test_pruning_collapses_equal_leaves():
    # maxDepth 2: the root splits x <= 2.5; its right child (x 3..8, labels 1 1 0 1 1 1) splits best at x <= 5.5
    # (weighted child gini 3/6 * 4/9 against 4/6 * 3/8 at 4.5) into two leaves at maxDepth that both predict 1, so
    # toNode(prune = true) turns it into a leaf
    y = [0, 0, 1, 1, 0, 1, 1, 1]
    x = np.arange(1, 9, dtype=float)[:, None]
    f, info = fr.train(np.array(y, float), x, 2, 1, "auto", "gini", 2, 32, return_nodes=True)
    nodes = info["trees"][0]
    assert not nodes[3]["leaf"] and nodes[3]["threshold"] == 5.5
    assert nodes[6]["leaf"] and nodes[7]["leaf"] and nodes[6]["prediction"] == nodes[7]["prediction"] == 1
    assert list(f["feature"]) == [0, -1, -1] and list(f["prediction"]) == [1, 0, 1]
    assert f["impurity"][2] == (1.0 - (1 / 6) * (1 / 6)) - (5 / 6) * (5 / 6) and f["count"][2] == 6
    assert list(f["depth"]) == [1]
    assert np.array_equal(fr.predict(f, x), [0, 0, 1, 1, 1, 1, 1, 1])


# ---- thresholds ----------------------------------------------------------------------------------------------------
def test_thresholds_every_midpoint_with_duplicates():
    v, c = np.unique(np.array([3.0, 1.0, 1.0, 2.0, 3.0, -0.0, 0.0]), return_counts=True)
    assert list(fr.thresholds(v, c, 10)) == [0.5, 1.5, 2.5]


def test_thresholds_fewer_distinct_values_than_bins():
    assert list(fr.thresholds(np.array([1.0, 4.0]), np.array([5, 5]), 100)) == [2.5]
    assert list(fr.thresholds(np.array([1.0]), np.array([9]), 100)) == []


def test_thresholds_stride_walk():
    # 10 distinct values, counts 1, numBins 3 -> stride 10/3: the running count is closest to 3.33 at 3 (after value 2)
    # and to 6.67 at 7 (after value 6)
    v = np.arange(10, dtype=float)
    t = fr.thresholds(v, np.ones(10, int), 3)
    assert list(t) == [2.5, 6.5]
    # counts 1, 10, 1, 1, numBins 2 -> stride 6.5: 11 is closer to 6.5 than 12 is; the only midpoint is after value 1
    t = fr.thresholds(np.array([0.0, 1.0, 2.0, 3.0]), np.array([1, 10, 1, 1]), 2)
    assert list(t) == [1.5]


# ---- featureSubsetStrategy -------------------------------------------------------------------------------------------
@pytest.mark.parametrize("s,F,T,k", [
    ("auto", 10, 1, 10), ("auto", 10, 5, 4), ("all", 10, 5, 10), ("sqrt", 10, 1, 4), ("sqrt", 9, 1, 3),
    ("log2", 1, 1, 1), ("log2", 8, 1, 3), ("log2", 9, 1, 4), ("onethird", 10, 1, 4), ("onethird", 9, 1, 3),
    ("1", 10, 1, 1), ("1.0", 10, 1, 10), ("3", 10, 1, 3), ("30", 10, 1, 10), ("0.5", 10, 1, 5), ("0.25", 10, 1, 3),
    (".5", 3, 1, 2), ("5.", 10, 1, 0), ("1.", 10, 1, 10), ("+2", 10, 1, 2), ("1e-1", 10, 1, 1),
    ("0", 10, 1, 0), ("-1", 10, 1, 0), ("1.5", 10, 1, 0), ("0.0", 10, 1, 0), ("x", 10, 1, 0), ("", 10, 1, 0),
    ("Sqrt", 10, 1, 0), ("inf", 10, 1, 0), ("nan", 10, 1, 0), ("2147483648", 10, 1, 0),
])
def test_subset_size(s, F, T, k):
    assert fr.subset_size(s, F, T) == k


# ---- rejections ------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("kw,msg", [
    (dict(num_classes=1), "must have numClasses >= 2, but numClasses = 1."),
    (dict(num_classes=65), "numClasses = 65: at most 64 classes are supported."),
    (dict(num_trees=0), "RandomForest requires numTrees > 0, but was given numTrees = 0."),
    (dict(strategy="half"), "RandomForest given invalid featureSubsetStrategy: half. Supported values: auto, all, "
                            "onethird, sqrt, log2, (0.0-1.0], [1-n]."),
    (dict(max_depth=-1), "invalid maxDepth parameter: -1.  Valid values are integers >= 0."),
    (dict(max_depth=31), "only supports maxDepth <= 30, but was given maxDepth = 31."),
    (dict(max_bins=1), "invalid maxBins parameter: 1.  Valid values are integers >= 2."),
    (dict(max_bins=65537), "maxBins = 65537: at most 65536 bins are supported."),
    (dict(impurity="variance"), "Did not recognize Impurity name: variance"),
    (dict(categorical={0: 2}), "categoricalFeaturesInfo must be empty"),
])
def test_argument_rejections(kw, msg):
    with pytest.raises(ValueError) as e:
        _train([0, 1], [1, 2], **kw)
    assert msg in str(e.value)


@pytest.mark.parametrize("y,x,imp,msg", [
    ([0, 2], [1, 2], "gini", "GiniAggregator given label 2.0 but requires label < numClasses (= 2)."),
    ([0, 7.5], [1, 2], "entropy", "EntropyAggregator given label 7.5 but requires label < numClasses (= 2)."),
    ([-0.5, 1], [1, 2], "gini", "GiniAggregator given label -0.5but requires label is non-negative."),
    ([0, np.nan], [1, 2], "gini", "label of row 1 is not finite (nan)."),
    ([5, 1], [1, np.inf], "gini", "feature 0 of row 1 is not finite (inf)."),
])
def test_label_and_value_rejections(y, x, imp, msg):
    with pytest.raises(ValueError) as e:
        _train(y, x, impurity=imp)
    assert str(e.value) == msg


def test_fractional_labels_truncate():
    f = _train([0.9, 0.2, 1.7, 1.1], [1, 2, 3, 4])
    assert list(f["prediction"]) == [0, 0, 1]


# ---- forest_splits.h against the restatement ------------------------------------------------------------------------
DRIVER = r"""
#include <cstdio>
#include <cstring>
#include <iostream>
#include <string>
#include <vector>
#include "forest_splits.h"
using namespace pio;
int main() {
  std::string cmd;
  while (std::cin >> cmd) {
    if (cmd == "subset") {            // subset <strategy|-> F T
      std::string s; int F, T;
      std::cin >> s >> F >> T;
      if (s == "-") s = "";
      std::printf("%d\n", rf_subset_size(s.c_str(), F, T));
    } else if (cmd == "thr") {        // thr nb m v0 c0 v1 c1 ...  (values as hex bits)
      long long nb, m;
      std::cin >> nb >> m;
      std::vector<double> v(m); std::vector<int64_t> c(m);
      for (long long i = 0; i < m; ++i) { unsigned long long b; std::cin >> std::hex >> b >> std::dec >> c[i]; std::memcpy(&v[i], &b, 8); }
      std::vector<double> out;
      rf_thresholds(v.data(), c.data(), m, nb, out);
      std::printf("%zu", out.size());
      for (double t : out) { unsigned long long b; std::memcpy(&b, &t, 8); std::printf(" %llx", b); }
      std::printf("\n");
    } else if (cmd == "poisson") {
      double cdf[RF_POISSON_N];
      rf_poisson_table(cdf);
      for (double t : cdf) { unsigned long long b; std::memcpy(&b, &t, 8); std::printf("%llx ", b); }
      std::printf("\n");
    } else if (cmd == "bag") {        // bag seed t n
      long long seed, t, n;
      std::cin >> seed >> t >> n;
      double cdf[RF_POISSON_N];
      rf_poisson_table(cdf);
      const uint64_t base = rf_stream(seed, RF_TAG_BAG, (uint64_t)t);
      for (long long r = 0; r < n; ++r) std::printf("%d ", rf_bag_weight(cdf, base, (uint64_t)r));
      std::printf("\n");
    } else if (cmd == "sample") {     // sample seed n max_bins
      long long seed, n; int mb;
      std::cin >> seed >> n >> mb;
      const double frac = rf_sample_fraction(n, mb);
      const uint64_t base = rf_stream(seed, RF_TAG_SAMPLE, 0);
      long long m = 0;
      for (long long r = 0; r < n; ++r) m += rf_sampled(base, (uint64_t)r, frac) ? 1 : 0;
      unsigned long long b; std::memcpy(&b, &frac, 8);
      std::printf("%llx %lld\n", b, m);
    } else if (cmd == "node") {       // node seed t heap F k
      long long seed, t, heap; int F, k;
      std::cin >> seed >> t >> heap >> F >> k;
      std::vector<int> out(F);
      rf_node_subset(rf_stream(seed, RF_TAG_SUBSET, (uint64_t)t), heap, F, k, out.data());
      for (int i = 0; i < (k < F ? k : F); ++i) std::printf("%d ", out[i]);
      std::printf("\n");
    } else if (cmd == "imp") {        // imp kind C c0 c1 ...
      int kind, C;
      std::cin >> kind >> C;
      std::vector<int64_t> c(C);
      for (auto& v : c) std::cin >> v;
      const double r = rf_impurity(c.data(), C, kind);
      unsigned long long b; std::memcpy(&b, &r, 8);
      std::printf("%llx\n", b);
    } else if (cmd == "groups") {     // groups T n budget per_pass
      long long T, n, budget; int pp;
      std::cin >> T >> n >> budget >> pp;
      for (auto& g : rf_plan_groups((int)T, n, budget, pp)) std::printf("%d:%d ", g.first, g.second);
      std::printf("\n");
    }
  }
}
"""


def _bits(v):
    return int(np.float64(v).view(np.uint64))


@pytest.fixture(scope="module")
def splits(tmp_path_factory):
    if shutil.which("g++") is None:
        pytest.skip("needs g++")
    d = tmp_path_factory.mktemp("forest_splits")
    (d / "driver.cpp").write_text(DRIVER)
    exe = d / "driver"
    subprocess.run(["g++", "-std=c++17", "-Wall", "-Wextra", "-Werror", "-O2", "-I", str(CSRC), "-o", str(exe),
                    str(d / "driver.cpp")], check=True)

    def run(lines):
        out = subprocess.run([str(exe)], input="\n".join(lines) + "\n", capture_output=True, text=True, check=True)
        return out.stdout.splitlines()
    return run


def test_splits_subset_sizes(splits):
    cases = [(s, F, T) for s in ("auto", "all", "sqrt", "log2", "onethird", "1", "1.0", "2", "0.3", "1e-1", ".5",
                                  "5.", "+3", "-3", "0", "0.0", "1.01", "x", "-", "Sqrt", "2147483648",
                                  "00000000001", "1e400", "inf")
             for F in (1, 2, 3, 7, 8, 9, 100, 1000) for T in (1, 5)]
    got = splits([f"subset {s} {F} {T}" for s, F, T in cases])
    want = [str(fr.subset_size("" if s == "-" else s, F, T)) for s, F, T in cases]
    assert got == want


def test_splits_thresholds(splits):
    rng = np.random.default_rng(5)
    cases = []
    for _ in range(60):
        vals = np.unique(np.round(rng.normal(size=rng.integers(1, 300)) * rng.choice([1, 10, 1000]), rng.integers(0, 4)))
        cnt = rng.integers(1, 20, vals.size)
        cases.append((int(rng.choice([2, 3, 5, 32, 100, 400])), vals, cnt))
    lines = [f"thr {nb} {v.size} " + " ".join(f"{_bits(a):x} {c}" for a, c in zip(v, cnt)) for nb, v, cnt in cases]
    got = splits(lines)
    for (nb, v, cnt), line in zip(cases, got):
        want = fr.thresholds(v, cnt, nb)
        parts = line.split()
        assert int(parts[0]) == want.size
        assert [int(p, 16) for p in parts[1:]] == [_bits(t) for t in want]


def test_splits_poisson_and_draws(splits):
    got = splits(["poisson", "bag 7 0 2000", "bag 7 3 2000", "bag -5 1 50", "sample 3 50000 32", "sample 3 9000 32",
                  "sample 11 200000 100", "node 1 0 1 10 3", "node 1 4 77 10 3", "node 9 2 5 1000 32",
                  "node 9 2 5 5 5"])
    assert [int(h, 16) for h in got[0].split()] == [_bits(c) for c in fr.poisson_table()]
    for line, (seed, t, n) in zip(got[1:4], [(7, 0, 2000), (7, 3, 2000), (-5, 1, 50)]):
        assert [int(w) for w in line.split()] == list(fr.bag_weights(seed, t, n))
    w = fr.bag_weights(7, 0, 200000)
    assert abs(w.mean() - 1.0) < 0.01 and w.max() <= 16
    for line, (seed, n, mb) in zip(got[4:7], [(3, 50000, 32), (3, 9000, 32), (11, 200000, 100)]):
        frac = fr.sample_fraction(n, mb)
        m = n if frac >= 1 else int((fr.u53(fr.draw(fr.stream(seed, fr.TAG_SAMPLE, 0), np.arange(n, dtype=np.uint64)))
                                    < frac).sum())
        assert line.split() == [f"{_bits(frac):x}", str(m)]
    for line, (seed, t, heap, F, k) in zip(got[7:], [(1, 0, 1, 10, 3), (1, 4, 77, 10, 3), (9, 2, 5, 1000, 32),
                                                     (9, 2, 5, 5, 5)]):
        assert [int(v) for v in line.split()] == list(fr.node_subset(seed, t, heap, F, k))


def test_splits_impurity_and_groups(splits):
    rng = np.random.default_rng(2)
    cases = [(kind, rng.integers(0, rng.choice([2, 50, 10 ** 6]), rng.integers(2, 65))) for kind in (0, 1)
             for _ in range(40)]
    cases += [(0, np.zeros(4, int)), (1, np.array([0, 3, 0]))]
    got = splits([f"imp {kind} {c.size} " + " ".join(map(str, c)) for kind, c in cases])
    for (kind, c), line in zip(cases, got):
        assert int(line, 16) == _bits(fr.impurity_of(c, kind))
    got = splits(["groups 100 10000000 1073741824 0", "groups 5 10 1073741824 0", "groups 64 1000 0 1",
                  "groups 7 1000 4000000000 3"])
    assert got[0].split()[:2] == ["0:26", "26:52"] and got[0].split()[-1] == "78:100"
    assert got[1] == "0:5 " and got[2].split()[5] == "5:6" and got[3] == "0:3 3:6 6:7 "
