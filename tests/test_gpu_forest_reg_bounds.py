"""GPU tests (-m gpu) of the RandomForest regressor (pio_rf_train_regressor / pio_rf_predict_regression) at the
boundaries of its own code: continuous features with more bins than one 256-wide block scan and on both sides of the
shared-memory histogram, label sums past 2^64 (both signs, bagged, cancelling), trees 30 levels deep, label quantisation
at its extremes and ties, equal and Double.MaxValue centroids across the in-block / multi-block category ranking and
its 2048-wide tiles, wide categorical features under histogram chunks and tree groups, ties between duplicated
features, and predictions on NaN, infinities, signed zeros, the ends of int32, fractional categories and every
threshold give or take one ulp.  Plus the lead scoring sessions (pio_lead_sessions) under contention and at the ends of
the int64 range.

Every case trains through mllib.RandomForest.trainRegressor and must equal the restatement tests/forest_reg_ref.py node
for node (doubles bit for bit), predict on the training rows and on held-out rows must equal the restatement's,
native.rf_train_paths() must be the record tests/test_forest_reg_paths.py predicts, and each fixture must show in the
restatement that it reaches what it is named after.  tests/test_forest_reg_paths.py (CPU) checks that the cases still
straddle every boundary."""
import functools
from collections import namedtuple

import numpy as np
import pytest

from pio_b200 import mllib
from pio_b200 import native
from tests import forest_ref as fr
from tests import forest_reg_ref as rr
from tests.test_gpu_forest_bounds import _held_near, _rng, ties_to_smaller_copy
from tests.test_gpu_forest_reg import _assert_same

pytestmark = pytest.mark.gpu

# make() -> (labels, x, {feature: arity}, held-out x); budget: PIO_RF_HIST_BUDGET (None: the default); check(forest,
# info, y, x): what the restatement's forest must show for the case to test what it is named after
Case = namedtuple("Case", "name make T strategy depth bins budget seed check", defaults=(None,))

PREDICT_ROWS = 3000            # training rows predicted (a subsample above this: the restatement walks rows in Python)
N_BIG = (1 << 22) + 4099       # rows whose label sums pass 2^64


# ---- fixtures -------------------------------------------------------------------------------------------------------
def bins(m, seed, tie=False, rows=4):
    """One continuous feature of m distinct values (m - 1 thresholds, m bins), `rows` rows each.  tie: labels exactly 0
    on the first a1 and the last a2 values (equal row counts) and about 10 on the 256 values between, so the root's two
    best splits have bit-equal gains 256 positions apart, in one thread of the block scan; else labels wander."""
    def make():
        rng = _rng(seed)
        vals = np.arange(m) * 0.5 - 7.0
        cnt = np.full(m, rows)
        if tie:
            a1 = (m - 256) // 2
            a2 = m - 256 - a1
            cnt[0] += (a2 - a1) * rows                   # the two zero blocks hold the same number of rows
            per_row = np.repeat(np.arange(m), cnt)
            y = np.where((per_row < a1) | (per_row >= m - a2), 0.0, 10.0 + rng.normal(size=per_row.size))
        else:
            per_row = np.repeat(np.arange(m), cnt)
            walk = np.cumsum(rng.normal(size=m))
            y = walk[per_row] + 0.5 * rng.normal(size=per_row.size)
        x = vals[per_row][:, None]
        perm = rng.permutation(per_row.size)
        x, y = x[perm], y[perm]
        return y, x, {}, _held_near(x, m, 0)
    return make


def tie_zero_blocks(m):
    """The root's best gain is shared by the split after the first zero block and the one before the last, 256
    positions apart; the first is taken."""
    def check(want, info, y, x):
        a1 = (m - 256) // 2
        a2 = m - 256 - a1
        g = _root_gains(y, x[:, 0], info, m)
        assert g[a1 - 1] == g[m - 1 - a2] == g.max() and g.argmax() == a1 - 1
        assert want["threshold"][0] == info["thresholds"][0][a1 - 1]
    return check


def _root_gains(y, col, info, m):
    """Gains of every candidate of a one-tree root on one continuous feature (all rows, weight 1)."""
    yq, s = rr.quantize(y)
    b = np.searchsorted(info["thresholds"][0], col, side="left")
    W, S, Q = rr._node_stats(b, np.ones(len(y), object), np.array(yq, object),
                             np.array([v * v for v in yq], object), m)
    return rr._gains(np.cumsum(W), np.cumsum(S), np.cumsum(Q), s, m - 1)


# the sticky bit of a 65-bit |S|: its low 13 bits 0b0_1000_0000_0001 are a tie on the top 64 bits with the last kept
# bit even, which only the sticky bit rounds up
STICKY_LOW, STICKY_MASK = 0x801, 0x1FFF


def big_sums(sign, T, seed, mixed=False):
    """N_BIG rows of one 8-category feature (category 7 on over half of them), labels -(0.75 + 0.25 u) 2^20 - 0.37 x with full mantissas (times sign,
    or a random sign each when mixed): |sum w yq| of the root passes 2^64 (mixed: it cancels while sum w yq^2 passes
    2^100).  One row's label moves by a few units of 2^-s so that the root's |S| of tree 0 ends in STICKY_LOW."""
    def make():
        rng = _rng(seed)
        xc = rng.integers(0, 8, N_BIG)
        xc[rng.random(N_BIG) < 0.5] = 7                # over half the rows: the child holding them passes 2^64 too
        y = -(0.75 + 0.25 * rng.random(N_BIG)) * 2.0 ** 20 - 0.37 * xc
        if mixed:
            y *= np.where(rng.random(N_BIG) < 0.5, -1.0, 1.0)
        y *= sign
        x = xc.astype(np.float64)[:, None]
        if not mixed:
            w = np.ones(N_BIG, np.int64) if T == 1 else fr.bag_weights(seed, 0, N_BIG)
            s, yq, S = label_sums(y, w)
            k = (STICKY_LOW - (abs(S) & STICKY_MASK)) % (STICKY_MASK + 1)
            r = int(np.flatnonzero((w == 1) & (np.abs(yq) < (1 << 43)))[0])
            y[r] = float(int(yq[r]) + (k if S > 0 else -k)) * 2.0 ** -s
        held = np.concatenate([x[:200], np.array([[-0.0], [7.5], [8.0], [np.nan]])])
        return y, x, {0: 8}, held
    return make


def label_sums(y, w):
    """(s, yq, exact sum of w yq) of labels y and integer weights w, as the restatement quantises them."""
    m = float(np.abs(y).max())
    s = rr.LABEL_BITS - np.frexp(m)[1]
    yq = np.rint(np.ldexp(y, s)).astype(np.int64)
    S = 0
    for r0 in range(0, len(y), 1 << 14):               # |w yq| <= 2^48: int64 block sums of 2^14 rows stay below 2^62
        S += int(np.sum(w[r0:r0 + (1 << 14)] * yq[r0:r0 + (1 << 14)]))
    return s, yq, S


def s_past_2_64(sticky):
    """The root's |S| of tree 0 has 65 bits (and a child's too), with the sticky-bit tie when `sticky`."""
    def check(want, info, y, x):
        nodes = info["trees"][0]
        root = nodes[1]["stats"][1]
        assert abs(root).bit_length() == 65
        assert max(abs(nodes[i]["stats"][1]).bit_length() for i in (2, 3)) == 65
        if sticky:
            assert abs(root) & STICKY_MASK == STICKY_LOW
    return check


def s_cancels(want, info, y, x):
    W, S, Q = info["trees"][0][1]["stats"]
    assert abs(S) < 2 ** 64 < 2 ** 100 < Q


def comb_geometric(n):
    """x = 0 .. n - 1 with labels 2.55^(n - 1 - x): each level peels the smallest x off to the left, so the surviving
    node is always a right child and the heap indices run 2^(d+1) - 1 up to 2^31 - 1.  (Ratio 2 peels two rows at some
    levels; 3 quantises the smallest labels to 0 before depth 30.)"""
    def make():
        x = np.arange(float(n))[:, None]
        y = 2.55 ** (n - 1 - np.arange(n))
        return y, x, {}, np.arange(-0.5, n + 0.5, 0.25)[:, None]
    return make


def reaches_depth_30(want, info, y, x):
    assert want["depth"].max() == 30
    assert max(info["trees"][0]) > 2 ** 30


def _cat_labels(n, arity, seed, scale=1.0, halves=False):
    """A categorical column of `arity` categories and a continuous one, and labels from both."""
    rng = _rng(seed)
    c = rng.integers(0, arity, n).astype(np.float64)
    v = np.round(rng.normal(size=n) * 3, 1)
    y = np.sin(c * 0.9) * 3 + 0.4 * v + rng.normal(size=n) * 0.3
    if halves:
        y = np.round(y * 2) / 2
    return y * scale, np.column_stack([c, v])


def labels(kind, seed=31):
    """Quantisation edges: the accepted extremes, a maximum that rounds to 2^44, exact half-way ties, subnormals next to
    a normal maximum."""
    def make():
        y, x = _cat_labels(3000, 6, seed, halves=kind == "ties")
        rng = _rng(seed + 1)
        if kind == "min":
            y = y / np.abs(y).max() * 2.0 ** -256                     # max |y| = 2^-256 exactly
        elif kind == "max":
            y = y / np.abs(y).max() * np.nextafter(2.0 ** 256, 0)     # just below 2^256
        elif kind == "round_to_2_44":
            top = np.nextafter(2.0, 0.0)                               # y 2^43 = 2^44 - 2^-9: rounds to 2^44
            y = np.clip(y / np.abs(y).max() * 2.0, -top, top)
            y[rng.integers(0, 3000, 40)] = top
            y[rng.integers(0, 3000, 40)] = -top
        elif kind == "ties":
            y = y + 0.5 * (rng.random(3000) < 0.5)                     # y 2^0 on .5: half-way ties
            y[7] = 2.0 ** 43 + 0.5                                     # max |y| in [2^43, 2^44): s = 0
        elif kind == "subnormal":
            tiny = float.fromhex("0x0.0000000000001p-1022")
            y = y / np.abs(y).max()
            y[rng.integers(0, 3000, 300)] = tiny
            y[rng.integers(0, 3000, 300)] = -tiny
            y[rng.integers(0, 3000, 300)] = float.fromhex("0x1p-1022")
            y[5] = 1.0
        return y, x, {0: 6}, _held(x, 6)
    return make


def quantisation(kind):
    def check(want, info, y, x):
        yq, s = rr.quantize(y)
        if kind == "min":
            assert np.abs(y).max() == 2.0 ** -256 and s == 44 + 255
        elif kind == "max":
            assert np.abs(y).max() == np.nextafter(2.0 ** 256, 0) and s == 44 - 256
        elif kind == "round_to_2_44":
            assert max(abs(v) for v in yq) == 2 ** 44 and s == 43
            w = [fr.bag_weights(5, t, len(y)) for t in range(5)]
            assert max(int(wt[np.abs(y) == np.abs(y).max()].max()) for wt in w) >= 4
        elif kind == "ties":
            assert s == 0
            half = np.ldexp(y, s) % 1 == 0.5
            assert half.sum() > 500 and (np.rint(np.ldexp(y, s))[half] % 2 == 0).all()
        elif kind == "subnormal":
            assert (np.abs(y[y != 0]).min() < 2.0 ** -1022) and sum(v == 0 for v in yq) > 300
    return check


def flat_labels(value, n=2000):
    def make():
        y, x = _cat_labels(n, 5, 41)
        return np.full(n, value), x, {0: 5}, _held(x, 5)
    return make


def leaves_only(want, info, y, x):
    assert (want["feature"] == -1).all() and want["feature"].size == want["tree_off"].size - 1


def inexact_constant(want, info, y, x):
    assert info["trees"][0][1]["impurity"] != 0.0


def exact_children():
    """Categories of constant labels with full mantissas and odd row counts: a constant child's fp64 impurity
    (Q - S S / W) / W comes out 0 for some and tiny or negative for others."""
    def make():
        rng = _rng(51)
        a = 12
        lab = rng.uniform(1.0, 2.0, a) * 1.0e5
        cnt = rng.integers(3, 40, a)
        cnt[0] = 32
        c = np.repeat(np.arange(a), cnt).astype(np.float64)
        y = lab[c.astype(np.int64)]
        x = np.column_stack([c, np.round(rng.normal(size=c.size), 1)])
        perm = rng.permutation(c.size)
        return y[perm], x[perm], {0: a}, _held(x, a)
    return make


def impurity_rule_both_ways(want, info, y, x):
    exact = [(r["impurity"], r["leaf"]) for nodes in info["trees"] for r in nodes.values()
             if r["stats"][0] * r["stats"][2] == r["stats"][1] ** 2]
    assert any(imp == 0.0 for imp, _ in exact)
    assert any(imp != 0.0 for imp, _ in exact)


def _held(x, arity):
    """Held-out rows: training rows, and the first column at fractional, negative and out-of-range values."""
    h = np.concatenate([x[:100]] * 2)
    h[100:, 0] = np.concatenate([np.arange(-1.0, arity + 1.0, 0.5), np.full(100, np.nan)])[:100]
    return h


def equal_centroids(arity, seed):
    """One categorical feature of `arity` categories, three rows each except a few empty ones: a category's labels are
    the pattern of its group c % 5, so the groups' centroids are exactly equal, and categories 2047 / 2048 (and 4095 /
    4096) share a group, while 2046 / 2049 and 4094 / 4097 are empty (Double.MaxValue ties)."""
    def make():
        rng = _rng(seed)
        pat = rng.normal(size=(5, 3)) * 2 + np.arange(5)[:, None]
        cats = np.array([c for c in range(arity) if c not in (2046, 2049, 4094, 4097) and c % 97 != 13])
        grp = np.where(np.isin(cats, (2048, 4096)), cats - 1, cats) % 5
        c = np.repeat(cats, 3).astype(np.float64)
        y = pat[np.repeat(grp, 3), np.tile(np.arange(3), cats.size)]
        v = np.round(rng.normal(size=c.size) * 2, 1)
        x = np.column_stack([c, v])
        perm = rng.permutation(c.size)
        return y[perm], x[perm], {0: arity}, _held(x, arity)
    return make


def straddling_ties(arity):
    def check(want, info, y, x):
        W, S, _ = rr._node_stats(x[:, 0].astype(np.int64), np.ones(len(y), object),
                                 np.array(rr.quantize(y)[0], object), np.zeros(len(y), object), arity)
        cen = np.array([float(s) / float(w) if w else rr.DMAX for w, s in zip(W, S)])
        for b in (2048, 4096):
            if b < arity:
                assert W[b - 1] > 0 and cen[b - 1] == cen[b]
                assert W[b - 2] == 0 and (b + 1 >= arity or W[b + 1] == 0)
    return check


def one_category_nodes(seed=61):
    """Six regions of a continuous column; in each, the categorical columns (arities 40 and 3000) take one category,
    so every node below a region split has one non-empty category and arity - 1 Double.MaxValue ties."""
    def make():
        rng = _rng(seed)
        n = 3000
        v = rng.uniform(0, 6, n)
        reg = np.floor(v).astype(np.int64)
        c0 = (reg * 7 + 3).astype(np.float64)
        c1 = (reg * 450 + 500).astype(np.float64)
        y = np.sin(v * 2.1) * 4 + reg + rng.normal(size=n) * 0.2
        x = np.column_stack([c0, c1, np.round(v, 2)])
        held = np.concatenate([x[:200], np.array([[3.0, 999.0, 2.5], [-0.0, 2999.0, 0.0], [40.0, 3000.0, 7.0]])])
        return y, x, {0: 40, 1: 3000}, held
    return make


def single_category_split(want, info, y, x):
    """Some split below the root runs on rows of one category of feature 1."""
    paths = _paths(want, x)
    below = [i for i in range(1, want["tree_off"][1]) if want["feature"][i] >= 0]
    assert any(np.unique(x[paths[:, i], 1]).size == 1 for i in below)


def _paths(forest, x):
    """[n, nodes of tree 0]: whether each row passes through each node."""
    n = x.shape[0]
    out = np.zeros((n, forest["tree_off"][1]), bool)
    feat, thr, lft, rgt = forest["feature"], forest["threshold"], forest["left"], forest["right"]
    co, ci = forest["cat_off"], forest["cat_ids"]
    for r in range(n):
        i = 0
        while True:
            out[r, i] = True
            if feat[i] < 0:
                break
            v = x[r, feat[i]]
            go = bool(np.any(ci[co[i]:co[i + 1]] == v)) if co[i + 1] > co[i] else v <= thr[i]
            i = int(lft[i] if go else rgt[i])
    return out


def wide_pair(seed=71):
    """Categorical columns of arities 3000 and 5000 and a continuous one, about three rows per category."""
    def make():
        rng = _rng(seed)
        n = 16000
        c0 = rng.integers(0, 3000, n)
        c1 = rng.integers(0, 5000, n)
        v = np.round(rng.normal(size=n) * 3, 1)
        y = np.sin(c0 * 0.37) * 2 + np.cos(c1 * 0.11) * 2 + 0.3 * v + rng.normal(size=n) * 0.2
        x = np.column_stack([c0, c1, v]).astype(np.float64)
        return y, x, {0: 3000, 1: 5000}, _held(x, 3000)
    return make


def copies(F, dups, n=1000, seed=81):
    """F continuous columns where column b copies column a for each (a, b) in dups."""
    def make():
        rng = _rng(seed)
        x = np.round(rng.normal(size=(n, F)) * 3, 1)
        for a, b in dups:
            x[:, b] = x[:, a]
        y = x[:, 0] - 0.8 * x[:, 3] + 0.4 * x[:, 1] + rng.normal(size=n)
        return y, x, {}, np.round(rng.normal(size=(300, F)) * 3, 1)
    return make


def copy_ties(to, seed, n_feat):
    """No split uses a copy while an earlier copy of the same column was in the node's subset, and some split had a later
    copy beside it (tests/test_gpu_forest_bounds.ties_to_smaller_copy)."""
    check = ties_to_smaller_copy(lambda f: to.get(f, f), seed, n_feat, n_feat)
    return lambda want, info, y, x: check(want, info, None)


def predict_edges(seed=91):
    """A categorical column trained on fractional (2.5, 4.25) and signed-zero values and a continuous one; held-out
    rows at NaN, +-inf, -0.0, 2^31 - 1, 2^31, fractional categories and every threshold give or take one ulp."""
    def make():
        rng = _rng(seed)
        n = 4000
        c = rng.integers(0, 6, n).astype(np.float64)
        c[rng.random(n) < 0.1] = 2.5
        c[rng.random(n) < 0.1] = 4.25
        c[(c == 0) & (rng.random(n) < 0.5)] = -0.0
        v = np.round(rng.normal(size=n) * 2, 2)
        y = np.where(np.trunc(c) % 2 == 0, 3.0, -1.0) + 0.7 * v + rng.normal(size=n) * 0.2
        x = np.column_stack([c, v])
        near = _held_near(x, 64, 0)
        edge = np.array([np.nan, np.inf, -np.inf, -0.0, 0.0, 2.0 ** 31 - 1, 2.0 ** 31, 2.5, 4.25, 0.5, 5.0, 6.0, -1.0,
                         -2.0 ** 31, 1e300])
        e = np.array(np.meshgrid(edge, edge)).reshape(2, -1).T
        return y, x, {0: 6}, np.concatenate([near, e])
    return make


# ---- cases ----------------------------------------------------------------------------------------------------------
CASES = [
    # continuous bins (K = 1): 255 / 256 uint8, 257 uint16 codes from thresholds alone; 512 / 513 two block-scan tiles;
    # 2457 bins = 98 280 B of 40-byte entries in a 96 KiB shared histogram, 2458 the global one
    Case("nb255", bins(255, 1), 1, "all", 9, 255, None, 0),
    Case("nb256_uint8", bins(256, 2), 1, "all", 9, 256, None, 0),
    Case("nb257_uint16", bins(257, 3), 1, "all", 9, 257, None, 0),
    Case("nb512_tie", bins(512, 4, tie=True), 1, "all", 8, 512, None, 0, tie_zero_blocks(512)),
    Case("nb513", bins(513, 5), 1, "all", 8, 513, None, 0),
    Case("nb2457_smem", bins(2457, 6, tie=True), 1, "all", 6, 2457, None, 0, tie_zero_blocks(2457)),
    Case("nb2458_global", bins(2458, 7, tie=True), 1, "all", 6, 2458, None, 0, tie_zero_blocks(2458)),
    # label sums past 2^64: negative, positive, bagged (weights up to 16 in the 128-bit sums), cancelling
    Case("sums_negative", big_sums(1.0, 1, 101), 1, "all", 3, 32, None, 0, s_past_2_64(True)),
    Case("sums_positive", big_sums(-1.0, 1, 101), 1, "all", 3, 32, None, 0, s_past_2_64(True)),
    Case("sums_bagged", big_sums(1.0, 3, 102), 3, "all", 3, 32, None, 102, s_past_2_64(True)),
    Case("sums_cancel", big_sums(1.0, 1, 103, mixed=True), 1, "all", 3, 32, None, 0, s_cancels),
    # depth 30, heap indices up to 2^31 - 1
    Case("depth30", comb_geometric(40), 1, "all", 30, 64, None, 0, reaches_depth_30),
    # quantisation: extremes, a maximum rounding to 2^44 (bagged), half-way ties, subnormals, zero and constant labels,
    # constant children whose fp64 impurity is and is not 0
    Case("label_min", labels("min"), 3, "all", 5, 32, None, 1, quantisation("min")),
    Case("label_max", labels("max"), 3, "all", 5, 32, None, 1, quantisation("max")),
    Case("label_round_to_2_44", labels("round_to_2_44"), 5, "all", 5, 32, None, 5, quantisation("round_to_2_44")),
    Case("label_ties", labels("ties"), 3, "all", 5, 32, None, 1, quantisation("ties")),
    Case("label_subnormal", labels("subnormal"), 3, "all", 5, 32, None, 1, quantisation("subnormal")),
    Case("labels_zero", flat_labels(0.0), 3, "all", 5, 32, None, 1, leaves_only),
    Case("labels_constant", flat_labels(-3.0), 3, "all", 5, 32, None, 1, leaves_only),
    # 3001 rows of 0.3 (a full mantissa): the fp64 impurity of the constant root is not 0
    Case("labels_constant_inexact", flat_labels(0.3, 3001), 1, "all", 4, 32, None, 0, inexact_constant),
    Case("exact_children", exact_children(), 1, "all", 6, 32, None, 0, impurity_rule_both_ways),
    # category order: equal centroids across categories 2048 / 4096 (rank tiles), one-category nodes
    Case("ties_arity4097", equal_centroids(4097, 111), 1, "all", 4, 4097, None, 0, straddling_ties(4097)),
    Case("ties_arity6000", equal_centroids(6000, 112), 2, "all", 4, 6000, None, 2, straddling_ties(6000)),
    Case("one_category_nodes", one_category_nodes(), 1, "all", 6, 3000, None, 0, single_category_split),
    # 300 subset features with copies: equal gains go to the earlier subset position
    Case("k300_copies", copies(300, [(0, 150), (3, 4), (1, 299), (0, 201), (3, 17)]), 2, "all", 4, 32, None, 1,
         copy_ties({150: 0, 4: 3, 299: 1, 201: 0, 17: 3}, 1, 300)),
    # predict edges
    Case("predict_edges", predict_edges(), 3, "all", 6, 64, None, 3),
]


def _train_ref(case, y, x, cat):
    return rr.train(y, x, case.T, case.strategy, "variance", case.depth, case.bins, seed=case.seed, categorical=cat,
                    return_nodes=True)


def _predict_rows(x, held, seed):
    rows = x if x.shape[0] <= PREDICT_ROWS else x[np.sort(_rng(seed).choice(x.shape[0], PREDICT_ROWS, replace=False))]
    return np.concatenate([rows, held])


def run_case(case, monkeypatch, per_pass=None, made=None, ref=None):
    from tests import test_forest_reg_paths as P
    y, x, cat, held = made or case.make()
    for k, v in (("PIO_RF_HIST_BUDGET", case.budget), ("PIO_RF_TREES_PER_PASS", per_pass)):
        if v is None:
            monkeypatch.delenv(k, raising=False)
        else:
            monkeypatch.setenv(k, str(v))
    m = mllib.RandomForest.trainRegressor(y, x, cat, case.T, case.strategy, "variance", case.depth, case.bins,
                                          seed=case.seed)
    got_paths = native.rf_train_paths()
    want, info = ref or _train_ref(case, y, x, cat)
    _assert_same(m.nodes, want)
    assert got_paths == P.expected_record(case, x, cat, info["level_slots"], per_pass), case.name
    q = _predict_rows(x, held, case.seed)
    np.testing.assert_array_equal(m.predictBatch(q).view(np.uint64), rr.predict(want, q).view(np.uint64))
    return m, want, info, (y, x, cat, held)


@pytest.mark.parametrize("case", CASES, ids=[c.name for c in CASES])
def test_regressor_at_boundary(case, monkeypatch):
    _, want, info, (y, x, _, _) = run_case(case, monkeypatch)
    if case.check is not None:
        case.check(want, info, y, x)


def test_arity_2048_and_2049_give_the_same_forest(monkeypatch):
    """The same rows at arity 2048 (ordered inside select_var_kernel) and 2049 with category 2048 empty (ordered by
    cat_centroid_kernel + cat_rank_kernel): identical forests, without trusting the restatement."""
    y, x, _, held = equal_centroids(2048, 121)()
    forests = []
    for a in (2048, 2049):
        case = Case(f"arity{a}", None, 2, "all", 5, 4096, None, 4)
        m, _, _, _ = run_case(case, monkeypatch, made=(y, x, {0: a}, held))
        forests.append(m.nodes)
    _assert_same(forests[1], forests[0])


WIDE = wide_pair()
# K NB (40 + 4 + 8) = 3 x 5000 x 52 = 780 000 bytes a slot: one and two slots a chunk
WIDE_SLOT = 3 * 5000 * 52
WIDE_CASES = [Case(f"wide_budget{b}", WIDE, 4, "all", 4, 5000, b * WIDE_SLOT, 6) for b in (1, 2)]


@functools.lru_cache(maxsize=1)
def _wide_ref():
    y, x, cat, held = WIDE()
    return (y, x, cat, held), _train_ref(WIDE_CASES[0], y, x, cat)


@pytest.mark.parametrize("per_pass", [1, 2, 3])
@pytest.mark.parametrize("slots", [1, 2])
def test_wide_categories_under_chunks_and_groups(monkeypatch, per_pass, slots):
    made, ref = _wide_ref()
    case = WIDE_CASES[slots - 1]
    run_case(case, monkeypatch, per_pass=per_pass, made=made, ref=ref)
    paths = native.rf_train_paths()
    assert paths["max_chunks"] >= 3 and paths["groups"] == -(-case.T // per_pass)


# ---- lead scoring sessions ------------------------------------------------------------------------------------------
def sessions_ref(sess, is_buy, t, n_sessions):
    """tests/leadscoring_ref.py's rule in NumPy: per session the earliest view time, the last event among the views at
    that time (-1: no view), and whether some buy is strictly after it."""
    landing = np.full(n_sessions, -1, np.int64)
    buy = np.zeros(n_sessions, bool)
    v = np.flatnonzero(is_buy == 0)
    if v.size:
        order = np.lexsort((-v, t[v], sess[v]))          # by session, then time, then the later event first
        vs = v[order]
        first = np.r_[True, sess[vs][1:] != sess[vs][:-1]]
        landing[sess[vs[first]]] = vs[first]
    b = np.flatnonzero(is_buy != 0)
    has = landing[sess[b]] >= 0
    after = t[b] > np.where(has, t[landing[sess[b]].clip(0)], 0)
    buy[sess[b[has & after]]] = True
    return landing, buy


def _sessions(kind, seed):
    rng = _rng(seed)
    i64 = np.iinfo(np.int64)
    if kind == "contended":
        n, ns = 1 << 20, 300
        sess = rng.integers(0, ns, n)
        t = rng.integers(-5000, 5000, n)
    elif kind == "same_ms":
        n, ns = 200000, 40
        sess = rng.integers(0, ns, n)
        t = np.where(rng.random(n) < 0.9, 1234567, rng.integers(1234567, 1234600, n))
    else:                                                # the ends of int64
        n, ns = 100000, 500
        sess = rng.integers(0, ns, n)
        t = rng.choice(np.array([i64.min, i64.min + 1, -1, 0, 1, i64.max - 1, i64.max]), n)
    is_buy = (rng.random(n) < 0.3).astype(np.uint8)
    only_buys = rng.choice(ns, 7, replace=False)         # sessions with buys and no view
    is_buy[np.isin(sess, only_buys)] = 1
    # ten more sessions: views at t0, t0 + 5 and t0 again (the later one lands), buys at t0 and before it, so none
    # follows the landing
    t0 = t[:10]
    q_sess = np.repeat(np.arange(ns, ns + 10), 5)
    q_buy = np.tile(np.array([0, 0, 0, 1, 1], np.uint8), 10)
    q_t = np.stack([t0, t0 + (t0 < i64.max - 5) * 5, t0, t0, t0 - (t0 > i64.min)], axis=1).reshape(-1)
    return (np.concatenate([sess, q_sess]).astype(np.int32), np.concatenate([is_buy, q_buy]),
            np.concatenate([t, q_t]).astype(np.int64), ns + 10, only_buys)


@pytest.mark.parametrize("kind", ["contended", "same_ms", "int64_ends"])
def test_sessions_equal_restatement(kind):
    sess, is_buy, t, ns, only_buys = _sessions(kind, 131)
    landing, buy = native.lead_sessions(sess, is_buy, t, ns)
    want_l, want_b = sessions_ref(sess, is_buy, t, ns)
    np.testing.assert_array_equal(landing, want_l)
    np.testing.assert_array_equal(buy, want_b)
    # the fixture reaches what it is named after
    assert (landing[only_buys] == -1).all() and not buy[only_buys].any()
    assert buy.any()
    quiet = np.arange(ns - 10, ns)
    assert (landing[quiet] == len(sess) - 50 + 5 * np.arange(10) + 2).all() and not buy[quiet].any()
    views = is_buy == 0
    ties = np.bincount(sess[views & (t == t[landing[sess].clip(0)])], minlength=ns)
    if kind == "contended":
        assert np.bincount(sess, minlength=ns)[:ns - 10].min() > 3000      # thousands of atomics on each session
    else:
        assert ties.max() > (1000 if kind == "same_ms" else 10)                     # views on the landing time
    if kind == "int64_ends":
        lt = t[landing[landing >= 0]]
        assert (lt == np.iinfo(np.int64).min).any()
        assert ((t == np.iinfo(np.int64).max) & views).any()


def test_sessions_ref_matches_leadscoring_ref():
    """The NumPy rule above against tests/leadscoring_ref.py's event-by-event reduce."""
    from tests import leadscoring_ref as ref
    sess, is_buy, t, ns, _ = _sessions("int64_ends", 7)
    sess, is_buy, t = sess[:3000], is_buy[:3000], t[:3000]
    evs = [{"event": "buy" if b else "view", "t_ms": int(tt), "target": str(r), "properties": {"sessionId": f"s{s}"}}
           for r, (s, b, tt) in enumerate(zip(sess, is_buy, t))]
    landing, buy = sessions_ref(sess, is_buy, t, ns)
    seen = {}
    for s in sess:
        seen.setdefault(int(s), len(seen))
    by_sid = {}
    for s in seen:
        if landing[s] >= 0:
            by_sid[f"s{s}"] = (str(int(landing[s])), bool(buy[s]))
    evs = [e for e in evs if e["properties"]["sessionId"] in by_sid]
    got = {sid: (target, b) for sid, target, _, _, b in ref.sessions(evs)}
    assert got == by_sid
