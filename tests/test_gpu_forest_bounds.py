"""GPU tests (-m gpu) of the RandomForest classifier at the boundaries of its kernel instantiations and branches: uint8
and uint16 bin codes up to the top code of each width, thresholds staged in shared memory or read from global memory,
shared-memory and global histograms, levels split into histogram chunks, more subset features than select warps, more
classes than one warp, trees 30 levels deep, degenerate inputs, the split sample and several tree groups.

Every case trains through mllib.RandomForest.trainClassifier and must equal the restatement tests/forest_ref.py node for
node (gini: bit for bit), predict on the training rows and on held-out rows must equal the restatement's vote, and
native.rf_train_paths() must be the record tests/test_forest_paths.py predicts, so each case provably ran the path it
is named after.  tests/test_forest_paths.py (CPU) checks that the cases still straddle every boundary."""
from collections import namedtuple

import numpy as np
import pytest

from pio_b200 import mllib
from pio_b200 import native
from tests import forest_ref as fr
from tests.test_gpu_forest import _assert_same, _data

pytestmark = pytest.mark.gpu

# make() -> (labels, x, held-out x); budget: PIO_RF_HIST_BUDGET (None: the default); check(forest, info, held): what
# the case's fixture must show in the restatement's forest for the case to test what it is named after
Case = namedtuple("Case", "name make C T strategy depth bins budget seed check", defaults=(None,))


def _rng(seed):
    return np.random.default_rng(seed)


def _specials(m):
    """m distinct ascending values with the edges of fp64 in them: -1.7e308 and -1e308 (their midpoint overflows to
    -inf), +-0.0 (one value), subnormals and adjacent-ulp pairs whose midpoints round onto a data value, 1e308 on top
    (the top bin code), integers between."""
    tiny = float.fromhex("0x0.0000000000001p-1022")                 # 5e-324
    one_up = np.nextafter(1.0, 2.0)
    v = [-1.7e308, -1e308, -2.0, -tiny, 0.0, tiny, 2 * tiny, 3 * tiny, float.fromhex("0x1p-1022"), 1.0, one_up,
         np.nextafter(one_up, 2.0), 1e308]
    v += [float(k) for k in range(3, 3 + m - len(v))]
    return np.unique(np.array(v[:m]))


def _on_values(vals, rows_per, n_class, seed, extra_cols=1):
    """Rows over the distinct values `vals` (each at least `rows_per` times; -0.0 for some 0.0 rows), a label per value
    from its rank in runs of 1 to 4 ranks (mostly: 5 % noise), and `extra_cols` noise columns of few values."""
    rng = _rng(seed)
    m = len(vals)
    col = np.repeat(vals, rows_per)
    rank = np.repeat(np.arange(m), rows_per)
    col = np.where((col == 0.0) & (rng.uniform(size=col.size) < 0.5), -0.0, col)
    run = np.cumsum(rng.integers(1, 5, m))
    lab = (np.searchsorted(run, np.arange(m), side="right") * 7 + 3) % n_class
    y = lab[rank].astype(np.float64)
    noise = rng.uniform(size=y.size) < 0.05
    y[noise] = rng.integers(0, n_class, noise.sum())
    x = np.column_stack([col] + [np.round(rng.normal(size=col.size), 1) for _ in range(extra_cols)])
    perm = rng.permutation(col.size)
    return y[perm], x[perm]


def _held_near(x, bins, seed):
    """Held-out rows exactly on each training threshold and one ulp either side of it, plus the training values."""
    thr = fr.find_thresholds(x, bins, seed)
    n_feat = x.shape[1]
    cols = []
    for f in range(n_feat):
        t = thr[f] if thr[f].size else np.unique(x[:, f])
        c = np.concatenate([t, np.nextafter(t, -np.inf), np.nextafter(t, np.inf), x[:300, f]])
        cols.append(c[np.isfinite(c)])
    m = min(len(c) for c in cols)
    rng = _rng(seed)
    return np.column_stack([rng.permutation(c)[:m] if len(c) > m else c for c in cols])


def width(m, bins, rows_per):
    def make():
        y, x = _on_values(_specials(m), rows_per, 3, seed=m)
        return y, x, _held_near(x, bins, 0)
    return make


def wide(m, seed):
    """A first column of m distinct values (an integer grid with the fp64 edges at both ends), labels from its rank."""
    def make():
        vals = np.unique(np.concatenate([_specials(16), np.arange(20.0, 20.0 + m - 16)]))
        y, x = _on_values(vals, 1, 2, seed=seed)
        return y, x, _held_near(x, m, 0)
    return make


def staging(m0, m1):
    """Two columns of m0 and m1 distinct values."""
    def make():
        rng = _rng(m0 + m1)
        n = 2 * max(m0, m1)
        a = np.concatenate([np.arange(m0), rng.integers(0, m0, n - m0)]) * 0.5
        b = np.concatenate([np.arange(m1), rng.integers(0, m1, n - m1)]) * 0.25 - 100.0
        rng.shuffle(b)
        y = ((np.floor(a / 37) + np.floor((b + 100.0) / 53)) % 3).astype(np.float64)
        x = np.column_stack([a, b])
        return y, x, _held_near(x, max(m0, m1), 0)
    return make


def classes(n, F, C, m, present=None, seed=1):
    """_data's rows with the first column replaced by m distinct values that decide the label (C classes or only
    `present` of them)."""
    def make():
        rng = _rng(seed)
        k = present or C
        y, x = _data(n, F, C, seed=seed, present=present)
        v = rng.integers(0, m, n)
        v[:m] = np.arange(m)
        x[:, 0] = v * 0.5
        y = np.where(rng.uniform(size=n) < 0.9, (v * k) // m, y).astype(np.float64)
        _, held = _data(400, F, C, seed=seed + 1)
        return y, x, held
    return make


def _base(dups):
    """The column each column of warps(F, dups) copies (itself when none)."""
    to = {b: a for a, b in dups}
    return lambda f: to.get(f, f)


def warps(F, dups, n=3000, seed=5):
    """F columns where column b is a copy of column a for each (a, b) in dups; the label depends on columns 0 and 3
    (and 1), so that the copies tie with their originals at the nodes that split them."""
    def make():
        rng = _rng(seed)
        x = np.round(rng.normal(size=(n, F)) * 3, 1)
        for a, b in dups:
            x[:, b] = x[:, a]
        s = x[:, 0] - 0.8 * x[:, 3 % F] + 0.4 * x[:, 1] + rng.normal(size=n)
        y = np.digitize(s, np.quantile(s, [1 / 3, 2 / 3])).astype(np.float64)
        return y, x, np.round(rng.normal(size=(300, F)) * 3, 1)
    return make


def copies(F, base, n=3000, seed=6):
    """F columns, each a copy of one of `base` columns (f % base): every node's subset ties between copies."""
    def make():
        rng = _rng(seed)
        b = np.round(rng.normal(size=(n, base)) * 3, 1)
        x = b[:, np.arange(F) % base].copy()
        s = b[:, 0] + 0.7 * b[:, 1] + rng.normal(size=n)
        y = np.digitize(s, np.quantile(s, [1 / 3, 2 / 3])).astype(np.float64)
        return y, x, np.round(rng.normal(size=(300, F)) * 3, 1)
    return make


def symmetric():
    """One column 0 .. 51, class 0 on the first and last 10 values, class 1 between: x <= 9.5 and x <= 41.5 split with
    exactly equal gains, thresholds 32 apart (two select trips of one warp); the first, the smaller, must win."""
    def make():
        v = np.arange(52.0)
        y = np.where((v < 10) | (v >= 42), 0.0, 1.0)
        x = np.repeat(v, 3)[:, None]
        return np.repeat(y, 3), x, np.arange(-1.0, 53.0, 0.5)[:, None]
    return make


def comb(n):
    """Alternating labels on one column 0 .. n - 1: every level peels one row off, so a tree reaches depth 30."""
    def make():
        x = np.arange(float(n))[:, None]
        return (np.arange(n) % 2).astype(np.float64), x, np.arange(-0.5, n + 0.5, 0.25)[:, None]
    return make


def constant(n, F, C):
    def make():
        rng = _rng(n)
        x = np.tile(np.arange(1.0, F + 1.0), (n, 1))
        y = rng.integers(0, C, n).astype(np.float64)
        return y, x, np.round(rng.normal(size=(50, F)), 1)
    return make


def plain(n, F, C, decimals=1, seed=3):
    def make():
        y, x = _data(n, F, C, seed=seed, decimals=decimals)
        _, held = _data(300, F, C, seed=seed + 1, decimals=decimals)
        return y, x, held
    return make


def groups(n, seed=7):
    """One column of few values and a label that follows it: cheap to restate at n rows times many trees."""
    def make():
        rng = _rng(seed)
        x = rng.integers(0, 16, (n, 1)).astype(np.float64)
        y = ((x[:, 0] >= 8) ^ (rng.uniform(size=n) < 0.2)).astype(np.float64)
        return y, x, np.arange(-1.0, 17.0, 0.5)[:, None]
    return make


# ---- what each fixture must show in the restatement's forest --------------------------------------------------------
def ties_to_smaller_copy(base_of, seed, n_feat, k):
    """Copies of a column tie with it: no split uses a copy while a smaller copy was in the node's subset, and some
    split had a larger copy in its subset (so the tie arose)."""
    def check(want, info, held):
        arose = 0
        for t, nodes in enumerate(info["trees"]):
            for i, r in nodes.items():
                if r["leaf"]:
                    continue
                f = r["feature"]
                same = [g for g in fr.node_subset(seed, t, i, n_feat, k) if base_of(g) == base_of(f) and g != f]
                assert all(g > f for g in same), (t, i, f, same)
                arose += bool(same)
        assert arose > 0
    return check


def vote_ties(want, info, held):
    v = _votes(want, held)
    assert ((v == v.max(axis=1)[:, None]).sum(axis=1) > 1).any(), "no vote tie on the held-out rows"


def reaches_depth(d):
    def check(want, info, held):
        assert want["depth"].max() == d
    return check


def root_tie_32_apart(want, info, held):
    g, r = info["runner_up"][0]                 # the root's best gain and the best with other left counts
    assert g == r and want["threshold"][0] == 9.5


def leaves_only(want, info, held):
    assert (want["feature"] == -1).all() and want["feature"].size == want["tree_off"].size - 1



CHUNK_SMEM = classes(3000, 3, 4, 32, seed=11)        # K NB C = 3 x 32 x 4: a 3072-byte slot, 64 slots per pass
CHUNK_GLOBAL = classes(3000, 3, 33, 256, seed=12)     # 3 x 256 x 33: a 202 752-byte slot, beyond one pass
SLOT_SMEM, SLOT_GLOBAL = 3 * 32 * 4 * 8, 3 * 256 * 33 * 8

CASES = [
    # bin width: NB = 256 (uint8, top code 255) / 257 (uint16); NB = 65536 (top code 65535)
    Case("nb256_uint8", width(256, 256, 8), 3, 3, "all", 10, 256, None, 1),
    Case("nb257_uint16", width(257, 257, 8), 3, 3, "all", 10, 257, None, 1),
    Case("nb65536", wide(65536, 2), 2, 1, "all", 4, 65536, None, 0),
    # thresholds: 3072 + 3072 = 6144 staged in shared memory, 3072 + 3073 read from global memory
    Case("thr6144_staged", staging(3073, 3073), 3, 2, "all", 5, 3073, None, 0),
    Case("thr6145_global", staging(3073, 3074), 3, 2, "all", 5, 3074, None, 0),
    # K NB C = 3 x 256 x 32 = 24 576: one slot per 96 KB pass; C = 33: the global histogram (and two carry trips)
    Case("smem_one_slot_c32", classes(4000, 3, 32, 256, seed=2), 32, 2, "all", 5, 256, None, 3),
    Case("global_c33", classes(4000, 3, 33, 256, seed=2), 33, 2, "all", 5, 256, None, 3),
    # 3 x 64 x 32: four slots per pass; a shallow forest needs one pass per level, a deep one several
    Case("passes_shallow", classes(4000, 3, 32, 64, seed=4), 32, 2, "all", 2, 64, None, 1),
    Case("passes_deep", classes(4000, 3, 32, 64, seed=4), 32, 2, "all", 7, 64, None, 1),
    # a level chunked at the default 512 MB budget: 2 x 65536 x 64 x 8 = 64 MB a slot, 8 slots a chunk, 10 slots
    Case("chunked_default", classes(70000, 2, 64, 65536, seed=9), 64, 5, "all", 2, 65536, None, 2),
    # subset features vs select warps (8): K = 8, 9, 16, 17 and sqrt of 100; copies in one warp and across warps
    *[Case(f"k{F}", warps(F, d), 3, 3, "all", 6, 32, None, 1, ties_to_smaller_copy(_base(d), 1, F, F))
      for F, d in ((8, [(3, 4), (0, 7)]), (9, [(0, 8), (3, 4)]), (16, [(0, 8), (3, 4), (7, 15)]),
                   (17, [(0, 8), (0, 16), (3, 4), (1, 9)]))],
    Case("k10_sqrt100", copies(100, 3), 3, 5, "sqrt", 6, 32, None, 1, ties_to_smaller_copy(lambda f: f % 3, 1, 100, 10)),
    Case("tie_32_apart", symmetric(), 2, 1, "all", 3, 64, None, 0, root_tie_32_apart),
    # classes: 2 and 64 (all present / five present); two and four trees give vote ties
    Case("c2", plain(3000, 3, 2), 2, 4, "auto", 6, 32, None, 1, vote_ties),
    Case("c64_all", classes(8000, 9, 64, 128, seed=3), 64, 4, "all", 8, 128, None, 1, vote_ties),   # 2 trips a warp
    Case("c64_five", classes(3000, 4, 64, 128, present=5, seed=3), 64, 2, "sqrt", 6, 128, None, 2, vote_ties),
    # depth 30
    Case("depth30_comb", comb(40), 2, 1, "all", 30, 64, None, 0, reaches_depth(30)),
    # degenerate: every feature constant (NB = 1), one and two rows, maxBins > n
    Case("constant", constant(500, 3, 3), 3, 3, "all", 5, 32, None, 0, leaves_only),
    Case("n1", lambda: (np.array([1.0]), np.array([[2.0, 3.0]]), np.array([[1.0, 1.0], [3.0, 4.0]])), 2, 2, "all", 4,
         32, None, 0),
    Case("n2", lambda: (np.array([1.0, 0.0]), np.array([[2.0], [-0.0]]), np.array([[1.0], [0.0], [3.0], [-1.0]])), 2,
         3, "all", 4, 65536, None, 0),
    # split sample: n = max(maxBins^2, 10000) (every row) and one row more (a sample)
    Case("sample_all_90000", plain(90000, 2, 3, decimals=3), 3, 3, "auto", 4, 300, None, 1),
    Case("sample_some_90001", plain(90001, 2, 3, decimals=3), 3, 3, "auto", 4, 300, None, 1),
    # two tree groups at the default 1 GiB node budget: 2^28 / n trees a group
    Case("two_groups", groups(1 << 22), 2, 65, "all", 1, 32, None, 1),
]
# chunk budgets: one, two and three slots a chunk, and less than one slot (clamped to one), for both histograms
CHUNK_BUDGETS = [None, 1, 2, 3, 0.3]
CHUNK_CASES = [Case(f"chunk_{kind}_{b}", make, C, 5, "all", 6, bins, None if b is None else int(b * slot), 4)
               for kind, make, C, bins, slot in (("smem", CHUNK_SMEM, 4, 32, SLOT_SMEM),
                                                 ("global", CHUNK_GLOBAL, 33, 256, SLOT_GLOBAL))
               for b in CHUNK_BUDGETS]


def _votes(forest, x):
    """Per-row class votes of the restatement's forest [n, C]."""
    n = x.shape[0]
    votes = np.zeros((n, forest["num_classes"]), np.int64)
    feat, thr, lft, rgt = forest["feature"], forest["threshold"], forest["left"], forest["right"]
    for t in range(len(forest["tree_off"]) - 1):
        at = np.full(n, forest["tree_off"][t], np.int64)
        while (feat[at] >= 0).any():
            r = np.flatnonzero(feat[at] >= 0)
            at[r] = np.where(x[r, feat[at[r]]] <= thr[at[r]], lft[at[r]], rgt[at[r]])
        votes[np.arange(n), forest["prediction"][at]] += 1
    return votes


def run_case(case, monkeypatch):
    from tests import test_forest_paths as P
    y, x, held = case.make()
    if case.budget is None:
        monkeypatch.delenv("PIO_RF_HIST_BUDGET", raising=False)
    else:
        monkeypatch.setenv("PIO_RF_HIST_BUDGET", str(case.budget))
    monkeypatch.delenv("PIO_RF_TREES_PER_PASS", raising=False)
    m = mllib.RandomForest.trainClassifier(y, x, case.C, {}, case.T, case.strategy, "gini", case.depth, case.bins,
                                           seed=case.seed)
    got_paths = native.rf_train_paths()
    want, info = fr.train(y, x, case.C, case.T, case.strategy, "gini", case.depth, case.bins, seed=case.seed,
                          return_nodes=True)
    _assert_same(m.nodes, want)
    np.testing.assert_array_equal(m.depth, want["depth"])
    assert got_paths == P.expected_record(case, x, info["level_slots"]), case.name
    for rows in (x, held):
        np.testing.assert_array_equal(m.predictBatch(rows), fr.predict(want, rows))
    return m, want, info, held


@pytest.mark.parametrize("case", CASES, ids=[c.name for c in CASES])
def test_forest_at_boundary(case, monkeypatch):
    _, want, info, held = run_case(case, monkeypatch)
    if case.check is not None:
        case.check(want, info, held)


@pytest.mark.parametrize("kind", ["smem", "global"])
def test_chunked_levels_equal_across_budgets(kind, monkeypatch):
    cases = [c for c in CHUNK_CASES if c.name.startswith(f"chunk_{kind}_")]
    forests = [run_case(c, monkeypatch)[0].nodes for c in cases]
    for f in forests[1:]:
        _assert_same(f, forests[0])
