"""GPU tests (-m gpu) of the RandomForest regressor (pio_rf_train_regressor / pio_rf_predict_regression,
mllib.RandomForest.trainRegressor): every node of every forest equals the NumPy restatement tests/forest_reg_ref.py,
doubles compared bit for bit, at the label, arity, path and grouping boundaries; the predictions equal the
restatement's; bad input raises before any device work; and classifier forests are untouched."""
import pickle

import numpy as np
import pytest

from pio_b200 import mllib
from pio_b200 import native
from tests import forest_reg_ref as rr

pytestmark = pytest.mark.gpu

INT_KEYS = ("tree_off", "feature", "left", "right", "count", "cat_off", "cat_ids")
F64_KEYS = ("threshold", "prediction", "impurity", "gain")
CAT_SMEM_ARITY = 2048          # forest.cuh: wider categorical features are ordered by cat_rank_kernel


def _assert_same(got, want):
    for k in INT_KEYS:
        np.testing.assert_array_equal(got[k], want[k], err_msg=k)
    for k in F64_KEYS:
        np.testing.assert_array_equal(got[k].view(np.uint64), want[k].view(np.uint64), err_msg=k)


def _check(y, x, cat, T, strategy, depth, bins, seed=0, held=None):
    m = mllib.RandomForest.trainRegressor(y, x, cat, T, strategy, "variance", depth, bins, seed=seed)
    want = rr.train(y, x, T, strategy, "variance", depth, bins, seed=seed, categorical=cat)
    _assert_same(m.nodes, want)
    assert m.algo == "Regression" and m.numTrees == T
    q = x if held is None else np.concatenate([x, held])
    got = m.predictBatch(q)
    np.testing.assert_array_equal(got.view(np.uint64), rr.predict(want, q).view(np.uint64))
    return m, want


def _cat_data(n, arities, n_cont, seed, labels="binary"):
    """Categorical columns (Zipf-like, so some categories are empty) plus n_cont continuous ones, and labels that
    depend on them."""
    rng = np.random.default_rng(seed)
    cols, score = [], np.zeros(n)
    for a in arities:
        v = np.minimum(rng.zipf(1.3, n) - 1, a - 1).astype(np.float64)
        perm = rng.permutation(a)
        v = perm[v.astype(np.int64)].astype(np.float64)
        cols.append(v)
        score += np.sin(v * 0.37)
    for _ in range(n_cont):
        v = np.round(rng.normal(size=n) * 3, 1)
        cols.append(v)
        score += 0.3 * v
    x = np.stack(cols, axis=1)
    noise = rng.normal(size=n)
    if labels == "binary":
        y = (score + noise > np.median(score)).astype(np.float64)
    elif labels == "int":
        y = np.round(score * 3 + noise)
    elif labels == "half":
        y = np.round((score + noise) * 2) / 2
    else:
        y = score * 1.7 + noise * 0.1
    return y, x


CASES = [
    # name, n, arities, continuous, labels, T, strategy, depth, bins
    ("template", 3000, (40, 12, 5), 0, "binary", 5, "auto", 4, 100),
    ("one_tree", 2000, (30, 8), 1, "real", 1, "auto", 6, 64),
    ("ints", 2500, (9, 7), 2, "int", 8, "all", 5, 32),
    ("halves", 2500, (6,), 2, "half", 4, "onethird", 6, 32),
    ("arity2", 1500, (2, 2), 1, "real", 3, "all", 4, 32),
    ("arity31", 3000, (31,), 1, "real", 3, "all", 4, 64),
    ("arity32", 3000, (32,), 1, "real", 3, "all", 4, 64),
    ("arity33", 3000, (33,), 1, "real", 3, "all", 4, 64),
    ("arity256_uint8", 6000, (256,), 0, "real", 2, "all", 3, 256),
    ("arity257_uint16", 6000, (257,), 0, "real", 2, "all", 3, 300),
    ("smem_arity_top", 12000, (CAT_SMEM_ARITY,), 1, "real", 2, "all", 3, 4096),
    ("rank_arity_low", 12000, (CAT_SMEM_ARITY + 1,), 1, "real", 2, "all", 3, 4096),
    ("arity65536", 70000, (65536,), 0, "real", 1, "all", 3, 65536),
    ("many_trees", 1500, (10, 6), 1, "real", 40, "auto", 5, 32),
    ("mixed_sqrt", 3000, (20, 5, 3), 3, "int", 6, "sqrt", 6, 32),
]


@pytest.mark.parametrize("case", CASES, ids=[c[0] for c in CASES])
def test_regression_forest_equals_restatement(case):
    name, n, arities, n_cont, labels, T, strategy, depth, bins = case
    y, x = _cat_data(n, arities, n_cont, seed=n + T, labels=labels)
    cat = {f: a for f, a in enumerate(arities)}
    held = np.concatenate([x[:50], -x[:3], x[:3] + 0.5])
    for f in cat:                                   # out-of-range and fractional values predict on the right
        held[-6:-3, f] = -1.0
    _, want = _check(y, x, cat, T, strategy, depth, bins, seed=T, held=held)
    # a variance entry is 40 bytes: slots wider than the 96 KiB shared-memory histogram take the global one
    k = rr.subset_size(strategy, x.shape[1], T)
    _, info = rr.train(y, x, T, strategy, "variance", depth, bins, seed=T, categorical=cat, return_nodes=True)
    nb = max([a for a in arities] + [len(t) + 1 for t in info["thresholds"]])
    paths = native.rf_train_paths()
    assert paths["bin_bytes"] == (1 if nb <= 256 else 2)
    if k * nb * 40 > 96 * 1024:
        assert paths["global_launches"] > 0 and paths["smem_launches"] == 0
    else:
        assert paths["smem_launches"] > 0 and paths["global_launches"] == 0


def test_square_carries_into_the_high_word_on_every_row():
    # |yq| in [2^43, 2^44] on every row: yq^2 >= 2^86 has a nonzero high word for every row and bag weight
    rng = np.random.default_rng(1)
    x = rng.integers(0, 6, size=(4000, 2)).astype(np.float64)
    y = np.where(rng.random(4000) < 0.5, -1.0, 1.0) * (1.0 + rng.random(4000) * 0.999) * 3.0e7
    _check(y, x, {0: 6}, 5, "all", 5, 32, seed=2)


def test_negative_and_large_labels():
    y, x = _cat_data(3000, (15,), 2, seed=9, labels="real")
    _check(-y * 1e70, x, {0: 15}, 3, "all", 5, 32)                  # max |y| ~ 8e70, inside [2^-256, 2^256)
    _check(y * 1e-60, x, {0: 15}, 3, "all", 5, 32)


def test_continuous_only_and_split_sample():
    y, x = _cat_data(60000, (), 3, seed=4, labels="real")
    _check(y, x, {}, 3, "all", 5, 32)


@pytest.mark.parametrize("per_pass,budget", [("1", None), ("2", None), ("3", "200000"), (None, "50000"),
                                             ("4", "1000")])
def test_forest_independent_of_grouping_and_chunks(monkeypatch, per_pass, budget):
    y, x = _cat_data(3000, (25, 9), 1, seed=11, labels="real")
    cat = {0: 25, 1: 9}
    want = rr.train(y, x, 7, "auto", "variance", 5, 32, seed=3, categorical=cat)
    for k, v in (("PIO_RF_TREES_PER_PASS", per_pass), ("PIO_RF_HIST_BUDGET", budget)):
        if v is None:
            monkeypatch.delenv(k, raising=False)
        else:
            monkeypatch.setenv(k, v)
    m = mllib.RandomForest.trainRegressor(y, x, cat, 7, "auto", "variance", 5, 32, seed=3)
    _assert_same(m.nodes, want)
    paths = native.rf_train_paths()
    if budget == "1000":
        assert paths["max_chunks"] > 1
    if per_pass is not None:
        assert paths["groups"] == -(-7 // int(per_pass))


def test_model_pickles_and_classifier_default():
    y, x = _cat_data(800, (5,), 1, seed=5, labels="real")
    m = mllib.RandomForest.trainRegressor(y, x, {0: 5}, 3, "auto", "variance", 3, 16)
    m2 = pickle.loads(pickle.dumps(m))
    assert m2.algo == "Regression"
    np.testing.assert_array_equal(m2.predictBatch(x), m.predictBatch(x))
    assert m2.predict(x[0]) == m.predictBatch(x[:1])[0]
    c = mllib.RandomForest.trainClassifier((y > np.median(y)).astype(float), x, 2, {}, 3, "auto", "gini", 3, 16)
    assert c.algo == "Classification" and "algo" not in vars(c)


@pytest.mark.parametrize("kw,msg", [
    (dict(impurity="gini"), "invalid impurity for Regression: gini"),
    (dict(cat={0: 40}, bins=32), "maxBins (= 32) to be at least as large"),
    (dict(cat={0: 4}, bad=4.0), "Feature 0 is categorical with values in {0,...,3}, but a data point gives it value 4.0."),
    (dict(cat={0: 4}, bad=-0.5), "gives it value -0.5."),
    (dict(y0=float("inf")), "label of row 0 is not finite (inf)."),
    (dict(y0=2.0 ** 300), "label of row 0 is out of range"),
    (dict(T=0), "numTrees > 0"),
    (dict(strategy="zero"), "invalid featureSubsetStrategy: zero"),
])
def test_rejections_match_restatement(kw, msg):
    y, x = _cat_data(200, (4,), 1, seed=6, labels="real")
    if "bad" in kw:
        x[17, 0] = kw["bad"]
    if "y0" in kw:
        y[0] = kw["y0"]
    args = (kw.get("cat", {0: 4}), kw.get("T", 3), kw.get("strategy", "auto"), kw.get("impurity", "variance"), 3,
            kw.get("bins", 32))
    with pytest.raises(ValueError) as ref:
        rr.train(y, x, args[1], args[2], args[3], 3, args[5], categorical=args[0])
    with pytest.raises(ValueError) as dev:
        mllib.RandomForest.trainRegressor(y, x, *args)
    assert msg in str(ref.value) and str(dev.value) == str(ref.value)


def test_classifier_entry_still_rejects_variance():
    with pytest.raises(native.NativeError):
        native.rf_train(np.zeros(4), np.zeros((4, 1)), 2, 1, "all", native.RF_VARIANCE, 2, 8)
