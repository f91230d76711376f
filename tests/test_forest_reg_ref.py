"""CPU: the RandomForest regressor's restatement (tests/forest_reg_ref.py) against hand-computed splits, its category
order, label quantisation, argument and data rejections, pruning and the averaged predict; and the host-side
rejections of mllib.RandomForest.trainRegressor, which run before the library is touched."""
import math

import numpy as np
import pytest

from tests import forest_ref as fr
from tests import forest_reg_ref as rr


def _train(y, x, T=1, strategy="all", depth=4, bins=32, cat=None, seed=0):
    return rr.train(y, x, T, strategy, "variance", depth, bins, seed=seed, categorical=cat)


def test_variance_split_by_hand():
    # y = 0, 0, 1, 1 at x = 0, 1, 2, 3: the best split is x <= 1.5 with gain 0.25
    f = _train([0, 0, 1, 1], np.arange(4.0)[:, None], depth=1)
    assert f["feature"].tolist() == [0, -1, -1]
    assert f["threshold"][0] == 1.5 and f["gain"][0] == 0.25
    assert f["impurity"].tolist() == [0.25, 0.0, 0.0]
    assert f["prediction"].tolist() == [0.5, 0.0, 1.0]
    assert f["count"].tolist() == [4, 2, 2]


def test_variance_of_unequal_children():
    # y = 1, 2, 3, 10: variance 12.5; split after 3 leaves var(1,2,3) = 2/3 and 0: gain 12.5 - 0.75 * 2/3 = 12
    y = np.array([1.0, 2.0, 3.0, 10.0])
    f = _train(y, np.arange(4.0)[:, None], depth=1)
    assert f["impurity"][0] == 12.5
    assert f["threshold"][0] == 2.5
    assert f["gain"][0] == 12.5 - 0.75 * ((14.0 - 36.0 / 3.0) / 3.0)


def test_category_order_sorts_by_centroid_with_empty_categories_last_and_ties_by_category():
    # categories 0..4: means 1, 0, (empty), 1, 0.5 -> order 1, 4, 0, 3, 2 (0 before 3: equal means keep category order)
    x = np.array([0, 0, 1, 1, 3, 4, 4], np.float64)[:, None]
    y = np.array([1, 1, 0, 0, 1, 0, 1], np.float64)
    yq, s = rr.quantize(y)
    W = np.zeros(5, object)
    S = np.zeros(5, object)
    W[:] = 0
    S[:] = 0
    for v, q in zip(x[:, 0].astype(int), yq):
        W[v] += 1
        S[v] += q
    assert rr.category_order(W, S, s, 5).tolist() == [1, 4, 0, 3, 2]
    f = _train(y, x, depth=1, cat={0: 5})
    assert f["feature"][0] == 0 and f["threshold"][0] == 0.0
    # prefixes {1}: gain 12/49 - 5/7 * 4/25 = 0.1306; {1, 4}: 12/49 - 4/7 * 3/16 = 0.1378 (right side pure); wider ones
    # are worse
    assert f["cat_ids"].tolist() == [1, 4] and f["cat_off"].tolist() == [0, 2, 2, 2]


def test_categorical_predict_needs_an_exact_member():
    x = np.array([0, 0, 1, 1, 2, 2], np.float64)[:, None]
    y = np.array([0, 0, 5, 5, 0, 0], np.float64)
    f = _train(y, x, depth=1, cat={0: 3})
    left = set(f["cat_ids"].tolist())
    assert left in ({1}, {0, 2})
    go = lambda v: f["prediction"][1] if v in left else f["prediction"][2]          # noqa: E731
    q = np.array([[0.0], [1.0], [2.0], [1.5], [-1.0], [7.0], [-0.0]])
    want = [go(0.0), go(1.0), go(2.0), f["prediction"][2], f["prediction"][2], f["prediction"][2], go(0.0)]
    assert rr.predict(f, q).tolist() == want


@pytest.mark.parametrize("y,shift", [
    ([1.0, 0.0], 43), ([2.0, -1.0], 42), ([0.75, 0.5], 44), ([0.0, 0.0], 0), ([-3.0, 1.0], 42),
    ([2.0 ** 100, 1.0], -57)])
def test_quantize_shift(y, shift):
    yq, s = rr.quantize(y)
    assert s == shift
    m = max(abs(v) for v in y)
    if m:
        assert 2 ** 43 <= max(abs(q) for q in yq) <= 2 ** 44
    assert all(q == round(v * 2.0 ** s) for q, v in zip(yq, y))


def test_quantize_ties_to_even():
    # max 1 -> s = 43; 2^-44 and 3 * 2^-44 are exact halves at that scale
    yq, s = rr.quantize([1.0, 2.0 ** -44, 3 * 2.0 ** -44, -(2.0 ** -44), 5 * 2.0 ** -44])
    assert s == 43 and yq == [2 ** 43, 0, 2, 0, 2]


def test_power_of_two_max_label_and_negative_labels_are_exact():
    y = np.array([-4.0, 4.0, -4.0, 4.0, 2.0, -2.0])
    f = _train(y, np.arange(6.0)[:, None], depth=0)
    assert f["prediction"][0] == 0.0 and f["impurity"][0] == np.mean(y ** 2)


def test_all_zero_labels_give_one_leaf():
    f = _train(np.zeros(10), np.arange(10.0)[:, None], T=3, strategy="auto")
    assert f["feature"].tolist() == [-1, -1, -1] and f["prediction"].tolist() == [0.0] * 3


def test_pruning_collapses_equal_leaves_and_keeps_the_left_prediction():
    # depth 2 with labels 0 0 1 1 | 1 1 1 1 gives equal children on the right; they collapse
    x = np.arange(8.0)[:, None]
    y = np.array([0, 0, 1, 1, 1, 1, 1, 1.0])
    forest, info = rr.train(y, x, 1, "all", "variance", 2, 32, return_nodes=True)
    nodes = info["trees"][0]
    assert not nodes[1]["leaf"]
    assert all(f == -1 or f == 0 for f in forest["feature"])
    pred = forest["prediction"]
    leaves = forest["feature"] == -1
    assert sorted(set(pred[leaves].tolist())) == [0.0, 1.0]
    # every internal node's two leaf children differ
    for i in np.flatnonzero(~leaves):
        l, r = forest["left"][i], forest["right"][i]
        if forest["feature"][l] < 0 and forest["feature"][r] < 0:
            assert pred[l] != pred[r]


def test_forest_predict_sums_in_tree_order_then_divides():
    rng = np.random.default_rng(3)
    x = rng.integers(0, 4, size=(200, 2)).astype(np.float64)
    y = rng.random(200) * 0.3 + x[:, 0]
    f = rr.train(y, x, 7, "auto", "variance", 3, 16, seed=5, categorical={1: 4})
    tp = rr.tree_predict(f, x)
    acc = np.zeros(200)
    for t in range(7):
        acc = acc + tp[t]
    assert np.array_equal(rr.predict(f, x), acc / 7.0)


def test_auto_is_onethird_for_a_forest():
    assert rr.subset_size("auto", 3, 5) == 1 and rr.subset_size("auto", 3, 1) == 3
    assert rr.subset_size("auto", 10, 2) == math.ceil(10 / 3) and fr.subset_size("auto", 10, 2) == 4


REJECT = [
    (dict(impurity="gini"), "invalid impurity for Regression: gini"),
    (dict(impurity="bogus"), "Did not recognize Impurity name: bogus"),
    (dict(cat={5: 3}), "categoricalFeaturesInfo names feature 5, but the data have 2 features."),
    (dict(cat={1: 1}), "feature 1 has 1 categories.  The number of categories should be >= 2."),
    (dict(T=0), "numTrees > 0"),
    (dict(strategy="sqrtx"), "invalid featureSubsetStrategy: sqrtx"),
    (dict(depth=31), "maxDepth <= 30"),
    (dict(bins=1), "invalid maxBins parameter: 1"),
    (dict(cat={1: 40}, bins=32), "maxBins (= 3) to be at least as large as the number of values in each categorical "
                                 "feature, but categorical feature 1 has 40 values."),
    (dict(cat={1: 3}), "Feature 1 is categorical with values in {0,...,2}, but a data point gives it value 3.0."),
    (dict(y0=float("nan")), "label of row 0 is not finite (nan)."),
    (dict(y0=2.0 ** 256), "label of row 0 is out of range"),
    (dict(y0=-(2.0 ** 256)), "label of row 0 is out of range"),
    (dict(tiny=True), "label of row 0 is out of range"),
]


def _reject_case(kw):
    x = np.array([[0.0, 1.0], [1.0, 3.0], [2.0, 0.0]])
    y = np.array([1.0, 0.0, 1.0])
    if "y0" in kw:
        y[0] = kw["y0"]
    if kw.get("tiny"):
        y = np.array([2.0 ** -257, 0.0, 0.0])
    return y, x, dict(num_trees=kw.get("T", 2), strategy=kw.get("strategy", "auto"),
                      impurity=kw.get("impurity", "variance"), max_depth=kw.get("depth", 3),
                      max_bins=kw.get("bins", 32), categorical=kw.get("cat"))


@pytest.mark.parametrize("kw,msg", REJECT)
def test_restatement_rejects(kw, msg):
    y, x, a = _reject_case(kw)
    with pytest.raises(ValueError) as e:
        rr.train(y, x, a["num_trees"], a["strategy"], a["impurity"], a["max_depth"], a["max_bins"],
                 categorical=a["categorical"])
    assert msg in str(e.value)


def test_largest_labels_accepted():
    y = np.array([2.0 ** 256 - 2.0 ** 203, 2.0 ** -256, 0.0])
    f = _train(y, np.arange(3.0)[:, None], depth=1)
    assert np.isfinite(f["impurity"]).all()
    f = _train(np.array([2.0 ** -256, 0.0]), np.arange(2.0)[:, None], depth=1)
    assert f["prediction"][0] == 2.0 ** -257


@pytest.mark.parametrize("kw,msg", [r for r in REJECT if r[0].keys() & {"impurity", "cat"} and
                                    "bins" not in r[0] and "a data point" not in r[1]])
def test_mllib_host_rejections(kw, msg):
    from pio_b200 import mllib
    y, x, a = _reject_case(kw)
    with pytest.raises(ValueError) as e:
        mllib.RandomForest.trainRegressor(y, x, a["categorical"], a["num_trees"], a["strategy"], a["impurity"],
                                          a["max_depth"], a["max_bins"])
    assert msg in str(e.value)
