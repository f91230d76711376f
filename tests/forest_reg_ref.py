"""NumPy restatement of the RandomForest regressor of pio_rf_train_regressor: the definition the GPU regression forest is
checked against.

It follows MLlib 2.4's `RandomForest.trainRegressor` with ordered categorical features, and reuses the classifier's
restatement (tests/forest_ref.py) for everything the two share: the split sample and thresholds of continuous features,
bagging, per-node feature subsets, level-wise growth over heap-numbered nodes, the validity and first-maximum rules of
a split, and the flat preorder layout.  From MLlib:
  - arguments, in this order: impurity must be "variance" (Strategy.assertValid); every categoricalFeaturesInfo key
    is a feature and every arity >= 2; the classifier's numeric checks minus numClasses; then, over the data, the
    largest arity <= min(maxBins, n) (DecisionTreeMetadata) and every categorical value v in 0 <= v < arity
    (TreePoint.findBin); its bin is trunc(v);
  - featureSubsetStrategy "auto" is all features for one tree and onethird for more (RandomForest.run, regression);
  - Variance.calculate(count, sum, sumSq) = (sumSq - sum * sum / count) / count, 0 for an empty node; a node predicts
    sum / count; gain = imp - (nL / n) impL - (nR / n) impR, invalid when nL < 1, nR < 1 or gain < 0;
  - an ordered categorical feature: per node, each category's centroid is its mean label (Double.MaxValue without
    rows), categories are stably sorted by centroid (equal centroids keep the smaller category first), and the
    arity - 1 candidates split that order after position j (the left side is its prefix);
  - predict: a continuous node sends x <= threshold left, a categorical node sends x left iff x equals one of its left
    categories (categories.contains), so a value out of range goes right; LearningNode.toNode(prune = true) collapses
    an internal node whose two leaf children have == predictions (the leaf keeps the left child's prediction); the
    forest averages its trees: predictions summed in tree order from 0.0, divided by numTrees.

This project's choice, which keeps the forest deterministic: label sums are exact integers.  With s the exponent that
puts max|y| in [2^43, 2^44) (s = 0 when every label is 0), each label becomes yq = round-half-even(y 2^s), |yq| <= 2^44.
Per (node, feature, bin) the sums sum(w), sum(w yq) and sum(w yq^2) are integers (below 2^123 for n < 2^31 and bag
weights <= 16), so they do not depend on summation order, and enter the fp64 formulas as W = float(sum w),
S = float(sum w yq) 2^-s and Q = float(sum w yq^2) 2^-2s, each conversion correctly rounded.  Labels must be finite,
below 2^256 in magnitude, and, unless all are 0, the largest at least 2^-256 in magnitude: that keeps 2^-s and 2^-2s
normal doubles and every Q, S * S finite.  Labels of 0 / 1, small integers and halves are exact.

A forest is forest_ref's dict of flat per-node arrays, with `prediction` in float64 and, per node, its left
categories: cat_off [n_nodes + 1] (int64) and cat_ids (int32, ascending per node); a categorical node has threshold 0.
"""
import math
import sys

import numpy as np

from tests import forest_ref as fr

VARIANCE = 2
LABEL_BITS = 44
LABEL_EXP_MAX = 256          # |y| < 2^256 and, unless every label is 0, max|y| >= 2^-256
DMAX = sys.float_info.max


def subset_size(s, n_feat, num_trees):
    if s == "auto":
        s = "all" if num_trees == 1 else "onethird"
    return fr.subset_size(s, n_feat, num_trees)


def check_args(num_trees, strategy, impurity, max_depth, max_bins, n_feat=1, categorical=None):
    if impurity != "variance":
        if impurity in fr.IMPURITIES:
            raise ValueError(f"DecisionTree Strategy given invalid impurity for Regression: {impurity}.  Valid settings: "
                             f"Variance")
        raise ValueError(f"Did not recognize Impurity name: {impurity}")
    for f, a in sorted((categorical or {}).items()):
        if not 0 <= f < n_feat:
            raise ValueError(f"categoricalFeaturesInfo names feature {f}, but the data have {n_feat} features.")
        if a < 2:
            raise ValueError(f"DecisionTree Strategy given invalid categoricalFeaturesInfo setting: feature {f} has {a} "
                             f"categories.  The number of categories should be >= 2.")
    if num_trees < 1:
        raise ValueError(f"RandomForest requires numTrees > 0, but was given numTrees = {num_trees}.")
    if subset_size(strategy, max(n_feat, 1), num_trees) == 0:
        raise ValueError(f"RandomForest given invalid featureSubsetStrategy: {strategy}. Supported values: "
                         f"{fr.STRATEGIES}, (0.0-1.0], [1-n].")
    fr.check_numeric(2, num_trees, "all", max_depth, max_bins, n_feat)


def check_data(labels, x, max_bins, categorical=None):
    n, n_feat = x.shape
    if n < 1 or n_feat < 1:
        raise ValueError("RandomForest requires at least one row and one feature.")
    if n >= 2 ** 31:
        raise ValueError("at most 2^31 - 1 rows are supported.")
    bad = ~np.isfinite(labels) | ~np.isfinite(x).all(axis=1)
    if bad.any():
        r = int(np.flatnonzero(bad)[0])
        if not np.isfinite(labels[r]):
            raise ValueError(f"label of row {r} is not finite ({fr.fmt_double(labels[r])}).")
        f = int(np.flatnonzero(~np.isfinite(x[r]))[0])
        raise ValueError(f"feature {f} of row {r} is not finite ({fr.fmt_double(x[r, f])}).")
    a = np.abs(labels)
    m = float(a.max())
    if m >= 2.0 ** LABEL_EXP_MAX or (0 < m < 2.0 ** -LABEL_EXP_MAX):
        r = int(np.flatnonzero(a == m)[0])
        raise ValueError(f"label of row {r} is out of range ({fr.fmt_double(labels[r])}): the largest |label| must be "
                         f"0 or in [2^-{LABEL_EXP_MAX}, 2^{LABEL_EXP_MAX}).")
    cat = dict(categorical or {})
    if cat:
        nb = min(max_bins, n)
        amax = max(cat.values())
        if amax > nb:
            f = min(f for f, v in cat.items() if v == amax)
            raise ValueError(f"DecisionTree requires maxBins (= {nb}) to be at least as large as the number of values in "
                             f"each categorical feature, but categorical feature {f} has {amax} values. Consider "
                             f"removing this and other categorical features with a large number of values, or add more "
                             f"training examples.")
        fs = sorted(cat)
        ar = np.array([cat[f] for f in fs], np.float64)
        v = x[:, fs]
        bad = (v < 0) | (v >= ar[None, :])
        if bad.any():
            r = int(np.flatnonzero(bad.any(axis=1))[0])
            k = int(np.flatnonzero(bad[r])[0])
            raise ValueError(f"DecisionTree given invalid data: Feature {fs[k]} is categorical with values in "
                             f"{{0,...,{cat[fs[k]] - 1}}}, but a data point gives it value {fr.fmt_double(v[r, k])}.")


def quantize(labels):
    """(yq: Python ints, s): yq = round-half-even(y 2^s) with s putting max|y| in [2^43, 2^44); s = 0 for all-zero."""
    labels = np.asarray(labels, np.float64)
    m = float(np.abs(labels).max()) if labels.size else 0.0
    s = 0 if m == 0 else LABEL_BITS - math.frexp(m)[1]
    q = np.rint(np.ldexp(labels, s))
    return [int(v) for v in q], s


def to_f64(W, S, Q, s):
    """The fp64 statistics of integer sums (scalars or object arrays)."""
    f = np.vectorize(float, otypes=[np.float64])
    return f(W), f(S) * (2.0 ** -s), f(Q) * (2.0 ** (-2 * s))


def variance(W, S, Q):
    """Variance.calculate on fp64 statistics (arrays), 0 where W == 0."""
    with np.errstate(divide="ignore", invalid="ignore"):
        v = (Q - (S * S) / W) / W
    return np.where(W == 0, 0.0, v)


def mean(W, S):
    with np.errstate(divide="ignore", invalid="ignore"):
        return np.where(W == 0, 0.0, S / W)


def _gains(Wc, Sc, Qc, s, n_cand):
    """Cumulative integer statistics [M] of one feature's bins in split order: gains of its first n_cand candidates
    (-inf when invalid) and the fp64 left statistics."""
    W, S, Q = to_f64(Wc, Sc, Qc, s)
    Wt, St, Qt = W[-1], S[-1], Q[-1]
    ip = variance(np.array([Wt]), np.array([St]), np.array([Qt]))[0]
    Wr, Sr, Qr = to_f64(Wc[-1] - Wc, Sc[-1] - Sc, Qc[-1] - Qc, s)
    n = Wt if Wt != 0 else 1.0
    gain = (ip - (W / n) * variance(W, S, Q)) - (Wr / n) * variance(Wr, Sr, Qr)
    j = np.arange(W.shape[0])
    ok = (j < n_cand) & (Wc >= 1) & (Wc[-1] - Wc >= 1) & (gain >= 0)
    return np.where(ok, gain, -np.inf)


def _node_stats(idx, w, wy, wy2, nb):
    W = np.zeros(nb, object)
    S = np.zeros(nb, object)
    Q = np.zeros(nb, object)
    W[:] = 0
    S[:] = 0
    Q[:] = 0
    np.add.at(W, idx, w)
    np.add.at(S, idx, wy)
    np.add.at(Q, idx, wy2)
    return W, S, Q


def category_order(W, S, s, arity):
    """The categories 0 .. arity - 1 stably sorted by centroid (mean label, Double.MaxValue without rows)."""
    Wf, Sf, _ = to_f64(W[:arity], S[:arity], S[:arity], s)
    cen = np.where(Wf == 0, DMAX, mean(Wf, Sf))
    return np.argsort(cen, kind="stable")


def train(labels, x, num_trees, strategy, impurity, max_depth, max_bins, seed=0, categorical=None, return_nodes=False):
    labels = np.asarray(labels, np.float64)
    x = np.asarray(x, np.float64)
    cat = {int(f): int(a) for f, a in (categorical or {}).items()}
    check_args(num_trees, strategy, impurity, max_depth, max_bins, x.shape[1], cat)
    check_data(labels, x, max_bins, cat)
    n, n_feat = x.shape
    yq, s = quantize(labels)
    k = subset_size(strategy, n_feat, num_trees)
    cont = [f for f in range(n_feat) if f not in cat]
    thr = [np.zeros(0)] * n_feat
    if cont:
        found = fr.find_thresholds(x[:, cont], max_bins, seed)
        for j, f in enumerate(cont):
            thr[f] = found[j]
    bins = np.stack([np.trunc(x[:, f]).astype(np.int64) if f in cat else
                     np.searchsorted(thr[f], x[:, f], side="left") for f in range(n_feat)], axis=1)
    trees, level_slots = [], []
    yq_o = np.array(yq, object)
    for t in range(num_trees):
        w = np.ones(n, np.int64) if num_trees == 1 else fr.bag_weights(seed, t, n)
        w_o = w.astype(object)
        wy, wy2 = w_o * yq_o, w_o * yq_o * yq_o
        nodes = {}
        at = np.ones(n, np.int64)
        active, level = [1], 0
        level_slots.append([])
        while active:
            level_slots[-1].append(len(active))
            nxt = []
            for i in active:
                rows = np.flatnonzero(at == i)
                sub = fr.node_subset(seed, t, i, n_feat, k)
                best = (-np.inf, None)
                tot = None
                for f in sub:
                    m = cat[f] if f in cat else len(thr[f]) + 1
                    W, S, Q = _node_stats(bins[rows, f], w_o[rows], wy[rows], wy2[rows], m)
                    if tot is None:
                        tot = (int(W.sum()), int(S.sum()), int(Q.sum()))
                    order = category_order(W, S, s, m) if f in cat else np.arange(m)
                    Wc, Sc, Qc = np.cumsum(W[order]), np.cumsum(S[order]), np.cumsum(Q[order])
                    g = _gains(Wc, Sc, Qc, s, m - 1)
                    j = int(np.argmax(g))
                    if g[j] > best[0]:
                        best = (g[j], (f, j, order, (int(Wc[j]), int(Sc[j]), int(Qc[j]))))
                _decide(nodes, nxt, at, bins, thr, cat, i, tot, best, s, level, max_depth)
            active, level = sorted(nxt), level + 1
        trees.append(nodes)
    forest = flatten(trees)
    if return_nodes:
        return forest, dict(thresholds=thr, subset_size=k, trees=trees, level_slots=level_slots, shift=s)
    return forest


def _record(st, s):
    W, S, Q = to_f64(*st, s)
    return dict(stats=st, count=st[0], impurity=float(variance(np.array([W]), np.array([S]), np.array([Q]))[0]),
                prediction=float(mean(np.array([W]), np.array([S]))[0]), gain=0.0, leaf=True, feature=-1,
                threshold=0.0, cats=None)


def _decide(nodes, nxt, at, bins, thr, cat, i, tot, best, s, level, max_depth):
    rec = _record(tot, s)
    nodes[i] = rec
    rows = at == i
    g, arg = best
    if not np.isfinite(g) or g <= 0 or level == max_depth:
        at[rows] = 0
        return
    f, j, order, left = arg
    rec.update(leaf=False, feature=int(f), gain=float(g))
    if f in cat:
        rec["cats"] = np.sort(order[:j + 1]).astype(np.int32)
        go_left = np.isin(bins[:, f], rec["cats"])
    else:
        rec["threshold"] = float(thr[f][j])
        go_left = bins[:, f] <= j
    right = tuple(a - b for a, b in zip(tot, left))
    for child, st in ((2 * i, left), (2 * i + 1, right)):
        cr = _record(st, s)
        if level + 1 == max_depth or cr["impurity"] == 0.0:
            nodes[child] = cr
        else:
            nxt.append(child)
    at[rows & go_left] = 2 * i if (2 * i) in nxt else 0
    at[rows & ~go_left] = 2 * i + 1 if (2 * i + 1) in nxt else 0


def _prune(nodes, i):
    r = nodes[i]
    if r["leaf"]:
        return (r, None)
    lt, rt = _prune(nodes, 2 * i), _prune(nodes, 2 * i + 1)
    if lt[1] is None and rt[1] is None and lt[0]["prediction"] == rt[0]["prediction"]:
        return (dict(r, leaf=True, feature=-1, threshold=0.0, gain=0.0, cats=None, prediction=lt[0]["prediction"]),
                None)
    return (r, (lt, rt))


def flatten(trees):
    cols = {k: [] for k in ("feature", "threshold", "left", "right", "prediction", "impurity", "gain", "count")}
    cats, off, depth = [], [0], []

    def emit(tree, d):
        r, ch = tree
        me = len(cols["feature"])
        cols["feature"].append(r["feature"] if ch else -1)
        cols["threshold"].append(r["threshold"] if ch else 0.0)
        cols["left"].append(-1)
        cols["right"].append(-1)
        cols["prediction"].append(r["prediction"])
        cols["impurity"].append(r["impurity"])
        cols["gain"].append(r["gain"] if ch else 0.0)
        cols["count"].append(r["count"])
        cats.append(r["cats"] if ch and r["cats"] is not None else np.zeros(0, np.int32))
        dd = d
        if ch:
            cols["left"][me], dl = emit(ch[0], d + 1)
            cols["right"][me], dr = emit(ch[1], d + 1)
            dd = max(dl, dr)
        return me, dd

    for nodes in trees:
        _, d = emit(_prune(nodes, 1), 0)
        off.append(len(cols["feature"]))
        depth.append(d)
    types = dict(feature=np.int32, threshold=np.float64, left=np.int32, right=np.int32, prediction=np.float64,
                 impurity=np.float64, gain=np.float64, count=np.int64)
    out = {k: np.array(v, types[k]) for k, v in cols.items()}
    out["tree_off"] = np.array(off, np.int32)
    out["depth"] = np.array(depth, np.int32)
    out["cat_off"] = np.concatenate([[0], np.cumsum([c.size for c in cats])]).astype(np.int64)
    out["cat_ids"] = (np.concatenate(cats) if cats else np.zeros(0)).astype(np.int32)
    return out


def tree_predict(forest, x):
    """Each tree's prediction [T, n]."""
    x = np.asarray(x, np.float64)
    n = x.shape[0]
    feat, thr, lft, rgt = forest["feature"], forest["threshold"], forest["left"], forest["right"]
    co, ci = forest["cat_off"], forest["cat_ids"]
    T = len(forest["tree_off"]) - 1
    out = np.zeros((T, n))
    for t in range(T):
        for r in range(n):
            i = int(forest["tree_off"][t])
            while feat[i] >= 0:
                v = x[r, feat[i]]
                if co[i + 1] > co[i]:
                    go = bool(np.any(ci[co[i]:co[i + 1]].astype(np.float64) == v))
                else:
                    go = v <= thr[i]
                i = int(lft[i] if go else rgt[i])
            out[t, r] = forest["prediction"][i]
    return out


def predict(forest, x):
    """The mean over trees: predictions summed in tree order from 0.0, divided by numTrees."""
    tp = tree_predict(forest, x)
    acc = np.zeros(tp.shape[1])
    for t in range(tp.shape[0]):
        acc = acc + tp[t]
    return acc / float(tp.shape[0])
