"""NumPy restatement of the RandomForest classifier of pio_rf_train: the definition the GPU forest is checked against.

It follows MLlib 2.4's `RandomForest.trainClassifier` (continuous features, no categorical ones) step by step:
  - arguments: Strategy.assertValid and RandomForest.run's checks, featureSubsetStrategy (auto|all|sqrt|log2|onethird,
    an integer k > 0 meaning min(k, F), a fraction r in (0, 1] meaning ceil(r F); auto = all for one tree, else sqrt);
  - labels: the class is trunc(label); a label < 0 or >= numClasses raises GiniAggregator's / EntropyAggregator's
    message;
  - findSplitsForContinuousFeature: numBins = min(maxBins, n); a Bernoulli split sample of fraction
    max(maxBins^2, 10000) / n when n is larger; every midpoint of the distinct sampled values when there are at most
    numBins - 1, else the greedy stride walk; a row goes left of t iff x <= t;
  - bagging: Poisson(1) weights per (tree, row) when numTrees > 1, weight 1 for a single tree;
  - level-wise growth over heap-numbered nodes (root 1, children 2i, 2i + 1), calculateImpurityStats' gain
    imp(parent) - nL/n imp(L) - nR/n imp(R), invalid when nL < 1, nR < 1 or gain < 0, binsToBestSplit's maxBy (the
    first maximum); a node is a leaf at maxDepth, at gain <= 0 or without a valid split, a child with impurity 0 is a
    leaf at once; LearningNode.toNode(prune = true) collapses an internal node whose two leaf children predict the same
    class;
  - predict: x[f] <= threshold goes left; the forest's majority vote.

This project's choices, where MLlib leaves things to Spark's partitioning or to chance:
  - every random draw is a pure function of (seed, stream, tree, index) through the splitmix64 finaliser (rf_mix),
    in place of Spark's per-partition XORShift; the bag weight is the inverse CDF of a 53-bit uniform over one fp64
    table of P(X <= k), k = 0 .. 15, so weights are capped at 16;
  - the feature subset of a node is the k features with the smallest keys, considered in ascending feature order, so
    ties between features go to the smaller feature, and ties between classes go to the smaller class (leaf prediction
    and vote);
  - log2 is ceil(log2 F) computed on integers; non-finite labels and features are rejected; -0.0 counts as 0.0;
  - the integer and decimal spellings of featureSubsetStrategy follow a fixed grammar (see subset_size);
  - limits: numClasses <= 64, maxBins <= 65536, n < 2^31.

A forest is a dict of flat per-node arrays, trees one after the other, each in preorder (node, left subtree, right
subtree): tree_off [numTrees + 1], feature (-1 at a leaf), threshold (0 at a leaf), left / right (indices into the flat
arrays, -1 at a leaf), prediction, impurity, gain (0 at a leaf) and count (the node's weighted row count).
"""
import math
import re

import numpy as np

GINI, ENTROPY = 0, 1
IMPURITIES = {"gini": GINI, "entropy": ENTROPY}
TAG_SAMPLE, TAG_BAG, TAG_SUBSET = 1, 2, 3
MAX_CLASSES, MAX_BINS, MAX_DEPTH, POISSON_N = 64, 65536, 30, 16
LN2 = float.fromhex("0x1.62e42fefa39efp-1")
_M64 = (1 << 64) - 1
STRATEGIES = "auto, all, onethird, sqrt, log2"


def mix_int(x):
    x = (x + 0x9E3779B97F4A7C15) & _M64
    z = ((x ^ (x >> 30)) * 0xBF58476D1CE4E5B9) & _M64
    z = ((z ^ (z >> 27)) * 0x94D049BB133111EB) & _M64
    return z ^ (z >> 31)


def mix(x):
    """rf_mix over a uint64 array (wrapping arithmetic)."""
    with np.errstate(over="ignore"):
        x = np.asarray(x, np.uint64) + np.uint64(0x9E3779B97F4A7C15)
        z = (x ^ (x >> np.uint64(30))) * np.uint64(0xBF58476D1CE4E5B9)
        z = (z ^ (z >> np.uint64(27))) * np.uint64(0x94D049BB133111EB)
        return z ^ (z >> np.uint64(31))


def stream(seed, tag, t):
    return mix_int(mix_int((int(seed) & _M64) ^ (tag << 56)) ^ int(t))


def draw(base, index):
    return mix(np.uint64(base) ^ np.asarray(index, np.uint64))


def u53(h):
    return (np.asarray(h, np.uint64) >> np.uint64(11)).astype(np.float64) * (1.0 / 9007199254740992.0)


def poisson_table():
    p, c, out = float.fromhex("0x1.78b56362cef38p-2"), 0.0, []
    for k in range(POISSON_N):
        if k > 0:
            p = p / k
        c = c + p
        out.append(c)
    return np.array(out)


def bag_weights(seed, t, n):
    cdf = poisson_table()
    u = u53(draw(stream(seed, TAG_BAG, t), np.arange(n, dtype=np.uint64)))
    return (cdf[None, :] <= u[:, None]).sum(axis=1).astype(np.int64)


_INT = re.compile(r"[+-]?([0-9]+)")
_DEC = re.compile(r"[+-]?([0-9]+(\.[0-9]*)?|\.[0-9]+)([eE][+-]?[0-9]+)?")


def subset_size(s, n_feat, num_trees):
    """Features per node for featureSubsetStrategy s, or 0 when MLlib rejects s."""
    if s == "auto":
        s = "all" if num_trees == 1 else "sqrt"
    if s == "all":
        return n_feat
    if s == "sqrt":
        return int(math.ceil(math.sqrt(n_feat)))
    if s == "log2":
        return max(1, (n_feat - 1).bit_length())
    if s == "onethird":
        return int(math.ceil(n_feat / 3.0))
    m = _INT.fullmatch(s)
    if m and len(m.group(1)) <= 10 and -2 ** 31 <= int(s) < 2 ** 31:
        return min(int(s), n_feat) if int(s) > 0 else 0
    if _DEC.fullmatch(s):
        r = float(s)
        if 0.0 < r <= 1.0:
            return int(math.ceil(r * n_feat))
    return 0


def fmt_double(v):
    """A label as the error messages print it: the shortest %g that reads back, with '.0' on an integral value."""
    for p in range(1, 18):
        s = "%.*g" % (p, v)
        if float(s) == v:
            break
    return s if any(ch in s for ch in ".en") else s + ".0"


def check_args(num_classes, num_trees, strategy, impurity, max_depth, max_bins, n_feat=1, categorical=None):
    """Raises ValueError with MLlib's message (or this implementation's, for its limits) for bad arguments."""
    if impurity not in IMPURITIES:
        raise ValueError(f"Did not recognize Impurity name: {impurity}")
    if categorical:
        raise ValueError("categoricalFeaturesInfo must be empty: categorical features are not supported")
    check_numeric(num_classes, num_trees, strategy, max_depth, max_bins, n_feat)


def check_numeric(num_classes, num_trees, strategy, max_depth, max_bins, n_feat):
    if num_classes < 2:
        raise ValueError(f"DecisionTree Strategy for Classification must have numClasses >= 2, but numClasses = "
                         f"{num_classes}.")
    if num_classes > MAX_CLASSES:
        raise ValueError(f"numClasses = {num_classes}: at most {MAX_CLASSES} classes are supported.")
    if num_trees < 1:
        raise ValueError(f"RandomForest requires numTrees > 0, but was given numTrees = {num_trees}.")
    if subset_size(strategy, max(n_feat, 1), num_trees) == 0:
        raise ValueError(f"RandomForest given invalid featureSubsetStrategy: {strategy}. Supported values: "
                         f"{STRATEGIES}, (0.0-1.0], [1-n].")
    if max_depth < 0:
        raise ValueError(f"DecisionTree Strategy given invalid maxDepth parameter: {max_depth}.  Valid values are "
                         f"integers >= 0.")
    if max_depth > MAX_DEPTH:
        raise ValueError(f"DecisionTree currently only supports maxDepth <= 30, but was given maxDepth = {max_depth}.")
    if max_bins < 2:
        raise ValueError(f"DecisionTree Strategy given invalid maxBins parameter: {max_bins}.  Valid values are "
                         f"integers >= 2.")
    if max_bins > MAX_BINS:
        raise ValueError(f"maxBins = {max_bins}: at most {MAX_BINS} bins are supported.")


def check_data(labels, x, num_classes, impurity):
    """Rows and labels, checked in row order: first every non-finite value, then the label range."""
    n, n_feat = x.shape
    if n < 1 or n_feat < 1:
        raise ValueError("RandomForest requires at least one row and one feature.")
    if n >= 2 ** 31:
        raise ValueError("at most 2^31 - 1 rows are supported.")
    bad = ~np.isfinite(labels) | ~np.isfinite(x).all(axis=1)
    if bad.any():
        r = int(np.flatnonzero(bad)[0])
        if not np.isfinite(labels[r]):
            raise ValueError(f"label of row {r} is not finite ({fmt_double(labels[r])}).")
        f = int(np.flatnonzero(~np.isfinite(x[r]))[0])
        raise ValueError(f"feature {f} of row {r} is not finite ({fmt_double(x[r, f])}).")
    agg = "GiniAggregator" if impurity == "gini" else "EntropyAggregator"
    bad = (labels >= num_classes) | (labels < 0)
    if bad.any():
        v = float(labels[int(np.flatnonzero(bad)[0])])
        if v >= num_classes:
            raise ValueError(f"{agg} given label {fmt_double(v)} but requires label < numClasses (= {num_classes}).")
        raise ValueError(f"{agg} given label {fmt_double(v)}but requires label is non-negative.")


def sample_fraction(n, max_bins):
    req = max(float(max_bins) * float(max_bins), 10000.0)
    return req / n if n > req else 1.0


def thresholds(v, cnt, num_bins):
    """findSplitsForContinuousFeature over distinct ascending values v with counts cnt."""
    m = len(v)
    if m <= 1:
        return np.zeros(0)
    num_splits = num_bins - 1
    if m - 1 <= num_splits:
        with np.errstate(over="ignore"):                        # the midpoint of two values near +-1.8e308 is +-inf
            return np.array([(v[i - 1] + v[i]) / 2.0 for i in range(1, m)])
    stride = float(int(np.sum(cnt))) / float(num_splits + 1)
    out, cur, target = [], int(cnt[0]), stride
    for i in range(1, m):
        prev = cur
        cur += int(cnt[i])
        if abs(prev - target) < abs(cur - target):
            out.append((v[i - 1] + v[i]) / 2.0)
            target += stride
    return np.array(out)


def find_thresholds(x, max_bins, seed):
    n, n_feat = x.shape
    frac = sample_fraction(n, max_bins)
    rows = np.arange(n)
    if frac < 1.0:
        rows = rows[u53(draw(stream(seed, TAG_SAMPLE, 0), rows.astype(np.uint64))) < frac]
    nb = min(max_bins, n)
    out = []
    for f in range(n_feat):
        vals, cnt = np.unique(x[rows, f] + 0.0, return_counts=True)
        out.append(thresholds(vals, cnt, nb))
    return out


def node_subset(seed, t, node, n_feat, k):
    if k >= n_feat:
        return np.arange(n_feat)
    keys = draw(int(draw(stream(seed, TAG_SUBSET, t), node)), np.arange(n_feat, dtype=np.uint64))
    order = np.lexsort((np.arange(n_feat), keys))
    return np.sort(order[:k])


def impurity_of(c, kind):
    """Gini / Entropy of the class counts c [..., C] (int64), class by class as MLlib accumulates them."""
    c = np.asarray(c, np.int64)
    tot = c.sum(axis=-1)
    n = np.where(tot == 0, 1, tot).astype(np.float64)
    out = np.full(tot.shape, 1.0 if kind == GINI else 0.0)
    with np.errstate(divide="ignore", invalid="ignore"):
        for k in range(c.shape[-1]):
            f = c[..., k].astype(np.float64) / n
            if kind == GINI:
                out = out - f * f
            else:
                out = np.where(c[..., k] != 0, out - f * (np.log(f) / LN2), out)
    return np.where(tot == 0, 0.0, out)


def _gains(hist, n_thr_sub, kind):
    """hist [S, K, NB, C]: every candidate's gain [S, K, NB - 1] (-inf when invalid) and left counts."""
    total = hist[:, 0].sum(axis=1)                              # [S, C]
    left = np.cumsum(hist, axis=2)[:, :, :-1, :]                # split j: bins 0..j
    right = total[:, None, None, :] - left
    nl, nr, nt = left.sum(-1), right.sum(-1), total.sum(-1)
    ip = impurity_of(total, kind)[:, None, None]
    il, ir = impurity_of(left, kind), impurity_of(right, kind)
    n = np.where(nt == 0, 1, nt).astype(np.float64)[:, None, None]
    gain = (ip - (nl / n) * il) - (nr / n) * ir
    j = np.arange(hist.shape[2] - 1)[None, None, :]
    ok = (j < n_thr_sub[:, :, None]) & (nl >= 1) & (nr >= 1) & (gain >= 0)
    return np.where(ok, gain, -np.inf), left, total


def train(labels, x, num_classes, num_trees, strategy, impurity, max_depth, max_bins, seed=0, categorical=None,
          return_nodes=False):
    labels = np.asarray(labels, np.float64)
    x = np.asarray(x, np.float64)
    check_args(num_classes, num_trees, strategy, impurity, max_depth, max_bins, x.shape[1], categorical)
    check_data(labels, x, num_classes, impurity)
    kind = IMPURITIES[impurity]
    n, n_feat = x.shape
    cls = np.trunc(labels).astype(np.int64)
    k = subset_size(strategy, n_feat, num_trees)
    thr = find_thresholds(x, max_bins, seed)
    n_thr = np.array([len(t) for t in thr])
    nb = int(n_thr.max()) + 1
    bins = np.stack([np.searchsorted(thr[f], x[:, f], side="left") for f in range(n_feat)], axis=1)
    trees, runner_up, level_slots = [], [], []
    for t in range(num_trees):
        w = np.ones(n, np.int64) if num_trees == 1 else bag_weights(seed, t, n)
        nodes = {}
        at = np.ones(n, np.int64)                               # heap index of each row's node; 0 = at a leaf
        active, level = [1], 0
        level_slots.append([])
        while active:
            level_slots[-1].append(len(active))
            act = np.array(active)
            sub = np.stack([node_subset(seed, t, i, n_feat, k) for i in active])           # [S, K]
            live = np.flatnonzero(at > 0)
            slot = np.searchsorted(act, at[live])              # each live row's slot, before this level moves any row
            nxt = []
            # the level's histograms and gains in batches of slots, so that a level of many large slots fits in memory
            step = max(1, BATCH_ENTRIES // (k * nb * num_classes))
            for b0 in range(0, len(act), step):
                b1 = min(len(act), b0 + step)
                sel = (slot >= b0) & (slot < b1)
                lr, ls = live[sel], slot[sel] - b0
                hist = np.zeros((b1 - b0, k, nb, num_classes), np.int64)
                for kk in range(k):
                    b = bins[lr, sub[b0 + ls, kk]]
                    idx = (ls * nb + b) * num_classes + cls[lr]
                    hist[:, kk] = np.bincount(idx, weights=w[lr], minlength=(b1 - b0) * nb * num_classes).astype(
                        np.int64).reshape(b1 - b0, nb, num_classes)
                gain, left, total = _gains(hist, n_thr[sub[b0:b1]], kind)
                flat = gain.reshape(b1 - b0, -1)
                best = flat.argmax(axis=1) if flat.shape[1] else np.zeros(b1 - b0, np.int64)
                for s in range(b1 - b0):
                    _decide(nodes, nxt, at, bins, thr, sub[b0 + s], active[b0 + s], flat[s], best[s], left[s],
                            total[s], nb, num_classes, kind, level, max_depth, runner_up)
            active, level = sorted(nxt), level + 1
        trees.append(nodes)
    forest = flatten(trees, num_classes)
    if return_nodes:
        return forest, dict(thresholds=thr, runner_up=runner_up, subset_size=k, trees=trees, level_slots=level_slots)
    return forest


# entries of one batch of slot histograms in train (int64; cumulative counts and impurities are as large again)
BATCH_ENTRIES = 1 << 22


def _decide(nodes, nxt, at, bins, thr, sub, i, flat, best, left, tot, nb, num_classes, kind, level, max_depth,
            runner_up):
    """Node i's record from its candidates' gains `flat` [K (NB - 1)], the first maximum `best`, left counts `left`
    [K, NB - 1, C] and class totals `tot`; its children go to `nxt` (or are leaves) and its rows move to them in `at`."""
    g = flat[best] if flat.shape[0] else -np.inf
    if np.isfinite(g):
        # the best gain among candidates whose left counts differ from the best's (equal counts give equal gains on
        # any device)
        lc = left.reshape(-1, num_classes)
        other = (lc != lc[best]).any(axis=1)
        runner_up.append((g, flat[other].max() if other.any() else -np.inf))
    rec = dict(counts=tot, impurity=float(impurity_of(tot, kind)), prediction=int(np.argmax(tot)), gain=0.0, leaf=True,
               feature=-1, threshold=0.0)
    nodes[i] = rec
    rows = at == i
    if not np.isfinite(g) or g <= 0 or level == max_depth:
        at[rows] = 0
        return
    kk, j = divmod(int(best), nb - 1)
    f = int(sub[kk])
    rec.update(leaf=False, feature=f, threshold=float(thr[f][j]), gain=float(g))
    lc = left[kk, j]
    for child, cc in ((2 * i, lc), (2 * i + 1, tot - lc)):
        ci = float(impurity_of(cc, kind))
        if level + 1 == max_depth or ci == 0.0:
            nodes[child] = dict(counts=cc, impurity=ci, prediction=int(np.argmax(cc)), gain=0.0, leaf=True, feature=-1,
                                threshold=0.0)
        else:
            nxt.append(child)
    go_left = bins[:, f] <= j
    at[rows & go_left] = 2 * i if (2 * i) in nxt else 0
    at[rows & ~go_left] = 2 * i + 1 if (2 * i + 1) in nxt else 0


def _prune(nodes, i):
    """LearningNode.toNode(prune = true): (record, children) with an internal node of two equal leaves collapsed."""
    r = nodes[i]
    if r["leaf"]:
        return (r, None)
    lt, rt = _prune(nodes, 2 * i), _prune(nodes, 2 * i + 1)
    if lt[1] is None and rt[1] is None and lt[0]["prediction"] == rt[0]["prediction"]:
        return (dict(r, leaf=True, feature=-1, threshold=0.0, gain=0.0, prediction=lt[0]["prediction"]), None)
    return (r, (lt, rt))


def flatten(trees, num_classes):
    cols = {k: [] for k in ("feature", "threshold", "left", "right", "prediction", "impurity", "gain", "count")}
    off, depth = [0], []

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
        cols["count"].append(int(np.sum(r["counts"])))
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
    types = dict(feature=np.int32, threshold=np.float64, left=np.int32, right=np.int32, prediction=np.int32,
                 impurity=np.float64, gain=np.float64, count=np.int64)
    out = {k: np.array(v, types[k]) for k, v in cols.items()}
    out["tree_off"] = np.array(off, np.int32)
    out["depth"] = np.array(depth, np.int32)
    out["num_classes"] = num_classes
    return out


def predict(forest, x):
    x = np.asarray(x, np.float64)
    n = x.shape[0]
    votes = np.zeros((n, forest["num_classes"]), np.int64)
    feat, thr, lft, rgt = forest["feature"], forest["threshold"], forest["left"], forest["right"]
    for t in range(len(forest["tree_off"]) - 1):
        at = np.full(n, forest["tree_off"][t], np.int64)
        while True:
            inner = feat[at] >= 0
            if not inner.any():
                break
            r = np.flatnonzero(inner)
            go = x[r, feat[at[r]]] <= thr[at[r]]
            at[r] = np.where(go, lft[at[r]], rgt[at[r]])
        votes[np.arange(n), forest["prediction"][at]] += 1
    return votes.argmax(axis=1).astype(np.float64)
