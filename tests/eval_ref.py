"""numpy restatement of the recommendation template's k-fold evaluation on global indices, as pio_eval_folds computes it
(csrc/eval_folds.cuh, DESIGN.md 4.11).  The template's definitions it restates (templates/recommendation.py):
DataSource.readEval (rating e is tested in fold e % kFold, the queries are the distinct test users in by_user order),
ALSAlgorithm.train (BiMap.stringInt of the fold's training users / items) and PrecisionAtK / PositiveCount.calculate_one.

user / item: global indices of all ratings (any dense numbering: the fold maps do not depend on it), rating: fp64."""
import numpy as np

NONE = np.iinfo(np.int64).max


def fold_map(g: np.ndarray, k_fold: int, f: int):
    """(loc, l2g): the fold-local index of every global id (-1 when it has no training rating in fold f) and the global id
    of every fold-local index, in order of first training occurrence.  The first training occurrence is computed the way
    the device does: e1 = the id's first position, e2 = its first position in a fold other than fold(e1); it is e1 when
    fold(e1) != f, else e2."""
    n = g.shape[0]
    n_ids = int(g.max()) + 1 if n else 0
    pos = np.arange(n, dtype=np.int64)
    e1 = np.full(n_ids, NONE, np.int64)
    np.minimum.at(e1, g, pos)
    other = pos % k_fold != e1[g] % k_fold
    e2 = np.full(n_ids, NONE, np.int64)
    np.minimum.at(e2, g[other], pos[other])
    t = np.where(e1 % k_fold != f, e1, e2)
    ids = np.flatnonzero(t != NONE)
    l2g = ids[np.argsort(t[ids], kind="stable")]
    loc = np.full(n_ids, -1, np.int64)
    loc[l2g] = np.arange(l2g.shape[0])
    return loc, l2g


def split(user, item, rating, k_fold: int):
    """Per fold f, a dict: user / item (l2g maps), train_user / train_item / train_rating (the training COO in rating
    order: fold-local indices, float32 ratings), query_user (global) / query_train_user (fold-local or -1), and test_q /
    test_item / test_rating (every test rating: its query, global item and fp64 value)."""
    user, item = np.asarray(user, np.int64), np.asarray(item, np.int64)
    rating = np.asarray(rating, np.float64)
    pos = np.arange(user.shape[0])
    folds = []
    for f in range(k_fold):
        uloc, ul2g = fold_map(user, k_fold, f)
        iloc, il2g = fold_map(item, k_fold, f)
        tr, te = pos % k_fold != f, pos % k_fold == f
        tu = user[te]
        _, first = np.unique(tu, return_index=True)
        qu = tu[np.sort(first)]                     # distinct test users in order of first occurrence
        qix = np.full(int(user.max()) + 1, -1, np.int64)
        qix[qu] = np.arange(qu.shape[0])
        folds.append(dict(user=ul2g, item=il2g, train_user=uloc[user[tr]], train_item=iloc[item[tr]],
                          train_rating=rating[tr].astype(np.float32), query_user=qu, query_train_user=uloc[qu],
                          test_q=qix[tu], test_item=item[te], test_rating=rating[te]))
    return folds


def rank_counts(fold: dict, items: np.ndarray, count: np.ndarray, k: int, threshold: float):
    """hits, npos, nraw per query of `fold` for a top-N result (items [n_queries, num] of fold-local indices, count valid
    entries per query): hits among the first min(k, count) items of a test item with a rating >= threshold, the number of
    distinct such test items, and the number of test ratings >= threshold."""
    nq = fold["query_user"].shape[0]
    num = items.shape[1]
    hits, npos, nraw = (np.zeros(nq, np.int64) for _ in range(3))
    for q in range(nq):
        mine = fold["test_q"] == q
        ok = fold["test_rating"][mine] >= threshold
        positives = set(fold["test_item"][mine][ok].tolist())
        nraw[q] = int(ok.sum())
        npos[q] = len(positives)
        kk = min(k, int(count[q]), num)
        hits[q] = sum(int(fold["item"][items[q, j]]) in positives for j in range(kk))
    return hits, npos, nraw


def precision_values(hits, npos, k: int):
    """PrecisionAtK's per-query values in query order, queries without positives left out."""
    return [h / min(k, p) for h, p in zip(hits.tolist(), npos.tolist()) if p > 0]
