"""Vectorised numpy restatement of the similarproduct template's CooccurrenceAlgorithm.trainCooccurrence, with the tie
rule of pio_cooc_train: distinct (user, item); every pair item1 < item2 of one user's items; the number of users per
pair; per item its partners ranked by (count descending, item ascending), the first topn kept.  Same outputs as
oracle.cooc_train (items [n_items, topn] padded with -1, counts [n_items, topn] padded with 0, n [n_items]), at numpy
speed: tens of millions of pairs."""
import numpy as np


def pair_total(user, item, n_items):
    """Number of (user, item1 < item2) pairs: sum over users of k (k - 1) / 2, k = the user's distinct items."""
    key = np.unique(np.asarray(user, np.int64) * n_items + np.asarray(item, np.int64))
    k = np.unique(key // n_items, return_counts=True)[1].astype(np.int64)
    return int((k * (k - 1) // 2).sum())


def cooc_train(user, item, n_items, topn):
    key = np.unique(np.asarray(user, np.int64) * n_items + np.asarray(item, np.int64))   # sorted by user, then item
    du, di = key // n_items, key % n_items
    m = key.shape[0]
    first = np.r_[True, du[1:] != du[:-1]]
    start = np.maximum.accumulate(np.where(first, np.arange(m), 0))
    rank = np.arange(m) - start                            # element e pairs with the rank[e] earlier items of its user
    e = np.repeat(np.arange(m), rank)
    t = np.arange(e.shape[0]) - np.repeat(np.cumsum(rank) - rank, rank)
    lo, hi = di[start[e] + t], di[e]
    oi = np.full((n_items, topn), -1, np.int32)
    oc = np.zeros((n_items, topn), np.int32)
    on = np.zeros(n_items, np.int32)
    if e.shape[0] == 0:
        return oi, oc, on
    pk, cnt = np.unique(lo * n_items + hi, return_counts=True)
    a, b = pk // n_items, pk % n_items
    it = np.r_[a, b]
    other = np.r_[b, a]
    c = np.r_[cnt, cnt]
    order = np.lexsort((other, -c, it))
    it, other, c = it[order], other[order], c[order]
    head = np.r_[True, it[1:] != it[:-1]]
    r = np.arange(it.shape[0]) - np.maximum.accumulate(np.where(head, np.arange(it.shape[0]), 0))
    keep = r < topn
    oi[it[keep], r[keep]] = other[keep]
    oc[it[keep], r[keep]] = c[keep]
    on[:] = np.minimum(np.bincount(it, minlength=n_items), topn)
    return oi, oc, on
