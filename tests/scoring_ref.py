"""fp64 NumPy restatement of top-k scoring (pio_als_recommend / pio_als_similar[_batch]), independent of oracle/.

Bit-exact by construction: the product of two fp32 values widened to fp64 is exact (48 significant bits fit in 53), so
the fused multiply-add fma(x, y, acc) of the kernels and the reference's `acc += x * y` both round once, to acc + x*y.
Looping over the features in index order, vectorised over items (and users), gives the same sums bit for bit.

  dot     score_i = (sum_t x_t * y_it) * weight_i
  cosine  score_i = (sum over the valid query vectors q, in query order, of d / (sqrt(n1) * sqrt(n2)), or 0 when that
          product is 0) * weight_i; only score > 0 is a candidate.  Duplicate query ids count twice; unknown, out-of-range
          and factor-less query ids are skipped; query ids are not candidates unless keep_query is set.
  both    items without a factor and masked items are not candidates; ranking by (-score, item id), so -0.0 ties +0.0 and
          ties go to the smaller id; scores are returned as float32(score); rows are padded with -1 / 0.
"""
from __future__ import annotations

import numpy as np


def _f64(a):
    return np.asarray(a, np.float32).astype(np.float64)


def _candidates(n_items, item_has, mask):
    ok = np.ones(n_items, bool) if item_has is None else np.asarray(item_has).astype(bool).copy()
    if mask is not None:
        ok &= np.asarray(mask) == 0
    return ok


def _rank(scores, ok, topk):
    """best `topk` of scores[ok] by (-score, id): (items int32[topk], scores float32[topk], count)."""
    ids = np.flatnonzero(ok)
    s = scores[ids]
    order = np.lexsort((ids, -s))[:topk]
    oi = np.full(topk, -1, np.int32)
    os_ = np.zeros(topk, np.float32)
    oi[:len(order)] = ids[order]
    os_[:len(order)] = s[order].astype(np.float32)
    return oi, os_, len(order)


def dot_scores(x, item_f):
    """fp64 index-order dot products: x [n, k] (fp32 values) x item_f [m, k] -> [n, m]."""
    x, y = _f64(x), _f64(item_f)
    acc = np.zeros((x.shape[0], y.shape[0]))
    for t in range(y.shape[1]):
        acc += x[:, t, None] * y[None, :, t]
    return acc


def recommend(user_f, user_has, item_f, item_has, users, topk, mask=None, weight=None, chunk=256):
    """pio_als_recommend: (items [n, topk], scores [n, topk], count [n]); an unknown user has no candidates."""
    users = np.asarray(users, np.int64)
    n_users, n_items = user_f.shape[0], item_f.shape[0]
    n = users.shape[0]
    oi = np.full((n, topk), -1, np.int32)
    os_ = np.zeros((n, topk), np.float32)
    oc = np.zeros(n, np.int32)
    ok = _candidates(n_items, item_has, mask)
    w = None if weight is None else np.asarray(weight, np.float64)
    known = (users >= 0) & (users < n_users)
    if user_has is not None:
        known[known] &= np.asarray(user_has)[users[known]].astype(bool)
    rows = np.flatnonzero(known)
    for c0 in range(0, rows.shape[0], chunk):
        r = rows[c0:c0 + chunk]
        s = dot_scores(np.asarray(user_f)[users[r]], item_f)
        if w is not None:
            s = s * w[None, :]
        for j, q in enumerate(r):
            oi[q], os_[q], oc[q] = _rank(s[j], ok, topk)
    return oi, os_, oc


def cosine_scores(item_f, item_has, query):
    """sum over the valid query vectors of cosine(y_q, y_i), fp64, for every item (before weights and filters)."""
    y = _f64(item_f)
    n_items, k = y.shape
    has = np.ones(n_items, bool) if item_has is None else np.asarray(item_has).astype(bool)
    n2 = np.zeros(n_items)
    for t in range(k):
        n2 += y[:, t] * y[:, t]
    sqrt_n2 = np.sqrt(n2)
    score = np.zeros(n_items)
    for q in np.asarray(query, np.int64):
        if q < 0 or q >= n_items or not has[q]:
            continue
        n1 = 0.0
        d = np.zeros(n_items)
        for t in range(k):
            n1 += y[q, t] * y[q, t]
            d += y[q, t] * y[:, t]
        n1n2 = np.sqrt(n1) * sqrt_n2
        with np.errstate(divide="ignore", invalid="ignore"):
            score += np.where(n1n2 == 0.0, 0.0, d / np.where(n1n2 == 0.0, 1.0, n1n2))
    return score


def similar(item_f, item_has, query, topk, mask=None, weight=None, keep_query=False):
    """pio_als_similar: (items [topk], scores [topk], count)."""
    n_items = item_f.shape[0]
    s = cosine_scores(item_f, item_has, query)
    if weight is not None:
        s = s * np.asarray(weight, np.float64)
    ok = _candidates(n_items, item_has, mask) & (s > 0)
    if not keep_query:
        q = np.asarray(query, np.int64)
        ok[q[(q >= 0) & (q < n_items)]] = False
    return _rank(s, ok, topk)


def similar_batch(item_f, item_has, queries, topk, mask=None, weight=None, keep_query=False):
    """pio_als_similar_batch: (items [n, topk], scores [n, topk], count [n])."""
    n = len(queries)
    oi = np.full((n, topk), -1, np.int32)
    os_ = np.zeros((n, topk), np.float32)
    oc = np.zeros(n, np.int32)
    for j, q in enumerate(queries):
        oi[j], os_[j], oc[j] = similar(item_f, item_has, q, topk, mask, weight, keep_query)
    return oi, os_, oc
