"""fp64 NumPy restatement of the filtered batch calls (pio_als_recommend_filtered / pio_als_similar_batch_filtered).

The definition is that of tests/test_gpu_filtered.py: the candidates of query j are the items the unfiltered call would
consider under the dense mask

    item_mask | item_sets[set_ix[j]] | (exclusion list of j) | (complement of the white list of j, if has_wl[j])

Ids below 0 or past the item range, and duplicates, match nothing.  set_ix[j] == -1 (or set_ix None) names no row; a
white list of None means "no white list", an empty one "no candidates".  Scores, the tie order (-score, item id) and the
-1 / 0 padding are those of tests/scoring_ref.py, which this module reuses for the arithmetic.

Unlike a per-query dense mask this is vectorised over chunks of queries: the candidate matrix of a chunk is built with
scatters, the scores with the index-order loops of scoring_ref, and the ranking with one lexsort along the item axis, so
the grid-split cases (hundreds of thousands of queries, a few thousand of them checked) stay in seconds on the host.
"""
from __future__ import annotations

import numpy as np

import scoring_ref


def _flat(lists, rows):
    """(query index within rows, item id) of every entry of lists[rows[c]]; None lists are empty."""
    qs, ids = [], []
    for c, j in enumerate(rows):
        l = lists[j]
        if l is None:
            continue
        a = np.asarray(l, np.int64).reshape(-1)
        if a.size:
            qs.append(np.full(a.size, c, np.int64))
            ids.append(a)
    if not qs:
        return np.zeros(0, np.int64), np.zeros(0, np.int64)
    return np.concatenate(qs), np.concatenate(ids)


def candidates(n_items, item_has, mask, rows, exclude=None, white=None, set_ix=None, item_sets=None):
    """bool [len(rows), n_items]: the candidates of the queries rows before scoring (the score > 0 rule of the cosine and
    the query's own items come on top)."""
    base = scoring_ref._candidates(n_items, item_has, mask)
    ok = np.repeat(base[None, :], len(rows), axis=0)
    rows = np.asarray(rows, np.int64)
    if set_ix is not None and item_sets is not None:
        r = np.asarray(set_ix, np.int64)[rows]
        sel = np.flatnonzero(r >= 0)
        if sel.size:
            ok[sel] &= np.asarray(item_sets)[r[sel]] == 0
    if exclude is not None:
        q, e = _flat(exclude, rows)
        keep = (e >= 0) & (e < n_items)
        ok[q[keep], e[keep]] = False
    if white is not None:
        has = np.array([white[j] is not None for j in rows], bool)
        allow = np.zeros_like(ok)
        q, w = _flat(white, rows)
        keep = (w >= 0) & (w < n_items)
        allow[q[keep], w[keep]] = True
        ok[has] &= allow[has]
    return ok


def rank_rows(scores, ok, topk):
    """best topk of every row of scores[ok] by (-score, id): (items [n, topk], scores float32 [n, topk], count [n])."""
    n, n_items = scores.shape
    key = np.where(ok, -scores, np.inf)          # non-candidates sort last; candidate scores are finite
    ids = np.broadcast_to(np.arange(n_items), scores.shape)
    order = np.lexsort((ids, key), axis=-1)[:, :topk]
    cnt = np.minimum(ok.sum(axis=1), topk)
    take = np.arange(order.shape[1])[None, :] < cnt[:, None]
    oi = np.full((n, topk), -1, np.int32)
    os_ = np.zeros((n, topk), np.float32)
    oi[:, :order.shape[1]] = np.where(take, order, -1)
    os_[:, :order.shape[1]] = np.where(take, np.take_along_axis(scores, order, axis=1), 0.0).astype(np.float32)
    return oi, os_, cnt.astype(np.int32)


def _chunk(n_items, budget=1 << 23):
    return max(1, budget // max(1, n_items))


def recommend(uf, uh, itf, ih, users, topk, mask=None, weight=None, exclude=None, white=None, set_ix=None,
              item_sets=None):
    """pio_als_recommend_filtered: (items [n, topk], scores [n, topk], count [n]); an unknown user has no candidates."""
    users = np.asarray(users, np.int64)
    n, n_items, n_users = users.shape[0], itf.shape[0], uf.shape[0]
    oi = np.full((n, topk), -1, np.int32)
    os_ = np.zeros((n, topk), np.float32)
    oc = np.zeros(n, np.int32)
    known = (users >= 0) & (users < n_users)
    if uh is not None:
        known[known] &= np.asarray(uh)[users[known]].astype(bool)
    w = None if weight is None else np.asarray(weight, np.float64)
    rows = np.flatnonzero(known)
    step = _chunk(n_items)
    for c0 in range(0, rows.shape[0], step):
        r = rows[c0:c0 + step]
        s = scoring_ref.dot_scores(np.asarray(uf)[users[r]], itf)
        if w is not None:
            s = s * w[None, :]
        ok = candidates(n_items, ih, mask, r, exclude, white, set_ix, item_sets)
        oi[r], os_[r], oc[r] = rank_rows(s, ok, topk)
    return oi, os_, oc


def similar_batch(itf, ih, queries, topk, mask=None, weight=None, keep_query=False, exclude=None, white=None,
                  set_ix=None, item_sets=None):
    """pio_als_similar_batch_filtered: (items [n, topk], scores [n, topk], count [n])."""
    y = scoring_ref._f64(itf)
    n_items, k = y.shape
    n = len(queries)
    has = np.ones(n_items, bool) if ih is None else np.asarray(ih).astype(bool)
    n2 = np.zeros(n_items)
    for t in range(k):
        n2 += y[:, t] * y[:, t]
    sqrt_n2 = np.sqrt(n2)
    w = None if weight is None else np.asarray(weight, np.float64)
    oi = np.full((n, topk), -1, np.int32)
    os_ = np.zeros((n, topk), np.float32)
    oc = np.zeros(n, np.int32)
    step = _chunk(n_items)
    for c0 in range(0, n, step):
        rows = np.arange(c0, min(n, c0 + step))
        qs = [np.asarray(queries[j], np.int64).reshape(-1) for j in rows]
        # the valid query vectors of the chunk, in query order: their row in the chunk and their position in the query
        vrow, vid, vpos = [], [], []
        for c, q in enumerate(qs):
            v = q[(q >= 0) & (q < n_items)]
            v = v[has[v]]
            vrow.append(np.full(v.size, c, np.int64))
            vid.append(v)
            vpos.append(np.arange(v.size))
        vrow, vid, vpos = np.concatenate(vrow), np.concatenate(vid), np.concatenate(vpos)
        s = np.zeros((rows.size, n_items))
        if vid.size:
            yq = y[vid]
            n1 = np.zeros(vid.size)
            d = np.zeros((vid.size, n_items))
            for t in range(k):
                n1 += yq[:, t] * yq[:, t]
                d += yq[:, t, None] * y[None, :, t]
            n1n2 = np.sqrt(n1)[:, None] * sqrt_n2[None, :]
            with np.errstate(divide="ignore", invalid="ignore"):
                term = np.where(n1n2 == 0.0, 0.0, d / np.where(n1n2 == 0.0, 1.0, n1n2))
            for p in range(int(vpos.max()) + 1):    # the terms of a query are summed in query order
                sel = np.flatnonzero(vpos == p)
                s[vrow[sel]] += term[sel]
        if w is not None:
            s = s * w[None, :]
        ok = candidates(n_items, ih, mask, rows, exclude, white, set_ix, item_sets) & (s > 0)
        if not keep_query:
            for c, q in enumerate(qs):
                ok[c, q[(q >= 0) & (q < n_items)]] = False
        oi[rows], os_[rows], oc[rows] = rank_rows(s, ok, topk)
    return oi, os_, oc
