"""Plain restatement of pio_popular_predict_filtered: the ecommerce template's predictDefault over one fixed per-item
score with a pio_als_query_filter's lists, and the split of a batch into parts.  No arithmetic on the scores: the GPU
tests compare with it bit for bit."""
import numpy as np

ENTRY_LIMIT = 1 << 32    # a query with this many entries (list entries plus output slots) or more is rejected


def predict(scores, n_queries, topk, exclude=None, white=None, set_ix=None, item_sets=None):
    """(items int32 [n, topk], scores float64 [n, topk], count int32 [n]).  The candidates of query j are the items i in
    [0, n_items) that are not in exclude[j], not set in item_sets[set_ix[j]], and in white[j] when that is a list (ids
    out of range and duplicates ignored).  They are ordered by scores[i] descending, -0.0 == +0.0, equal scores by item
    index ascending, and cut at topk; a score is returned as it is, so a -0.0 stays -0.0."""
    scores = np.asarray(scores, np.float64)
    n_items = scores.shape[0]
    oi = np.full((n_queries, topk), -1, np.int32)
    os_ = np.zeros((n_queries, topk), np.float64)
    oc = np.zeros(n_queries, np.int32)
    for j in range(n_queries):
        cand = np.ones(n_items, bool)
        if white is not None and white[j] is not None:
            cand[:] = False
            w = np.asarray(white[j], np.int64).reshape(-1)
            cand[w[(w >= 0) & (w < n_items)]] = True
        if exclude is not None and exclude[j] is not None:
            x = np.asarray(exclude[j], np.int64).reshape(-1)
            cand[x[(x >= 0) & (x < n_items)]] = False
        if set_ix is not None and set_ix[j] >= 0:
            cand &= item_sets[set_ix[j]] == 0
        ids = np.flatnonzero(cand)
        ids = ids[np.lexsort((ids, -scores[ids]))][:topk]   # numpy compares -0.0 == +0.0, as Python's sort does
        k = ids.shape[0]
        oi[j, :k], os_[j, :k], oc[j] = ids, scores[ids], k
    return oi, os_, oc


def entries(topk, exclude=None, white=None, j=0):
    """Query j's entries in the part rule: its exclusion and white-list entries as listed, plus its topk output slots."""
    n = topk
    for lists in (exclude, white):
        if lists is not None and lists[j] is not None:
            n += len(lists[j])
    return n


def parts(n_queries, topk, budget, exclude=None, white=None):
    """The first query of each part: a part closes before the query that would take its entries over the budget (capped
    at 2^32 - 1); every part holds at least one query.  ValueError for a query with 2^32 entries or more."""
    budget = min(budget, ENTRY_LIMIT - 1)
    first, acc = [], 0
    for j in range(n_queries):
        e = entries(topk, exclude, white, j)
        if e >= ENTRY_LIMIT:
            raise ValueError(f"query {j} is too large")
        if j == 0 or acc + e > budget:
            first.append(j)
            acc = 0
        acc += e
    return first
