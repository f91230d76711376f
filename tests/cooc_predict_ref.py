"""NumPy restatement of pio_cooc_predict_filtered: the similarproduct template's CooccurrenceAlgorithm.predict over the
model arrays (top_items / top_counts [n_items, n], top_n [n_items]) with a pio_als_query_filter's lists, and the split
of a batch into parts.  Integer work throughout: the GPU tests compare with it exactly."""
import numpy as np

SCAN_LIMIT = 1 << 32     # a query expanding to this many entries or more is rejected
IDS_LIMIT = 1 << 31      # a part's listed ids stay below this


def predict(top_items, top_counts, top_n, q_lists, topk, exclude=None, white=None, set_ix=None, item_sets=None):
    """(items int32 [n, topk], scores int64 [n, topk], count int32 [n]).  Query j's known items Q (ids outside the item
    range and repeats dropped) list their first top_n[q] entries; each candidate scores the sum of its counts over Q.  A
    candidate is dropped when it is in Q, when white[j] is a list that lacks it, when exclude[j] holds it, or when
    item_sets[set_ix[j]] marks it.  The rest: score descending, then item ascending, first topk."""
    n_items = top_n.shape[0]
    n = len(q_lists)
    oi = np.full((n, topk), -1, np.int32)
    os_ = np.zeros((n, topk), np.int64)
    oc = np.zeros(n, np.int32)
    for j, ql in enumerate(q_lists):
        ql = np.asarray(ql, np.int64).reshape(-1)
        q = np.unique(ql[(ql >= 0) & (ql < n_items)])
        if q.size == 0:
            continue
        cand = np.concatenate([top_items[i, :top_n[i]] for i in q]).astype(np.int64)
        cnt = np.concatenate([top_counts[i, :top_n[i]] for i in q]).astype(np.int64)
        if cand.size == 0:
            continue
        items, inv = np.unique(cand, return_inverse=True)
        score = np.zeros(items.shape[0], np.int64)
        np.add.at(score, inv, cnt)
        keep = ~np.isin(items, q)
        if white is not None and white[j] is not None:
            keep &= np.isin(items, np.asarray(white[j], np.int64))
        if exclude is not None and exclude[j] is not None:
            keep &= ~np.isin(items, np.asarray(exclude[j], np.int64))
        if set_ix is not None and set_ix[j] >= 0:
            keep &= item_sets[set_ix[j], items] == 0
        items, score = items[keep], score[keep]
        order = np.lexsort((items, -score))[:topk]
        k = order.shape[0]
        oi[j, :k], os_[j, :k], oc[j] = items[order], score[order], k
    return oi, os_, oc


def expansion(top_n, ql):
    """A query's listed expansion: top_n summed over its listed ids in the item range, a repeated id counted each time."""
    ql = np.asarray(ql, np.int64).reshape(-1)
    ql = ql[(ql >= 0) & (ql < top_n.shape[0])]
    return int(top_n[ql].astype(np.int64).sum())


def parts(top_n, q_lists, budget):
    """The first query of each part: a part closes before the query that would take its listed expansion over the
    budget (capped at 2^32 - 1) or its listed ids to 2^31; every part holds at least one query.  ValueError for a query
    that expands to 2^32 entries or more."""
    budget = min(budget, SCAN_LIMIT - 1)
    first, acc, acc_ids = [], 0, 0
    for j, ql in enumerate(q_lists):
        ex, ids = expansion(top_n, ql), len(ql)
        if ex >= SCAN_LIMIT or ids >= IDS_LIMIT:
            raise ValueError(f"query {j} is too large")
        if j == 0 or acc + ex > budget or acc_ids + ids >= IDS_LIMIT:
            first.append(j)
            acc = acc_ids = 0
        acc += ex
        acc_ids += ids
    return first
