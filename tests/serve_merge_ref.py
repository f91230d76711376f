"""Plain-Python restatement of pio_serve_zscore_merge: the similarproduct template's Serving.serve (z-score each
algorithm's list, sum per item, top num) over a batch given as arrays, and the split of a batch into parts.

Per algorithm a: items[a] int32 [Q, w_a] and scores[a] float64 [Q, w_a], of which the first count[a][j] entries of row j
are query j's list; num[j] >= 1 is query j's num.  All arithmetic is Python float (IEEE binary64, round to nearest), in
the association numpy and Serving.serve use, so the GPU tests compare with it bit for bit."""
import math

import numpy as np

PW_BLOCK = 128          # numpy's PW_BLOCKSIZE: pairwise_sum sums at most this many values without splitting
SCAN_LIMIT = 1 << 32    # a query with this many entries or more is rejected


def pairwise(v, lo, n):
    """numpy's pairwise_sum of v[lo:lo + n] (a list of floats): a plain loop from 0.0 below 8 values; eight accumulators
    over the first n - n % 8 values, combined ((r0 + r1) + (r2 + r3)) + ((r4 + r5) + (r6 + r7)), then the rest in order,
    up to PW_BLOCK values; above that the sums of the two halves, split at n // 2 rounded down to a multiple of 8."""
    if n < 8:
        res = 0.0
        for i in range(lo, lo + n):
            res += v[i]
        return res
    if n <= PW_BLOCK:
        r = v[lo:lo + 8]
        i = 8
        while i < n - n % 8:
            for k in range(8):
                r[k] += v[lo + i + k]
            i += 8
        res = ((r[0] + r[1]) + (r[2] + r[3])) + ((r[4] + r[5]) + (r[6] + r[7]))
        for t in range(i, n):
            res += v[lo + t]
        return res
    n2 = n // 2
    n2 -= n2 % 8
    return pairwise(v, lo, n2) + pairwise(v, lo + n2, n - n2)


def add_reduce(v):
    """np.add.reduce of a float64 vector: 0.0 + pairwise_sum."""
    v = [float(x) for x in v]
    return 0.0 + pairwise(v, 0, len(v))


def standardise(s, num):
    """One algorithm's list of scores as Serving.serve uses it: unchanged when num == 1, else z-scored with numpy's mean
    and sample standard deviation (0 when the list has fewer than two entries), and 0.0 wherever that deviation is 0."""
    s = [float(x) for x in s]
    if num == 1:
        return s
    n = len(s)
    mean = add_reduce(s) / n if n else 0.0
    sd = math.sqrt(add_reduce([(x - mean) * (x - mean) for x in s]) / (n - 1)) if n > 1 else 0.0
    return [0.0 if sd == 0 else (x - mean) / sd for x in s]


def merge_one(lists, num):
    """lists: per algorithm, a list of (item, score) pairs.  The served (item, score) pairs: each list standardised, the
    values summed per item as 0.0 + z0 + z1 + ... in algorithm then list order, ordered by sum descending with ties in
    order of first appearance, cut at num."""
    comb = {}
    for lst in lists:
        z = standardise([s for _, s in lst], num)
        for (it, _), v in zip(lst, z):
            comb[it] = comb.get(it, 0.0) + v
    return sorted(comb.items(), key=lambda kv: -kv[1])[:max(num, 0)]


def merge(items, scores, counts, num, topk):
    """(items int32 [Q, topk], scores float64 [Q, topk], count int32 [Q]) of the batch, padded with -1 / 0; query j keeps
    min(num[j], topk) results."""
    Q = len(num)
    oi = np.full((Q, topk), -1, np.int32)
    os_ = np.zeros((Q, topk), np.float64)
    oc = np.zeros(Q, np.int32)
    for j in range(Q):
        lists = [list(zip(items[a][j, :counts[a][j]].tolist(), scores[a][j, :counts[a][j]].tolist()))
                 for a in range(len(items))]
        top = merge_one(lists, int(num[j]))[:topk]
        oc[j] = len(top)
        for t, (it, v) in enumerate(top):
            oi[j, t], os_[j, t] = it, v
    return oi, os_, oc


def parts(counts, budget):
    """The first query of each part: a part closes before the query that would take its entries (the sum of its counts
    over the algorithms) over the budget, capped at 2^32 - 1; every part holds at least one query."""
    budget = min(budget, SCAN_LIMIT - 1)
    ent = np.sum([np.asarray(c, np.int64) for c in counts], axis=0)
    first, acc = [], 0
    for j, e in enumerate(ent.tolist()):
        if j == 0 or acc + e > budget:
            first.append(j)
            acc = 0
        acc += e
    return first
