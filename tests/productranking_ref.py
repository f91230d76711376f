"""The product ranking template's predict, restated on the CPU (docs/manual/source/templates/productranking/
dase.html.md.erb:471-530), and the plan of a pio_als_rank_lists call (csrc/rank_plan.h).

predict_literal transcribes the Scala predict for one query: the user's factor, each entry's Option[Double] score
(dotProduct: an fp64 sum in index order from 0 over the float factors widened to double), isOriginal when the user has
no factor or no entry has a score, and otherwise List.sorted(Ordering.by(_.score).reverse) -- a stable sort whose
comparison is java.lang.Double.compare, reversed.  rank_lists is the same rule vectorised over a batch, in the output
layout of pio_als_rank_lists.  A NaN score is returned as Java's canonical NaN (Double.doubleToLongBits)."""
from functools import cmp_to_key

import numpy as np

TILE = 2048                       # rank_plan.h RL_TILE
BUDGET = 1 << 24                  # PIO_RANK_LISTS_BUDGET
CANON_NAN = np.array([0x7FF8000000000000], np.uint64).view(np.float64)[0]
_SIGN = np.uint64(1 << 63)


def _bits(x: float) -> int:
    """Double.doubleToLongBits: the signed 64-bit pattern, every NaN folded to the canonical one."""
    if x != x:
        return 0x7FF8000000000000
    b = int(np.array([x], np.float64).view(np.int64)[0])
    return b


def double_compare(a: float, b: float) -> int:
    """java.lang.Double.compare."""
    if a < b:
        return -1
    if a > b:
        return 1
    ba, bb = _bits(a), _bits(b)
    return 0 if ba == bb else (-1 if ba < bb else 1)


def _canon(x: float) -> float:
    return float(CANON_NAN) if x != x else x


def _dot(f, g) -> float:
    d = 0.0
    for t in range(len(f)):
        d += float(f[t]) * float(g[t])
    return d


def predict_literal(user_f, user_has, item_f, item_has, user: int, items):
    """One query, as the Scala predict computes it: (positions, scores, isOriginal) -- positions[r] is the index in
    `items` of the r-th result."""
    items = [int(i) for i in items]
    not_ranked = (list(range(len(items))), [0.0] * len(items), True)
    if not (0 <= user < user_f.shape[0]) or not user_has[user]:
        return not_ranked
    uf = np.asarray(user_f[user], np.float32)
    scores = []
    for i in items:
        if 0 <= i < item_f.shape[0] and item_has[i]:
            scores.append(_dot(np.asarray(item_f[i], np.float32), uf))
        else:
            scores.append(None)
    if all(s is None for s in scores):
        return not_ranked
    entries = [(r, 0.0 if s is None else s) for r, s in enumerate(scores)]
    ranked = sorted(entries, key=cmp_to_key(lambda a, b: -double_compare(a[1], b[1])))   # stable
    return [r for r, _ in ranked], [_canon(s) for _, s in ranked], False


def order_key(scores) -> np.ndarray:
    """uint64 keys whose ascending order is Double.compare descending: NaN (any) first, +inf ... +0.0, -0.0, the
    negatives, -inf last."""
    s = np.asarray(scores, np.float64)
    b = np.where(np.isnan(s), CANON_NAN, s).view(np.uint64)
    return np.where((b & _SIGN) != 0, b, ~(b | _SIGN))


def rank_lists(user_f, user_has, item_f, item_has, users, list_ptr, items, chunk=1 << 16):
    """pio_als_rank_lists: (pos int32 [total], scores float64 [total], ranked bool [n])."""
    users = np.asarray(users, np.int64)
    ptr = np.asarray(list_ptr, np.int64)
    items = np.asarray(items, np.int64)[:ptr[-1]]
    n, total = users.shape[0], int(ptr[-1])
    user_has = np.ones(user_f.shape[0], bool) if user_has is None else np.asarray(user_has).astype(bool)
    item_has = np.ones(item_f.shape[0], bool) if item_has is None else np.asarray(item_has).astype(bool)
    uok = (users >= 0) & (users < user_f.shape[0])
    uok[uok] &= user_has[users[uok]]
    q_of = np.repeat(np.arange(n), np.diff(ptr))
    iok = (items >= 0) & (items < item_f.shape[0])
    iok[iok] &= item_has[items[iok]]
    has = iok & uok[q_of]
    scores = np.zeros(total)
    idx = np.flatnonzero(has)
    for a in range(0, idx.shape[0], chunk):
        e = idx[a:a + chunk]
        x = np.asarray(user_f, np.float32)[users[q_of[e]]].astype(np.float64)
        y = np.asarray(item_f, np.float32)[items[e]].astype(np.float64)
        acc = np.zeros(e.shape[0])
        with np.errstate(invalid="ignore", over="ignore"):   # inf * 0 and inf - inf are NaN, as on the device
            for t in range(y.shape[1]):
                acc += y[:, t] * x[:, t]
        scores[e] = acc
    scores[np.isnan(scores)] = CANON_NAN
    ranked = np.bincount(q_of[has], minlength=n) > 0
    order = np.lexsort((np.arange(total), order_key(scores), q_of))
    pos = (order - ptr[q_of]).astype(np.int32)
    return pos, scores[order], ranked


def plan(list_ptr, budget=BUDGET, tile=TILE):
    """rank_plan.h's plan_rank_lists: one dict per part (q0, q1, e0, e1, radix, tile_q, tile_ptr, tile_off, tile_n)."""
    ptr = [int(x) for x in list_ptr]
    parts, acc = [], 0
    for q in range(len(ptr) - 1):
        ln = ptr[q + 1] - ptr[q]
        if not parts or acc + ln > budget:
            parts.append(dict(q0=q, q1=q, e0=ptr[q], e1=ptr[q], radix=[], tile_q=[], tile_ptr=[0], tile_off=[],
                              tile_n=[]))
            acc = 0
        acc += ln
        p = parts[-1]
        p["q1"], p["e1"] = q + 1, ptr[q + 1]
        if ln > tile:
            p["radix"].append(q)
        elif ln > 0:
            if not p["tile_n"] or p["tile_n"][-1] + ln > tile:
                if p["tile_n"]:
                    p["tile_ptr"].append(len(p["tile_q"]))
                p["tile_n"].append(0)
            p["tile_q"].append(q)
            p["tile_off"].append(p["tile_n"][-1])
            p["tile_n"][-1] += ln
    for p in parts:
        if p["tile_n"]:
            p["tile_ptr"].append(len(p["tile_q"]))
    return parts
