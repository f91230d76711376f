"""Plain-Python restatement of the complementary purchase template's batch predict on the GPU (pio_assoc_predict,
csrc/assoc_predict.cuh, DESIGN.md 4.15.1).  The rules it restates are those of Algorithm.predict and assoc_ref.predict:

    query      its item ids; an id outside [0, n_items) is unknown; a repeated id keeps its first position
    conds      the subsets of size 1 .. maxRuleLength - 1 of the de-duplicated query, by size, then in lexicographic
               order of query positions; a subset holding an unknown item is skipped.  Skipping those subsets is the
               same as enumerating only over the known items, kept in query order: the subsets of a subsequence are
               exactly the subsets without the dropped items, and lexicographic order of positions is kept when
               positions are dropped (query_conds_known)
    rules      each cond the model has rules for gives (cond in query order, its first max(num, 0) rules); with
               num <= 0 the cond is still listed, with no rules

The device finds the conds without enumerating subsets.  The model's frequent sets form a prefix trie (set s = its
prefix set plus its largest item), and a cond with rules is a frequent set, so walking the trie over the query's
frequent items finds exactly the frequent sets inside the query (walk):
    L          the query's distinct frequent items sorted by item, each with its first position
    level 1    (level-1 set of L[u], u) for every u
    level k    every found (k-1)-set s at u extended by each trie child of s whose item is in L after u
    output     every found set with rules, its positions rebuilt from the prefix chain, ordered per level by (query,
               positions ascending)
A batch runs in parts of consecutive queries within a budget of entries (listed ids plus a bound on the sets found);
the result does not depend on the parts (plan).
"""
from itertools import combinations
from typing import Dict, List, Sequence, Tuple

Arrays = Tuple[List[int], List[int], List[int], List[int], List[int]]   # q_cond_ptr, cond_ptr, cond_items, first, n


def query_conds_known(items: Sequence, maxRuleLength: int, known) -> List[Tuple]:
    """assoc_ref.query_conds without the conds holding an unknown item, enumerated over the known items only."""
    seen = [x for x in dict.fromkeys(items) if known(x)]
    return [c for n in range(1, maxRuleLength) for c in combinations(seen, n)]


class Index:
    """The trie of a model in the flat layout of native.assoc_train / assoc_ref.flat, with what the device derives:
    each set's children and rule range, each item's level-1 set."""

    def __init__(self, model: dict, n_items: int):
        self.n_items = n_items
        self.level_off = [int(x) for x in model["level_off"]]
        self.n_levels = len(self.level_off) - 1
        self.prefix = [int(x) for x in model["set_prefix"]]
        self.item = [int(x) for x in model["set_item"]]
        self.children: Dict[int, List[int]] = {}
        for s, p in enumerate(self.prefix):
            if p >= 0:
                self.children.setdefault(p, []).append(s)
        self.rules: Dict[int, Tuple[int, int]] = {}
        for r, c in enumerate(int(x) for x in model["rule_cond"]):
            lo, _ = self.rules.get(c, (r, r))
            self.rules[c] = (lo, r + 1)
        self.item_set = {self.item[s]: s for s in range(self.level_off[1] if self.n_levels else 0)}

    def bound(self, f: int, K: int) -> int:
        """The most sets a query with f listed frequent ids can find: sum over k <= K of min(C(f, k), sets of level k)."""
        b, c = 0, 1
        for k in range(1, min(K, self.n_levels) + 1):
            c = c * max(f - k + 1, 0) // k
            b += min(c, self.level_off[k] - self.level_off[k - 1])
        return b


def walk(ix: Index, items: Sequence[int], num: int, K: int) -> List[Tuple[List[int], int, int]]:
    """One query's conds as (items in query order, first rule, rule count), in the contract's order."""
    first: Dict[int, int] = {}
    for p, it in enumerate(items):
        if 0 <= it < ix.n_items and it in ix.item_set and it not in first:
            first[it] = p
    L = sorted(first)                                   # items ascending
    front = [(ix.item_set[it], u) for u, it in enumerate(L)]
    out = []
    for k in range(1, K + 1):
        if not front:
            break
        level = []
        for s, u in front:
            if s in ix.rules:
                chain, t = [], s
                while t >= 0:
                    chain.append(first[ix.item[t]])
                    t = ix.prefix[t]
                pos = sorted(chain)
                lo, hi = ix.rules[s]
                level.append((pos, [items[p] for p in pos], lo, min(hi - lo, max(num, 0))))
        out.extend((its, lo, n) for _, its, lo, n in sorted(level, key=lambda e: e[0]))
        later = {it: u for u, it in enumerate(L)}
        front = [(c, later[ix.item[c]]) for s, u in front for c in ix.children.get(s, [])
                 if ix.item[c] in later and later[ix.item[c]] > u]
    return out


def plan(ix: Index, queries: Sequence[Sequence[int]], K: int, budget: int) -> List[int]:
    """The first query of every part, then len(queries): a part closes before the query that would take its entries
    over the budget; each part holds at least one query."""
    first, acc = [], 0
    for j, q in enumerate(queries):
        f = sum(1 for it in q if 0 <= it < ix.n_items and it in ix.item_set)
        w = len(q) + ix.bound(f, K)
        if j == 0 or acc + w > budget:
            first.append(j)
            acc = 0
        acc += w
    return first + [len(queries)]


def predict(model: dict, n_items: int, queries: Sequence[Sequence[int]], num: Sequence[int], max_cond_len: int,
            budget: int = 1 << 24) -> Arrays:
    """pio_assoc_predict's result arrays for a batch; the queries are walked part by part."""
    ix = Index(model, n_items)
    K = min(max_cond_len, ix.n_levels)
    qp, cp, ci, rf, rn = [0], [0], [], [], []
    bounds = plan(ix, queries, K, budget)
    for p in range(len(bounds) - 1):
        for j in range(bounds[p], bounds[p + 1]):
            for its, lo, n in walk(ix, queries[j], num[j], K):
                ci.extend(its)
                cp.append(len(ci))
                rf.append(lo)
                rn.append(n)
            qp.append(len(rf))
    return qp, cp, ci, rf, rn


def to_json(arrays: Arrays, model: dict, name=lambda i: i) -> List[dict]:
    """The JSON of every query's PredictedResult, as assoc_ref.predict writes it."""
    qp, cp, ci, rf, rn = arrays
    out = []
    for j in range(len(qp) - 1):
        rules = []
        for c in range(qp[j], qp[j + 1]):
            rules.append({"cond": [name(i) for i in ci[cp[c]:cp[c + 1]]], "itemScores": [
                {"item": name(int(model["rule_conseq"][r])), "support": float(model["support"][r]),
                 "confidence": float(model["confidence"][r]), "lift": float(model["lift"][r])}
                for r in range(rf[c], rf[c] + rn[c])]})
        out.append({"rules": rules})
    return out
