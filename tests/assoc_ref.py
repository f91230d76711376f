"""Plain-Python statement of the complementary purchase template's training and predict
(docs/manual/source/templates/complementarypurchase/dase.html.md.erb; the doc elides how transactions, counts and rules
are built, lines 293-314, and the reference has no source file for this template, so this file is the spec the device
matches).  Parity with the Spark template is not pinned: where it leaves an order open, the rule here is this project's.

Events are (user, item, t): user and item indices (the item index is BiMap.stringInt of the buy events' item ids in
order of first occurrence), t = eventTime.getMillis = floor(time_us / 1000).

    transactions   per user, buys by t; a new basket at the first buy and at every gap > basketWindow * 1000 ms (a
                   gap equal to the window stays; each buy extends the basket); a basket is the SET of its items;
                   baskets with fewer than minBasketSize items are dropped; T = how many are kept
    item sets      every subset of size 1 .. maxRuleLength of every kept basket, counted; frequent when
                   count >= minSupport * T (fp64, minSupport * T as a double)
    rules          every frequent S, |S| >= 2, and c in S: cond = S - {c}, support = count(S) / T, confidence =
                   count(S) / count(cond), lift = confidence / (count({c}) / T), in fp64 in this order; kept when
                   confidence >= minConfidence and lift >= minLift
    ranking        per cond: lift descending, then the conseq's item index ascending; the first maxNumRulesPerCond
    predict        the query's items de-duplicated (first occurrence kept); conds = their subsets of size 1 ..
                   maxRuleLength - 1, by size, then in lexicographic order of positions in the query; for every cond
                   the model has, Rule(cond in query order, its first `num` rules)
"""
from itertools import combinations
from typing import Dict, FrozenSet, List, Sequence, Tuple

Rule = Tuple[int, float, float, float]   # (conseq, support, confidence, lift)


def check_params(basketWindow, maxRuleLength, minSupport, minConfidence, minLift, minBasketSize, maxNumRulesPerCond):
    """The parameter checks: ValueError before any work."""
    if maxRuleLength < 2:
        raise ValueError(f"maxRuleLength must be at least 2 (got {maxRuleLength})")
    if minBasketSize < 2:
        raise ValueError(f"minBasketSize must be at least 2 (got {minBasketSize})")
    if not 0.0 <= minSupport <= 1.0:
        raise ValueError(f"minSupport must be in [0, 1] (got {minSupport})")
    if not 0.0 <= minConfidence <= 1.0:
        raise ValueError(f"minConfidence must be in [0, 1] (got {minConfidence})")
    if maxNumRulesPerCond < 1:
        raise ValueError(f"maxNumRulesPerCond must be at least 1 (got {maxNumRulesPerCond})")


def millis(time_us: int) -> int:
    """Joda's getMillis of a microsecond time: floor toward -inf."""
    return time_us // 1000


def transactions(events: Sequence[Tuple[int, int, int]], basketWindow: int, minBasketSize: int) -> List[FrozenSet[int]]:
    """The kept baskets, as item sets, in (user, first buy) order."""
    by_user: Dict[int, List[Tuple[int, int]]] = {}
    for u, i, t in events:
        by_user.setdefault(u, []).append((t, i))
    window = basketWindow * 1000
    out = []
    for u in sorted(by_user):
        buys = sorted(by_user[u], key=lambda ti: ti[0])   # ties in t do not change the baskets
        baskets, last = [], None
        for t, i in buys:
            if last is None or t - last > window:
                baskets.append(set())
            baskets[-1].add(i)
            last = t
        out.extend(frozenset(b) for b in baskets if len(b) >= minBasketSize)
    return out


def train(events, basketWindow, maxRuleLength, minSupport, minConfidence, minLift, minBasketSize, maxNumRulesPerCond):
    """(T, frequent sets {frozenset: count}, rules {cond frozenset: [Rule, ...] ranked and cut})."""
    check_params(basketWindow, maxRuleLength, minSupport, minConfidence, minLift, minBasketSize, maxNumRulesPerCond)
    trans = transactions(events, basketWindow, minBasketSize)
    T = len(trans)
    counts: Dict[FrozenSet[int], int] = {}
    for b in trans:
        items = sorted(b)
        for n in range(1, maxRuleLength + 1):
            for s in combinations(items, n):
                fs = frozenset(s)
                counts[fs] = counts.get(fs, 0) + 1
    thr = minSupport * T
    freq = {s: c for s, c in counts.items() if c >= thr}
    rules: Dict[FrozenSet[int], List[Rule]] = {}
    for s, cs in freq.items():
        if len(s) < 2:
            continue
        for c in s:
            cond = s - {c}
            support = cs / T
            confidence = cs / freq[cond]
            lift = confidence / (freq[frozenset([c])] / T)
            if confidence >= minConfidence and lift >= minLift:
                rules.setdefault(cond, []).append((c, support, confidence, lift))
    for cond in rules:
        rules[cond] = sorted(rules[cond], key=lambda r: (-r[3], r[0]))[:maxNumRulesPerCond]
    return T, freq, rules


def query_conds(items: Sequence, maxRuleLength: int) -> List[Tuple]:
    """The conds of a query, each a tuple of its items in query order."""
    seen = list(dict.fromkeys(items))
    return [c for n in range(1, maxRuleLength) for c in combinations(seen, n)]


def predict(rules: Dict[FrozenSet, List[Rule]], items: Sequence, num: int, maxRuleLength: int,
            name=lambda i: i, index=lambda x: x) -> dict:
    """The JSON of PredictedResult: {"rules": [{"cond": [...], "itemScores": [{"item", "support", "confidence",
    "lift"}]}]}.  `index` maps a query item to the model's key (None: unknown), `name` an item index to its id."""
    out = []
    for cond in query_conds(items, maxRuleLength):
        keys = [index(x) for x in cond]
        if any(k is None for k in keys):
            continue
        vec = rules.get(frozenset(keys))
        if vec is None:
            continue
        out.append({"cond": list(cond), "itemScores": [
            {"item": name(c), "support": s, "confidence": cf, "lift": lf} for c, s, cf, lf in vec[:max(num, 0)]]})
    return {"rules": out}


def index_events(buys: Sequence[Tuple[str, str, int]]):
    """(events as (user index, item index, t), item ids by index) of (user, item, t) string events: both numbered in
    order of first occurrence."""
    users: Dict[str, int] = {}
    items: Dict[str, int] = {}
    ev = []
    for u, i, t in buys:
        ev.append((users.setdefault(u, len(users)), items.setdefault(i, len(items)), t))
    return ev, list(items)


def flat(T, freq, rules, maxRuleLength=None) -> dict:
    """The model in the flat layout of native.assoc_train: sets by length then lexicographic order of their sorted
    items, each as (index of its prefix, largest item, count); rules grouped by cond in set order."""
    order = sorted(freq, key=lambda s: (len(s), sorted(s)))
    ix = {s: k for k, s in enumerate(order)}
    levels = max((len(s) for s in order), default=0)
    level_off = [0] * (levels + 1)
    for s in order:
        level_off[len(s)] += 1
    for l in range(1, levels + 1):
        level_off[l] += level_off[l - 1]
    out = {"level_off": level_off, "set_prefix": [], "set_item": [], "set_count": [], "rule_cond": [],
           "rule_conseq": [], "support": [], "confidence": [], "lift": [], "n_transactions": T}
    for s in order:
        it = sorted(s)
        out["set_prefix"].append(ix[frozenset(it[:-1])] if len(it) > 1 else -1)
        out["set_item"].append(it[-1])
        out["set_count"].append(freq[s])
    for cond in sorted(rules, key=lambda s: ix[s]):
        for c, sup, cf, lf in rules[cond]:
            out["rule_cond"].append(ix[cond])
            out["rule_conseq"].append(c)
            out["support"].append(sup)
            out["confidence"].append(cf)
            out["lift"].append(lf)
    return out
