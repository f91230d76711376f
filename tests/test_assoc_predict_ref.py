"""CPU checks of the batch predict restatement (tests/assoc_predict_ref.py): the trie walk with its per-level order and
parts equals assoc_ref.predict and the template's predict on trained and hand-built models, with repeats, unknown
items interleaved, every kind of num, maxRuleLength 2 .. 6, an empty model and empty queries."""
import numpy as np
import pytest

import assoc_predict_ref as apr
import assoc_ref as ref
from pio_b200 import storage as s
from pio_b200 import workflow as w
from pio_b200.templates import complementarypurchase as cp

PARAMS = dict(basketWindow=120, maxRuleLength=2, minSupport=0.0, minConfidence=0.0, minLift=0.0, minBasketSize=2,
              maxNumRulesPerCond=3)
NUMS = (-1, 0, 1, 2, 1000)


def _events(seed, n_users=30, n_items=14, n=600):
    rng = np.random.default_rng(seed)
    t = np.cumsum(rng.integers(0, 9_000, n))   # a user's buys ~4.5 min apart on average: baskets of a few items
    return [(int(rng.integers(0, n_users)), int(rng.zipf(1.5)) % n_items, int(x)) for x in t]


def _queries(seed, n_items, n=40, unknown=3):
    """Queries of 0 .. 9 ids with repeats and ids outside [0, n_items) interleaved."""
    rng = np.random.default_rng(seed)
    out = [[]]
    for _ in range(n):
        q = [int(x) for x in rng.integers(-unknown, n_items + unknown, int(rng.integers(1, 10)))]
        if q and rng.random() < 0.5:
            q.insert(int(rng.integers(0, len(q))), q[0])        # a repeat
        out.append(q)
    return out + [[], list(range(n_items)), list(reversed(range(n_items)))]


def _check(flat, rules, n_items, queries, length, budget=1 << 24):
    known = lambda x: x if 0 <= x < n_items else None      # noqa: E731
    for num in NUMS:
        got = apr.predict(flat, n_items, queries, [num] * len(queries), length - 1, budget)
        js = apr.to_json(got, flat)
        for q, g in zip(queries, js):
            assert g == ref.predict(rules, q, num, length, index=known), (q, num)
    return got


@pytest.mark.parametrize("length", [2, 3, 4, 5, 6])
def test_trained_models_equal_assoc_ref(length):
    ev = _events(length)
    T, freq, rules = ref.train(ev, **{**PARAMS, "maxRuleLength": length, "minSupport": 0.01})
    flat = ref.flat(T, freq, rules)
    assert len(flat["level_off"]) - 1 >= min(length, 3)          # the walk goes past level 2
    queries = _queries(length, 14)
    base = _check(flat, rules, 14, queries, length)
    for budget in (1, 7, 50):                                    # parts of one query and more: the same arrays
        assert apr.predict(flat, 14, queries, [1000] * len(queries), length - 1, budget) == base
    assert apr.plan(apr.Index(flat, 14), queries, length - 1, 1) == list(range(len(queries) + 1))


def _hand_built(width, depth):
    """Every subset of `width` items up to `depth` items frequent, rules for every cond, hand-set scores."""
    items = list(range(width))
    freq = {frozenset(c): 100 - len(c) for k in range(1, depth + 1) for c in ref.combinations(items, k)}
    rules = {}
    for S in freq:
        if len(S) < 2:
            continue
        for c in sorted(S):
            rules.setdefault(S - {c}, []).append((c, 0.5 / len(S), 1.0 / (1 + c), 1.0 + c / 8))
    for cond in rules:
        rules[cond] = sorted(rules[cond], key=lambda r: (-r[3], r[0]))[:4]
    return ref.flat(200, freq, rules), rules


@pytest.mark.parametrize("length", [2, 4, 6])
def test_hand_built_trie_equals_assoc_ref(length):
    flat, rules = _hand_built(7, 5)
    queries = [[6, 0, 3, 3, 9, 1], [5, 4, 3, 2, 1, 0, 6], [8, -1, 2], [0], []]
    _check(flat, rules, 10, queries, length)


def test_unknown_items_interleaved_are_the_known_subsequence():
    known = lambda x: isinstance(x, int) and 0 <= x < 5       # noqa: E731
    for items in ([7, 0, "x", 1, 0, 9, 2], ["a", "b"], [], [3, 3, 3]):
        for length in range(2, 6):
            full = [c for c in ref.query_conds(items, length) if all(known(x) for x in c)]
            assert full == apr.query_conds_known(items, length, known)


def test_empty_model_and_empty_queries():
    empty = ref.flat(0, {}, {})
    assert empty["level_off"] == [0]
    got = apr.predict(empty, 3, [[0, 1], [], [2, 2]], [5, 5, 5], 4)
    assert got == ([0, 0, 0, 0], [0], [], [], [])
    flat, rules = _hand_built(4, 3)
    assert apr.predict(flat, 4, [], [], 3) == ([0], [0], [], [], [])
    assert apr.predict(flat, 4, [[], []], [1, 1], 3) == ([0, 0, 0], [0], [], [], [])
    assert apr.predict(flat, 4, [[0, 1]], [1], 0) == ([0, 0], [0], [], [], [])   # max_cond_len 0: no conds


def test_template_predict_equals_restatement():
    """The template's predict (the definition) on string queries equals the restatement's arrays mapped to strings."""
    length = 4
    ev = _events(11)
    T, freq, rules = ref.train(ev, **{**PARAMS, "maxRuleLength": length, "minSupport": 0.01})
    flat = ref.flat(T, freq, rules)
    names = [f"i{k}" for k in range(14)]
    model = cp.Model(flat, s.BiMap({x: k for k, x in enumerate(names)}), length)
    algo = cp.Algorithm(cp.AlgorithmParams(**{**PARAMS, "maxRuleLength": length}))
    queries = _queries(5, 14)
    name = lambda i: names[i] if 0 <= i < 14 else f"unknown{i}"   # noqa: E731
    for num in NUMS:
        got = apr.to_json(apr.predict(flat, 14, queries, [num] * len(queries), length - 1), flat, name)
        for q, g in zip(queries, got):
            assert w.to_json(algo.predict(model, cp.Query([name(i) for i in q], num))) == g
