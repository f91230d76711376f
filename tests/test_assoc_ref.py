"""CPU checks of the complementary purchase restatement (tests/assoc_ref.py) and of the template's host code: the
doc's worked numbers, the basket window, minBasketSize and minSupport boundaries, the parameter checks, predict's cond
order, de-duplication and JSON shape, and the template's object path against the restatement."""
import pickle

import numpy as np
import pytest

import assoc_ref as ref
from pio_b200 import storage as s
from pio_b200 import workflow as w
from pio_b200.templates import complementarypurchase as cp

PARAMS = dict(basketWindow=120, maxRuleLength=2, minSupport=0.0, minConfidence=0.0, minLift=0.0, minBasketSize=2,
              maxNumRulesPerCond=5)


def _train(events, **kw):
    return ref.train(events, **{**PARAMS, **kw})


def _apart(baskets, user0=0):
    """Events of baskets (lists of items), each basket its own user, buys one second apart."""
    return [(user0 + b, i, k * 1000) for b, items in enumerate(baskets) for k, i in enumerate(items)]


def test_doc_confidence_example():
    # "if A appears in 30 transactions and the item set [A, B] appears in 20 transactions, then the rule "A implies B"
    # has confidence of 0.66" (dase.html.md.erb, minConfidence)
    A, B, C = 0, 1, 2
    baskets = [[A, B]] * 20 + [[A, C]] * 10 + [[B, C]] * 5
    T, freq, rules = _train(_apart(baskets))
    assert T == 35 and freq[frozenset([A])] == 30 and freq[frozenset([A, B])] == 20
    (ab,) = [r for r in rules[frozenset([A])] if r[0] == B]
    assert ab[2] == 20 / 30 == 0.6666666666666666
    assert ab[1] == 20 / 35 and ab[3] == (20 / 30) / (25 / 35)


def test_window_boundary_and_chaining():
    W = 120
    at = [(0, 1, 0), (0, 2, W * 1000)]                  # gap == window: one basket
    assert ref.transactions(at, W, 2) == [frozenset([1, 2])]
    over = [(0, 1, 0), (0, 2, W * 1000 + 1)]            # window + 1 ms: two baskets of one item
    assert ref.transactions(over, W, 2) == []
    assert ref.transactions(over, W, 1) == [frozenset([1]), frozenset([2])]
    chain = [(0, k, k * W * 1000) for k in range(5)]     # every gap == window: the basket chains
    assert ref.transactions(chain, W, 2) == [frozenset(range(5))]
    shuffled = [chain[k] for k in (3, 0, 4, 2, 1)]       # order of events does not matter
    assert ref.transactions(shuffled, W, 2) == [frozenset(range(5))]
    ties = [(0, 1, 5), (0, 2, 5), (0, 1, 5)]             # equal times, a repeat buy collapses
    assert ref.transactions(ties, W, 2) == [frozenset([1, 2])]
    zero = [(0, 1, 7), (0, 2, 7), (0, 3, 8)]             # basketWindow 0: only equal times share a basket
    assert ref.transactions(zero, 0, 1) == [frozenset([1, 2]), frozenset([3])]


def test_millis_before_1970():
    # Joda's getMillis floors: -1 us is -1 ms, -1500 us is -2 ms
    assert [ref.millis(x) for x in (-1, -999, -1000, -1001, -1500, 0, 999, 1000)] == [-1, -1, -1, -2, -2, 0, 0, 1]
    assert cp._millis(np.array([-1, -999, -1000, -1001, -1500, 0, 999, 1000])).tolist() == [-1, -1, -1, -2, -2, 0, 0, 1]
    # a window of 1 s across the epoch: -1000.5 ms -> -1001 ms, so the gap to 0 is 1001 > 1000
    us = [-1_000_500, 0]
    ev = [(0, k, ref.millis(t)) for k, t in enumerate(us)]
    assert ref.transactions(ev, 1, 1) == [frozenset([0]), frozenset([1])]
    us = [-999_500, 0]                                   # -999.5 ms -> -1000 ms: gap == window
    ev = [(0, k, ref.millis(t)) for k, t in enumerate(us)]
    assert ref.transactions(ev, 1, 2) == [frozenset([0, 1])]


def test_min_basket_size_and_support_threshold():
    baskets = [[0, 1], [0, 1, 2], [0, 1, 2, 3], [4]]
    T, freq, _ = _train(_apart(baskets), minBasketSize=3)
    assert T == 2 and frozenset([4]) not in freq and freq[frozenset([0, 1])] == 2
    T, freq, _ = _train(_apart(baskets), minBasketSize=2)
    assert T == 3
    # minSupport * T exactly equal to a count keeps the set: 0.5 * 4 == 2.0
    baskets = [[0, 1], [0, 1], [2, 3], [2, 5]]
    T, freq, _ = _train(_apart(baskets), minSupport=0.5)
    assert T == 4 and freq[frozenset([0, 1])] == 2 and freq[frozenset([2])] == 2 and frozenset([3]) not in freq
    # a threshold computed in fp64: 0.28 * 25 = 7.000000000000001 > 7, so a count of 7 is not frequent
    baskets = [[0, 1]] * 7 + [[2, 3]] * 18
    T, freq, _ = _train(_apart(baskets), minSupport=0.28)
    assert 0.28 * 25 > 7 and T == 25 and frozenset([0]) not in freq and freq[frozenset([2, 3])] == 18
    T, freq, _ = _train(_apart(baskets), minSupport=0.27)
    assert freq[frozenset([0, 1])] == 7


def test_ranking_and_cut():
    # cond {0}: conseqs 1, 2, 3 with lift ties between 2 and 3 -> by item index; maxNumRulesPerCond cuts
    baskets = [[0, 1], [0, 2], [0, 3], [1, 9], [2, 8], [3, 7], [0, 1]]
    T, freq, rules = _train(_apart(baskets), maxNumRulesPerCond=2)
    assert [r[0] for r in rules[frozenset([0])]] == [1, 2]
    r0 = _train(_apart(baskets))[2][frozenset([0])]
    assert [r[0] for r in r0] == [1, 2, 3] and r0[1][3] == r0[2][3] < r0[0][3]


def test_parameter_checks():
    bad = [dict(maxRuleLength=1), dict(minBasketSize=1), dict(minSupport=-0.1), dict(minSupport=1.5),
           dict(minSupport=float("nan")), dict(minConfidence=-1e-9), dict(minConfidence=1.0000001),
           dict(maxNumRulesPerCond=0)]
    for kw in bad:
        with pytest.raises(ValueError):
            _train([(0, 0, 0), (0, 1, 0)], **kw)
        with pytest.raises(ValueError):   # the template checks before any device work
            cp.check_params(cp.AlgorithmParams(**{**PARAMS, **kw}))
        with pytest.raises(ValueError):
            cp.Algorithm(cp.AlgorithmParams(**{**PARAMS, **kw})).train(None, cp.TrainingData(
                buyEvents=[cp.BuyEvent("u", "a", 0), cp.BuyEvent("u", "b", 0)]))
    cp.check_params(cp.AlgorithmParams(**{**PARAMS, "minSupport": 1.0, "minConfidence": 1.0}))


def test_query_conds_order_and_dedup():
    assert ref.query_conds(["a", "b", "a", "c"], 3) == [("a",), ("b",), ("c",), ("a", "b"), ("a", "c"), ("b", "c")]
    assert ref.query_conds(["c", "a"], 2) == [("c",), ("a",)]


def _model(buys, **kw):
    p = {**PARAMS, **kw}
    ev, names = ref.index_events(buys)
    T, freq, rules = ref.train(ev, **p)
    imap = s.BiMap({x: k for k, x in enumerate(names)})
    return cp.Model(ref.flat(T, freq, rules), imap, p["maxRuleLength"]), rules, names


def _buys(seed, n_users=40, n_items=12, n=600):
    rng = np.random.default_rng(seed)
    t = np.cumsum(rng.integers(0, 200_000, n))
    return [(f"u{rng.integers(0, n_users)}", f"i{int(rng.zipf(1.6)) % n_items}", int(x)) for x in t]


@pytest.mark.parametrize("length", [2, 3, 4])
def test_template_predict_equals_restatement(length):
    buys = _buys(length)
    model, rules, names = _model(buys, maxRuleLength=length, minSupport=0.01, minBasketSize=2)
    assert model.rules.keys() == rules.keys()
    algo = cp.Algorithm(cp.AlgorithmParams(**{**PARAMS, "maxRuleLength": length}))
    imap = model.itemStringIntMap
    queries = [["i1", "i2"], ["i2", "i1", "i2", "i3"], ["nope", "i1"], [], list(names[:5]), ["i0"]]
    for items in queries:
        for num in (0, 1, 3, 100):
            got = w.to_json(algo.predict(model, cp.Query(items, num)))
            want = ref.predict(rules, items, num, length, name=lambda i: names[i], index=imap.get)
            assert got == want
    # JSON shape of the quickstart
    res = w.to_json(algo.predict(model, cp.Query(["i1", "i2"], 3)))
    assert set(res) == {"rules"} and res["rules"]
    for r in res["rules"]:
        assert set(r) == {"cond", "itemScores"} and isinstance(r["cond"], list)
        for x in r["itemScores"]:
            assert set(x) == {"item", "support", "confidence", "lift"}
    # a pickle of the model is the model
    m2 = pickle.loads(pickle.dumps(model))
    assert "_rules" not in m2.__dict__
    assert w.to_json(algo.predict(m2, cp.Query(["i1", "i2"], 3))) == res


def test_object_path_arrays_equal_restatement():
    buys = _buys(7)
    td = cp.TrainingData(buyEvents=[cp.BuyEvent(u, i, t) for u, i, t in buys])
    u, i, t, n_users, imap = cp.Algorithm(cp.AlgorithmParams(**PARAMS))._arrays(td)
    ev, names = ref.index_events(buys)
    assert list(zip(u.tolist(), i.tolist(), t.tolist())) == ev
    assert [imap.inverse(k) for k in range(imap.size)] == names and n_users == len({b[0] for b in buys})
    with pytest.raises(ValueError):
        cp.Algorithm(cp.AlgorithmParams(**PARAMS))._arrays(cp.TrainingData(buyEvents=[cp.BuyEvent("u", None, 0)]))


def test_buy_events_from_columns():
    def col(strs):
        enc = [x.encode() for x in strs]
        off = np.zeros(len(enc) + 1, np.int64)
        off[1:] = np.cumsum([len(b) for b in enc])
        return np.frombuffer(b"".join(enc), np.uint8), off
    t_us = np.array([-1_500, 1_234_567, 0], np.int64)
    cols = s.EventColumns(np.zeros(3, np.int32), np.zeros(3), np.zeros(3, bool), t_us, col(["u1", "u2", "u1"]),
                          col(["a", "b", "c"]), np.ones(3, bool))
    td = cp.TrainingData(columns=cols)
    assert td.buyEvents == [cp.BuyEvent("u1", "a", -2), cp.BuyEvent("u2", "b", 1234), cp.BuyEvent("u1", "c", 0)]


def test_engine_factory_and_serving():
    eng = w.get_engine("pio_b200.templates.complementarypurchase.ComplementaryPurchaseEngine")
    ep = eng.jValueToEngineParams({"datasource": {"params": {"appName": "A"}},
                                   "algorithms": [{"name": "algo", "params": PARAMS}]})
    assert ep.algorithmParamsList[0][1] == cp.AlgorithmParams(**PARAMS)
    pr = cp.PredictedResult([])
    assert cp.Serving().serve(cp.Query(["a"], 1), [pr, cp.PredictedResult([cp.Rule(["a"], [])])]) is pr
