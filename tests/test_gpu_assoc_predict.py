"""GPU tests (-m gpu) of pio_assoc_predict and the complementary purchase template's batch predict: the device's conds
equal the restatement (tests/assoc_predict_ref.py) exactly -- the same conds in the same order, the same items, first
rules and rule counts -- at its boundaries (empty batch, queries and model; unknown and repeated ids; cond sizes at
max_cond_len and past the model's levels; a deep and wide trie; long queries; budgets down to one query per part; a
rejected call followed by a good one), and the template's predictMany and BatchPredict equal predict byte for byte."""
import json
import pickle
from math import comb

import numpy as np
import pytest

import assoc_predict_ref as apr
import assoc_ref as ref
from pio_b200 import storage as s
from pio_b200 import workflow as w

pytestmark = pytest.mark.gpu

P = dict(basketWindow=120, maxRuleLength=4, minSupport=0.0, minConfidence=0.0, minLift=0.0, minBasketSize=2,
         maxNumRulesPerCond=3)


def _csr(queries):
    ptr = np.zeros(len(queries) + 1, np.int64)
    ptr[1:] = np.cumsum([len(q) for q in queries])
    flat = np.array([i for q in queries for i in q], np.int32)
    return ptr, flat


def _index(native, model, n_items):
    return native.AssocIndex(model["level_off"], model["set_prefix"], model["set_item"], model["rule_cond"], n_items)


def check(native, ix, model, n_items, queries, num, max_cond_len):
    """The device result equals the restatement's arrays."""
    ptr, flat = _csr(queries)
    got = ix.predict(ptr, flat, np.asarray(num, np.int32), max_cond_len)
    want = apr.predict(model, n_items, queries, list(num), max_cond_len)
    for g, x, name in zip(got, want, ("q_cond_ptr", "cond_ptr", "cond_items", "rule_first", "rule_n")):
        assert g.tolist() == list(x), name
    return got


def _hand_built(width, depth, n_rules=4):
    items = list(range(width))
    freq = {frozenset(c): 100 for k in range(1, depth + 1) for c in ref.combinations(items, k)}
    rules = {}
    for S in freq:
        for c in sorted(S) if len(S) > 1 else ():
            rules.setdefault(S - {c}, []).append((c, 0.25, 0.5, 1.0 + c))
    for cond in rules:
        rules[cond] = sorted(rules[cond], key=lambda r: (-r[3], r[0]))[:n_rules]
    return ref.flat(200, freq, rules)


def _trained(seed, length, n_items=40, n_events=4000):
    rng = np.random.default_rng(seed)
    t = np.cumsum(rng.integers(0, 6_000, n_events))
    ev = [(int(rng.integers(0, 50)), int(rng.zipf(1.4)) % n_items, int(x)) for x in t]
    return ref.flat(*ref.train(ev, **{**P, "maxRuleLength": length, "minSupport": 0.002}))


def _queries(seed, n_items, n=300, longest=12, unknown=5):
    rng = np.random.default_rng(seed)
    out = []
    for _ in range(n):
        q = [int(x) for x in rng.integers(-unknown, n_items + unknown, int(rng.integers(0, longest + 1)))]
        if len(q) > 1 and rng.random() < 0.5:
            q.insert(int(rng.integers(0, len(q))), q[int(rng.integers(0, len(q)))])
        out.append(q)
    return out


def test_empty_batch_queries_and_model(native):
    model = _hand_built(5, 3)
    ix = _index(native, model, 5)
    got = check(native, ix, model, 5, [], [], 3)
    assert got[0].tolist() == [0]
    check(native, ix, model, 5, [[], [], []], [1, 1, 1], 3)
    empty = ref.flat(0, {}, {})
    ex = _index(native, empty, 3)
    got = check(native, ex, empty, 3, [[0, 1, 2], [], [1]], [5, 5, 5], 4)
    assert got[0].tolist() == [0, 0, 0, 0] and got[1].tolist() == [0]
    check(native, ix, model, 5, [[0, 1, 2]], [3], 0)                           # max_cond_len 0: no conds


@pytest.mark.parametrize("length", [2, 3, 4, 5])
def test_trained_models_with_unknown_and_repeated_ids(native, length):
    model = _trained(length, length)
    ix = _index(native, model, 40)
    queries = _queries(length, 40)
    rng = np.random.default_rng(length)
    num = rng.choice([-3, -1, 0, 1, 2, 1000], len(queries)).tolist()
    check(native, ix, model, 40, queries, num, length - 1)
    check(native, ix, model, 40, queries, num, length + 3)                     # past the model's levels
    check(native, ix, model, 40, queries, num, 1)


@pytest.mark.parametrize("max_cond_len", [1, 2, 4, 5, 6, 9])
def test_deep_and_wide_trie(native, max_cond_len):
    model = _hand_built(12, 6)                                                  # 2509 sets, conds up to 5 items
    ix = _index(native, model, 16)
    queries = [list(range(16)), list(reversed(range(16))), [11, 3, 3, 7, 0, 15, 5, 9, 1, -2, 2],
               [4], [13, 14], _queries(1, 12, 1, 12)[0]]
    got = check(native, ix, model, 16, queries, [2] * len(queries), max_cond_len)
    k = min(max_cond_len, 5)
    assert got[0][1] == sum(comb(12, j) for j in range(1, k + 1))         # every cond inside the full query


def test_long_queries_against_the_restatement(native):
    rng = np.random.default_rng(7)
    n_items = 400
    t = np.cumsum(rng.integers(0, 3_000, 30_000))                              # a user's buys ~2 min apart
    ev = [(int(rng.integers(0, 60)), int(rng.zipf(1.2)) % n_items, int(x)) for x in t]
    model = ref.flat(*ref.train(ev, **{**P, "maxRuleLength": 4, "minSupport": 0.001}))
    assert np.diff(model["level_off"]).min() > 100                             # four well-filled levels
    ix = _index(native, model, n_items)
    queries = [[int(x) for x in rng.integers(-25, n_items + 25, L)] for L in (1000, 1500, 2500)]
    queries.append(queries[0] + queries[0][::-1])                              # every id repeated
    got = check(native, ix, model, n_items, queries, [3, 0, 1, 2], 3)
    assert got[0][1] > 1000 and np.diff(got[1]).max() == 3                    # conds of 1 .. 3 items


@pytest.mark.parametrize("budget", ["1", "40", "700", "100000000"])
def test_budgets_give_identical_results(native, monkeypatch, budget):
    model = _trained(3, 4)
    queries = _queries(9, 40, 200)
    num = [2] * len(queries)
    ptr, flat = _csr(queries)
    base = _index(native, model, 40).predict(ptr, flat, np.asarray(num, np.int32), 3)
    monkeypatch.setenv("PIO_ASSOC_PREDICT_BUDGET", budget)
    ix = _index(native, model, 40)
    got = check(native, ix, model, 40, queries, num, 3)
    for g, b in zip(got, base):
        assert g.tolist() == b.tolist()
    st = native.assoc_predict_stats()
    if budget == "1":
        assert st["parts"] == len(queries) and st["max_part_queries"] == 1
    assert st["parts"] == len(apr.plan(apr.Index(model, 40), queries, 3, int(budget))) - 1
    assert st["conds"] == len(got[3]) and st["entries"].get(1, 0) > 0


def test_rejections_leave_the_index_usable(native):
    model = _hand_built(6, 3)
    ix = _index(native, model, 6)
    check(native, ix, model, 6, [[0, 1, 2]], [1], 2)
    bad_ptr = np.array([0, 3, 2], np.int64)
    with pytest.raises(native.NativeError) as e:
        ix.predict(bad_ptr, np.array([0, 1, 2], np.int32), np.array([1, 1], np.int32), 2)
    assert e.value.code == native.ERR_ARG
    with pytest.raises(native.NativeError) as e:
        ix.predict(np.array([0, 1], np.int64), np.array([0], np.int32), np.array([1], np.int32), -1)
    assert e.value.code == native.ERR_ARG
    check(native, ix, model, 6, [[2, 1, 0, 5], [3, 3]], [2, 0], 2)              # the next call is unaffected
    # a bad trie is refused when the index is created
    broken = dict(model, set_item=list(model["set_item"]))
    broken["set_item"][1] = broken["set_item"][0]
    with pytest.raises(native.NativeError) as e:
        _index(native, broken, 6)
    assert e.value.code == native.ERR_ARG


# ---- the template ------------------------------------------------------------------------------------------------------
def _shop(seed, n_users=300, n_items=60):
    import datetime as dt
    rng = np.random.default_rng(seed)
    t0 = dt.datetime(2021, 1, 1, tzinfo=dt.timezone.utc)
    evs = []
    for usr in range(n_users):
        when = t0 + dt.timedelta(days=int(rng.integers(0, 30)))
        for _ in range(int(rng.integers(1, 5))):
            for _ in range(int(rng.integers(2, 7))):
                evs.append(dict(event="buy", entityType="user", entityId=f"u{usr}", targetEntityType="item",
                                targetEntityId=f"i{int(rng.zipf(1.3)) % n_items}", eventTime=when.isoformat()))
                when += dt.timedelta(seconds=int(rng.integers(0, 60)))
            when += dt.timedelta(days=int(rng.integers(1, 4)))
    return evs


def _string_queries(seed, n=400):
    rng = np.random.default_rng(seed)
    qs = []
    for _ in range(n):
        items = [f"i{int(rng.zipf(1.3)) % 70}" for _ in range(int(rng.integers(0, 9)))]
        if items and rng.random() < 0.3:
            items.append(items[0])
        qs.append({"items": items, "num": int(rng.choice([-1, 0, 1, 3, 10]))})
    return qs


def test_template_predict_many_pickle_and_batchpredict(native, tmp_path, monkeypatch):
    monkeypatch.setenv("PIO_EVENTDATA_DIR", str(tmp_path / "events"))
    monkeypatch.setenv("PIO_MODELDATA_DIR", str(tmp_path / "models"))
    from pio_b200.templates import complementarypurchase as cp
    s.import_events("CPP", _shop(3))
    params = {**P, "minSupport": 0.002}
    variant = tmp_path / "engine.json"
    variant.write_text(json.dumps({
        "id": "default", "engineFactory": "pio_b200.templates.complementarypurchase.ComplementaryPurchaseEngine",
        "datasource": {"params": {"appName": "CPP"}}, "algorithms": [{"name": "algo", "params": params}]}))
    inst = w.CreateWorkflow.main(["--engine-id", "cpp", "--engine-version", "1", "--engine-variant", f"file:{variant}"])
    server = w.deploy(inst.id)
    algo, model = server.algorithms[0], server.models[0]
    assert len(model.level_off) - 1 >= 3 and w.BatchPredict.columnar(server)
    queries = _string_queries(5)
    qobjs = [cp.Query(**q) for q in queries]
    want = [algo.predict(model, q) for q in qobjs]
    assert algo.predictMany(model, qobjs) == want
    assert sum(len(r.rules) for r in want) > len(queries)
    # the pickle holds no device index; a model pickled before the index existed (no `device`) loads and serves
    m2 = pickle.loads(pickle.dumps(model))
    assert "_index" not in m2.__dict__ and m2.device == model.device
    old = pickle.loads(pickle.dumps(model))
    del old.__dict__["device"]
    old = pickle.loads(pickle.dumps(old))
    assert not hasattr(old, "device")
    assert algo.predictMany(old, qobjs) == want and algo.predictMany(m2, qobjs) == want
    # BatchPredict: the column path's bytes equal a predict-then-serve loop's
    (tmp_path / "in.json").write_text("\n".join(json.dumps(q) for q in queries) + "\n")
    out = tmp_path / "out.json"
    assert w.BatchPredict.main(["--input", str(tmp_path / "in.json"), "--output", str(out), "--query-chunk", "97",
                                "--engine-instance-id", inst.id]) == len(queries)
    lines = [json.dumps({"query": w.to_json(q), "prediction": w.to_json(server.serving.serve(q, [p]))},
                        separators=(",", ":")) for q, p in zip(qobjs, want)]
    assert out.read_text().splitlines() == lines
