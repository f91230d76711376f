"""GPU tests (-m gpu) of pio_assoc_train and the complementary purchase template: the device model equals the
restatement (tests/assoc_ref.py) exactly -- the same frequent sets and counts, the same rules in the same order, and
support / confidence / lift equal as doubles -- at its parameter, tie, key-width and size boundaries, and end to end
from an event file through CreateWorkflow, deploy and BatchPredict."""
import datetime as dt
import json
from math import comb

import numpy as np
import pytest

import assoc_ref as ref
from pio_b200 import storage as s
from pio_b200 import workflow as w

pytestmark = pytest.mark.gpu

P = dict(basketWindow=120, maxRuleLength=2, minSupport=0.0, minConfidence=0.0, minLift=0.0, minBasketSize=2,
         maxNumRulesPerCond=5)


def _device(native, u, i, t, n_users, n_items, p):
    return native.assoc_train(u, i, t, n_users, n_items, p["basketWindow"], p["maxRuleLength"], p["minSupport"],
                              p["minConfidence"], p["minLift"], p["minBasketSize"], p["maxNumRulesPerCond"])


def check(native, u, i, t, n_users, n_items, **kw):
    """The device model of the events equals the restatement's, array for array (doubles with ==)."""
    p = {**P, **kw}
    u, i, t = (np.asarray(x, dt_) for x, dt_ in ((u, np.int32), (i, np.int32), (t, np.int64)))
    got = _device(native, u, i, t, n_users, n_items, p)
    want = ref.flat(*ref.train(list(zip(u.tolist(), i.tolist(), t.tolist())), **p))
    assert got["n_transactions"] == want["n_transactions"]
    for k in ("level_off", "set_prefix", "set_item", "set_count", "rule_cond", "rule_conseq"):
        assert got[k].tolist() == list(want[k]), k
    for k in ("support", "confidence", "lift"):
        assert got[k].tolist() == list(want[k]), k   # float == float: bit for bit (no NaN can occur)
    return got


def sessions(seed, n_users, n_items, n_sessions, per=(2, 6), a=1.3, gap_s=60):
    """Seeded buys: per session a user buys a few Zipf-popular items `gap_s` seconds apart; days between sessions."""
    rng = np.random.default_rng(seed)
    u, i, t = [], [], []
    clock = rng.integers(0, 10 ** 9, n_users).astype(np.int64) * 1000
    for _ in range(n_sessions):
        usr = int(rng.integers(0, n_users))
        k = int(rng.integers(per[0], per[1] + 1))
        for _ in range(k):
            u.append(usr)
            i.append(int(rng.zipf(a) - 1) % n_items)
            t.append(int(clock[usr]))
            clock[usr] += int(rng.integers(0, gap_s + 1)) * 1000
        clock[usr] += 86_400_000 * int(rng.integers(1, 5))
    perm = rng.permutation(len(u))
    return np.array(u)[perm], np.array(i)[perm], np.array(t)[perm]


@pytest.mark.parametrize("length", [2, 3, 4])
@pytest.mark.parametrize("min_support", [0.0, 0.002, 0.02])
def test_rule_lengths_and_supports(native, length, min_support):
    u, i, t = sessions(length, 300, 40, 2500)
    got = check(native, u, i, t, 300, 40, maxRuleLength=length, minSupport=min_support)
    assert got["rule_cond"].size > 0
    if min_support == 0.0:
        assert got["level_off"].size - 1 == length


@pytest.mark.parametrize("conf, lift", [(0.3, 1.0), (0.0, 1.5), (1.0, 0.0)])
def test_confidence_and_lift_filters(native, conf, lift):
    u, i, t = sessions(11, 200, 25, 2000)
    check(native, u, i, t, 200, 25, maxRuleLength=3, minSupport=0.005, minConfidence=conf, minLift=lift)


@pytest.mark.parametrize("per_cond", [1, 2, 1000])
def test_lift_ties_by_item_index_and_rule_cut(native, per_cond):
    # item 0 with each of 1 .. 6, equally often, so every rule of cond {0} ties on lift; the items are numbered so
    # that the tie order is not the order of first occurrence
    baskets = [[0, k] for k in (6, 3, 5, 1, 4, 2)] * 4 + [[k, 7] for k in range(1, 7)]
    u = [b for b, items in enumerate(baskets) for _ in items]
    i = [x for items in baskets for x in items]
    t = [k for items in baskets for k in range(len(items))]
    got = check(native, u, i, t, len(baskets), 8, maxNumRulesPerCond=per_cond)
    r0 = np.flatnonzero(got["rule_cond"] == 0)   # set 0 is {0}
    assert got["rule_conseq"][r0].tolist() == [1, 2, 3, 4, 5, 6][:per_cond]
    assert len(set(got["lift"][r0].tolist())) == 1


@pytest.mark.parametrize("n_items", [2, 3, 255, 256, 257, 65535, 65536, 65537, (1 << 20) + 1])
def test_item_counts_across_key_widths(native, n_items):
    u, i, t = sessions(n_items % 97, 150, 30, 1500)
    i = (n_items - 1 - i) % n_items        # ids at the top of the range
    check(native, u, i, t, 150, n_items, maxRuleLength=3, minSupport=0.003)


@pytest.mark.parametrize("n_baskets", [255, 256, 257, 4095, 4096, 4097])
def test_basket_counts_at_powers_of_two(native, n_baskets):
    rng = np.random.default_rng(n_baskets)
    size = rng.integers(1, 5, n_baskets)
    user = np.repeat(np.arange(n_baskets) // 3, size)          # three baskets per user, a day apart
    b = np.repeat(np.arange(n_baskets), size)
    t = (b % 3) * 86_400_000 + np.concatenate([np.arange(k) for k in size]) * 1000
    i = rng.integers(0, 20, size.sum())
    got = check(native, user, i, t, int(user.max()) + 1, 20, maxRuleLength=3)
    timing = native.assoc_train_timing()
    assert timing["baskets"] == n_baskets and timing["transactions"] == got["n_transactions"]


def test_one_user_with_a_thousand_item_basket(native):
    rng = np.random.default_rng(5)
    i = rng.permutation(1000)
    u = np.zeros(1000, np.int32)
    t = np.arange(1000) * 1000            # one second apart: one basket
    u2, i2, t2 = sessions(3, 50, 1000, 300)
    got = check(native, np.r_[u, u2 + 1], np.r_[i, i2], np.r_[t, t2 + 10 ** 12], 51, 1000, maxNumRulesPerCond=2000)
    assert got["rule_cond"].size >= 999 * 1000


def test_no_basket_survives(native):
    u, i, t = sessions(2, 40, 10, 100, per=(1, 3))
    got = check(native, u, i, t, 40, 10, minBasketSize=50)
    assert got["n_transactions"] == 0 and got["set_item"].size == 0 and got["rule_cond"].size == 0
    assert got["level_off"].tolist() == [0]
    got = _device(native, np.zeros(0, np.int32), np.zeros(0, np.int32), np.zeros(0, np.int64), 1, 1, P)
    assert got["n_transactions"] == 0 and got["level_off"].tolist() == [0]


def test_window_boundaries_and_times_before_1970(native):
    W = 120
    ms = [0, W * 1000, 2 * W * 1000 + 1, 2 * W * 1000 + 1, 3 * W * 1000 + 1]   # chain, split, tie, chain
    times = [-(10 ** 12) + x for x in ms] + [x - 60_000 for x in ms]              # before and across the epoch
    u = [0] * 5 + [1] * 5
    i = [0, 1, 2, 3, 4, 0, 1, 2, 3, 4]
    got = check(native, u, i, times, 2, 5, maxRuleLength=3, minBasketSize=2)
    assert got["n_transactions"] == 4
    for bw in (0, 1, -1):
        check(native, u, i, times, 2, 5, basketWindow=bw)


def test_candidate_limit_is_rejected_before_the_level_is_enumerated(native):
    # one basket of 64 items at minSupport 0: level k counts C(64, k) candidates, and C(64, 7) is over the limit
    m, length = 64, 7
    assert comb(m, length - 1) <= native.ASSOC_MAX_CANDIDATES < comb(m, length)
    u = np.zeros(m, np.int32)
    i = np.arange(m, dtype=np.int32)
    t = np.zeros(m, np.int64)
    p = {**P, "maxRuleLength": length}
    with pytest.raises(native.NativeError) as ei:
        _device(native, u, i, t, 1, m, p)
    assert ei.value.code == native.ERR_ARG
    assert "minSupport" in str(ei.value) and "maxRuleLength" in str(ei.value) and "basketWindow" in str(ei.value)
    timing = native.assoc_train_timing()
    assert timing["rejected_level"] == length and timing["levels_run"] == length - 2
    assert timing["candidates"] == {k: comb(m, k) for k in range(2, length + 1)}
    # the template raises ValueError; one level less trains
    from pio_b200.templates import complementarypurchase as cp
    td = cp.TrainingData(buyEvents=[cp.BuyEvent("u", f"i{k}", 0) for k in range(m)])
    with pytest.raises(ValueError):
        cp.Algorithm(cp.AlgorithmParams(**p)).train(w.WorkflowContext(), td)
    got = _device(native, u, i, t, 1, m, {**P, "maxRuleLength": 3, "maxNumRulesPerCond": 1})
    assert got["level_off"].tolist() == [0, m, m + comb(m, 2), m + comb(m, 2) + comb(m, 3)]


# ---- the template, end to end ---------------------------------------------------------------------------------------
DOC_PARAMS = {"basketWindow": 120, "maxRuleLength": 2, "minSupport": 0.1, "minConfidence": 0.6, "minLift": 1.0,
              "minBasketSize": 2, "maxNumRulesPerCond": 5}


def _shop_events(seed, n_users=120):
    """Seeded buys over a few items with strong pairs, sessions a minute apart within, days between."""
    rng = np.random.default_rng(seed)
    t0 = dt.datetime(2021, 1, 1, tzinfo=dt.timezone.utc)
    pairs = [("s2i1", "s2i2"), ("s2i1", "s2i3"), ("s2i4", "s2i5"), ("s2i6", "s2i7"), ("s2i2", "s2i3")]
    evs = []
    for usr in range(n_users):
        when = t0 + dt.timedelta(days=int(rng.integers(0, 30)), microseconds=int(rng.integers(0, 10 ** 6)))
        for _ in range(int(rng.integers(1, 5))):
            items = list(pairs[int(rng.integers(0, len(pairs)))])
            if rng.random() < 0.4:
                items.append(f"s2i{int(rng.integers(1, 10))}")
            for it in items:
                evs.append(dict(event="buy", entityType="user", entityId=f"u{usr}", targetEntityType="item",
                                targetEntityId=it, eventTime=when.isoformat()))
                when += dt.timedelta(seconds=int(rng.integers(0, 90)))
            when += dt.timedelta(days=int(rng.integers(1, 4)))
    evs += [dict(event="view", entityType="user", entityId="u0", targetEntityType="item", targetEntityId="s2i9",
                 eventTime=t0.isoformat())]   # not a buy
    return evs


def _restated(evs, params):
    buys = [(e["entityId"], e["targetEntityId"], ref.millis(s.time_us(s._parse_time(e["eventTime"]))))
            for e in evs if e["event"] == "buy"]
    ev, names = ref.index_events(buys)
    T, freq, rules = ref.train(ev, **params)
    return rules, names


def test_template_end_to_end(tmp_path, monkeypatch):
    monkeypatch.setenv("PIO_EVENTDATA_DIR", str(tmp_path / "events"))
    monkeypatch.setenv("PIO_MODELDATA_DIR", str(tmp_path / "models"))
    evs = _shop_events(4)
    s.import_events("CP", evs)
    variant = tmp_path / "engine.json"
    variant.write_text(json.dumps({
        "id": "default", "description": "Default settings",
        "engineFactory": "pio_b200.templates.complementarypurchase.ComplementaryPurchaseEngine",
        "datasource": {"params": {"appName": "CP"}},
        "algorithms": [{"name": "algo", "params": DOC_PARAMS}]}))
    inst = w.CreateWorkflow.main(["--engine-id", "cp", "--engine-version", "1", "--engine-variant", f"file:{variant}"])
    assert inst.status == "COMPLETED"
    rules, names = _restated(evs, DOC_PARAMS)
    assert rules
    index = {x: k for k, x in enumerate(names)}
    queries = [{"items": ["s2i4"], "num": 3}, {"items": ["s2i1", "s2i6", "s2i4", "s2i1"], "num": 3},
               {"items": ["s2i7", "s2i3", "nope"], "num": 1}, {"items": ["s2i1"], "num": 3}, {"items": [], "num": 3}]
    answers = []
    for reload in range(2):                   # the second deploy reloads the persisted model
        server = w.deploy(inst.id)
        for q in queries:
            res = server.query(q)
            assert res == ref.predict(rules, q["items"], q["num"], DOC_PARAMS["maxRuleLength"],
                                      name=lambda i: names[i], index=index.get)
            answers.append(res)
    assert answers[:len(queries)] == answers[len(queries):]
    assert [r["cond"] for r in answers[1]["rules"]] == [["s2i6"], ["s2i4"]]     # query order
    assert answers[0]["rules"][0]["itemScores"][0]["item"] == "s2i5" and answers[3] == {"rules": []}
    # BatchPredict writes what per-query predict gives
    (tmp_path / "in.json").write_text("\n".join(json.dumps(q) for q in queries) + "\n")
    out = tmp_path / "out.json"
    assert w.BatchPredict.main(["--input", str(tmp_path / "in.json"), "--output", str(out),
                                "--engine-instance-id", inst.id]) == len(queries)
    server = w.deploy(inst.id)
    algo, model = server.algorithms[0], server.models[0]
    qcls = algo.queryClass()
    want = [json.dumps({"query": w.to_json(w.extract_params(qcls, q)),
                        "prediction": w.to_json(algo.predict(model, w.extract_params(qcls, q)))}, separators=(",", ":"))
            for q in queries]
    assert out.read_text().splitlines() == want


def test_template_columns_equal_objects_and_missing_target(tmp_path, monkeypatch):
    monkeypatch.setenv("PIO_EVENTDATA_DIR", str(tmp_path / "events"))
    from pio_b200.templates import complementarypurchase as cp
    evs = _shop_events(9)
    s.import_events("CP2", evs)
    params = {**DOC_PARAMS, "maxRuleLength": 3, "minSupport": 0.01, "minConfidence": 0.0, "minLift": 0.0}
    sc = w.WorkflowContext()
    td = cp.DataSource(cp.DataSourceParams("CP2")).readTraining(sc)
    algo = cp.Algorithm(cp.AlgorithmParams(**params))
    m_cols = algo.train(sc, td)
    m_objs = algo.train(sc, cp.TrainingData(buyEvents=list(td.buyEvents)))
    for k in ("set_prefix", "set_item", "set_count", "rule_cond", "rule_conseq", "support", "confidence", "lift"):
        assert getattr(m_cols, k).tolist() == getattr(m_objs, k).tolist(), k
    assert m_cols.itemStringIntMap.toMap() == m_objs.itemStringIntMap.toMap()
    rules, names = _restated(evs, params)
    assert {frozenset(names[i] for i in c) for c in rules} == {
        frozenset(m_cols.itemIntStringMap(i) for i in c) for c in m_cols.rules}
    s.import_events("CP2", [dict(event="buy", entityType="user", entityId="ux", targetEntityType="item",
                                 eventTime="2021-02-01T00:00:00Z")])
    with pytest.raises(ValueError, match="targetEntityId"):
        cp.DataSource(cp.DataSourceParams("CP2")).readTraining(sc)
