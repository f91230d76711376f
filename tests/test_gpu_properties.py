"""GPU tests (-m gpu) of the keyed event scan (pio_events_scan_keys), the $set / $unset / $delete fold
(pio_events_fold), PEventStore.aggregatePropertyColumns, and the similarproduct, ecommerce and classification templates
trained from columns against the same templates trained from the host path."""
import datetime as dt
import json
import random

import numpy as np
import pytest

import event_corpus as EC
import test_reference_specs as RS
from pio_b200 import storage as s
from test_event_keys import ENTITY_PROPS, _entity_line, run
from test_event_keys import driver  # noqa: F401  (the g++ driver fixture)

pytestmark = pytest.mark.gpu

KEYS = ["categories", "plan", "attr0", "w", "rating"]


@pytest.mark.parametrize("chunk,smem", [(None, "1"), ("4096", "1"), ("333", "1"), (None, "0"), ("4096", "0")])
def test_scan_keys_matches_cpu_driver(native, driver, monkeypatch, chunk, smem):  # noqa: F811
    monkeypatch.setenv("PIO_EVENTS_SMEM", smem)
    if chunk:
        monkeypatch.setenv("PIO_EVENTS_DEVICE_CHUNK", chunk)
    lines = EC.import_lines(2000, 71) + EC.mutate(EC.import_lines(300, 72), 3000, 73) + EC.edge_lines()
    lines += [_entity_line(ev, p, eid=f"e{k}") for k, ev in enumerate(["$set", "$unset", "$delete"] * 3)
              for p in ENTITY_PROPS]
    for f in (dict(EC.FILTERS[1], prop=None), dict(EC.FILTERS[2], prop=None)):
        r = native.events_scan_keys(b"\n".join(lines), KEYS, **{k: v for k, v in EC.native_filter_args(f).items()
                                                                if k != "prop"})
        assert r["n_lines"] == len(lines)
        at = {int(ln): k for k, ln in enumerate(r["line"])}
        fb = set(int(x) for x in r["fb_line"])
        nk = len(KEYS)
        for j, (line, (plain, keyed, present, number, vals)) in enumerate(zip(lines, run(driver, f, KEYS, lines))):
            oc = int(keyed.split(" ")[0])
            if chunk and len(line) >= int(chunk):
                assert j in fb and j not in at
            elif oc == EC.MATCHED:
                k = at[j]
                assert (int(r["present"][k]), int(r["number"][k])) == (present, number), (j, line[:120])
                for q in range(nk):
                    tok = r["tok_bytes"][r["tok_off"][k * nk + q]:r["tok_off"][k * nk + q + 1]].tobytes()
                    assert (r["num"][k, q].tobytes(), tok) == (np.float64(vals[q][0]).tobytes(), vals[q][1]), (j, q)
            elif oc == EC.FALLBACK:
                assert j in fb and j not in at
            else:
                assert j not in fb and j not in at


def test_bad_arguments_are_refused(native):
    text = _entity_line("$set", '{"a":1}')
    for keys in ([], ["a"] * 9, ["a", "a"], [""]):
        with pytest.raises(native.NativeError) as e:
            native.events_scan_keys(text, keys)
        assert e.value.code == native.ERR_ARG, keys
    with pytest.raises(native.NativeError) as e:
        native._events_scan(text, None, None, 0, None, "rating", None, None, 0, ["a"])   # filter->property set
    assert e.value.code == native.ERR_ARG
    eid = (np.frombuffer(b"ab", np.uint8), np.array([0, 1, 2], np.int64))
    for code, nk in (([0, 3], 1), ([0, -1], 1), ([0, 1], 9), ([0, 1], -1)):
        with pytest.raises(native.NativeError) as e:
            native.events_fold(eid, np.array(code, np.int32), np.zeros(2, np.int64), np.zeros(2, np.uint8), nk)
        assert e.value.code == native.ERR_ARG, (code, nk)


def _expected(app, entityType, keys, required=None, **kw):
    return [(k, {q: pm.fields[q] for q in keys if q in pm.fields}, s.time_us(pm.firstUpdated),
             s.time_us(pm.lastUpdated)) for k, pm in s.PEventStore.aggregateProperties(app, entityType, required=required,
                                                                                         **kw)]


def _got(app, entityType, keys, required=None, **kw):
    pc = s.PEventStore.aggregatePropertyColumns(app, entityType, keys, required=required, **kw)
    out = []
    columns = {q: pc.values(q) for q in keys}
    for i, k in enumerate(pc.entity_ids()):
        vals = {q: pc.value(i, q) for j, q in enumerate(keys) if pc.present[i, j]}
        for j, q in enumerate(keys):   # the number columns agree with the values
            if pc.has_number[i, j]:
                assert pc.number[i, j] == float(vals[q]) and not isinstance(vals[q], bool)
            elif pc.present[i, j] and isinstance(vals[q], int) and not isinstance(vals[q], bool):
                assert abs(vals[q]) > 2 ** 53   # an integer the device cannot hold exactly: its token only
        assert [columns[q][i] for q in keys] == [vals.get(q) for q in keys]
        out.append((k, vals, int(pc.first_us[i]), int(pc.last_us[i])))
    return out


def _same(a, b):
    """Equal lists of (id, values, first_us, last_us), value types included (json.loads of 1 and 1.0 differ)."""
    assert len(a) == len(b)
    for x, y in zip(a, b):
        assert x[0] == y[0] and x[2:] == y[2:], (x, y)
        assert json.dumps(x[1], sort_keys=True) == json.dumps(y[1], sort_keys=True), (x, y)


def test_reference_spec_fixtures(native, tmp_path, monkeypatch):
    monkeypatch.setenv("PIO_EVENTDATA_DIR", str(tmp_path))
    for name, evs in (("two", [RS.u1e5, RS.u2e2, RS.u1e3, RS.u1e1, RS.u2e3, RS.u2e1, RS.u1e4, RS.u1e2]),
                      ("del", [RS.u1e5, RS.u2e2, RS.u1e3, RS.u1ed, RS.u1e1, RS.u2e3, RS.u2e1, RS.u1e4, RS.u1e2]),
                      ("del2", [RS.u1e4, RS.u1e2, RS.u1ed, RS.u1e3, RS.u1e1, RS.u1e5])):
        s.import_events(name, evs)
        keys = ["a", "b", "d", "e", "g"]
        _same(_got(name, "user", keys), _expected(name, "user", keys))
        _same(_got(name, "user", keys, required=["e"]), _expected(name, "user", keys, required=["e"]))


def _entity_file(n_ent, n_ev, seed, n_views=0):
    rng = random.Random(seed)
    t0 = dt.datetime(2021, 1, 1, tzinfo=dt.timezone.utc)
    lines = []
    for _ in range(n_ev):
        name = rng.choice(["$set"] * 5 + ["$unset", "$delete"])
        t = t0 + dt.timedelta(seconds=rng.randint(-10 ** 9, 10 ** 4), microseconds=rng.choice([0, 1, 999999]))
        tz = dt.timezone(dt.timedelta(hours=rng.choice([0, 0, 3, -7])))
        props = {}
        for k in rng.sample(["categories", "plan", "attr0", "x"], rng.randint(0, 3)):
            props[k] = rng.choice([None, 1, -0.0, 2.5, "s", ["c1", "c2"], {"n": [1]}, True, 10 ** 20,
                                   0.30000000000000004])
        lines.append(json.dumps(dict(event=name, entityType=rng.choice(["item"] * 9 + ["user"]),
                                     entityId=f"e{rng.randrange(n_ent)}", properties=props,
                                     eventTime=t.astimezone(tz).isoformat())))
        if n_views and rng.random() < n_views:
            lines.append(json.dumps(dict(event="view", entityType="user", entityId=f"u{rng.randrange(100)}",
                                         targetEntityType="item", targetEntityId=f"e{rng.randrange(n_ent)}",
                                         eventTime=t.isoformat())))
    return lines


def test_seeded_file_chunks_collisions_windows(native, tmp_path, monkeypatch):
    """200 k entity events mixed with view events; then small pieces so that one entity's events span pieces, a 6-bit
    id hash so that different ids collide, time windows, required keys, and fallback lines."""
    monkeypatch.setenv("PIO_EVENTDATA_DIR", str(tmp_path))
    lines = _entity_file(20000, 200000, 5, n_views=0.5)
    lines[7] = lines[7].replace('"properties": {', '"properties": {"plan": 1.2345678901234567, ', 1)   # 17 digits
    lines[11] = lines[11] + " \x0c"   # outside the device grammar: the host parses it
    (tmp_path / "P.jsonl").write_text("\n".join(lines) + "\n")
    keys = ["categories", "plan", "attr0"]
    want = _expected("P", "item", keys)
    pc = s.PEventStore.aggregatePropertyColumns("P", "item", keys)
    assert pc.n_fallback >= 1
    _same(_got("P", "item", keys), want)
    _same(_got("P", "item", keys, chunk_bytes=1 << 16), want)
    monkeypatch.setenv("PIO_IDS_HASH_BITS", "6")
    _same(_got("P", "item", keys), want)
    monkeypatch.delenv("PIO_IDS_HASH_BITS")
    win = dict(startTime="2020-06-01T00:00:00Z", untilTime="2021-01-01T01:00:00+01:00")
    _same(_got("P", "item", keys, **win), _expected("P", "item", keys, **win))
    _same(_got("P", "item", keys, required=["plan", "x"]), _expected("P", "item", keys, required=["plan", "x"]))
    _same(_got("P", "user", ["plan"]), _expected("P", "user", ["plan"]))


# ---- templates ----------------------------------------------------------------------------------------------------------
def _template_events(seed, rating=True):
    rng = random.Random(seed)
    t0 = dt.datetime(1969, 12, 31, 23, 0, tzinfo=dt.timezone.utc)
    evs = [dict(event="$set", entityType="user", entityId=f"u{k}", eventTime=t0.isoformat()) for k in range(120)]
    evs += [dict(event="$set", entityType="item", entityId=f"i{k}", eventTime=t0.isoformat(),
                 properties={"categories": rng.choice([["a"], ["a", "b"], None, "c"])}) for k in range(45)]
    evs += [dict(event="$delete", entityType="user", entityId="u3", eventTime=(t0 + dt.timedelta(days=1)).isoformat())]
    for e in range(3000):
        t = t0 + dt.timedelta(seconds=rng.randint(0, 10 ** 6), microseconds=rng.randint(0, 999999))
        name = rng.choice(["view", "view", "like", "dislike", "rate", "buy"])
        d = dict(event=name, entityType="user", entityId=f"u{rng.randrange(125)}", targetEntityType="item",
                 targetEntityId=f"i{rng.randrange(50)}", eventTime=t.isoformat())
        if name == "rate" and rating:
            d["properties"] = {"rating": rng.choice([1, 2.5, 4, 5.0])}
        if e % 97 == 0:
            del d["targetEntityId"]
        evs.append(d)
    return evs


def _fit(eng, algo_json, td_cols, td_host, sc):
    ep = eng.jValueToEngineParams({"datasource": {"params": {"appName": "T"}}, "algorithms": [algo_json]})
    name, ap = ep.algorithmParamsList[0]
    algo = eng.algorithmClassMap[name](ap)
    return algo.train(sc, td_cols), algo.train(sc, td_host)


def test_similarproduct_columns_equal_host(native, tmp_path, monkeypatch):
    from pio_b200 import workflow as w
    from pio_b200.templates import similarproduct as sp
    monkeypatch.setenv("PIO_EVENTDATA_DIR", str(tmp_path))
    s.import_events("T", _template_events(1))
    sc = w.WorkflowContext()
    ds = sp.DataSource(sp.DataSourceParams(appName="T"))
    td = ds.readTraining(sc)
    host_users = {k: sp.User() for k, _ in s.PEventStore.aggregateProperties("T", "user")}
    host_items = {k: sp.Item(categories=pm.getOpt("categories")) for k, pm in s.PEventStore.aggregateProperties("T", "item")}
    views, likes = [], []
    for e in s.PEventStore.find("T", entityType="user", eventNames=["view", "like", "dislike"], targetEntityType="item"):
        t = int(e.eventTime.timestamp() * 1000)
        if e.event == "view":
            views.append(sp.ViewEvent(e.entityId, e.targetEntityId, t))
        else:
            likes.append(sp.LikeEvent(e.entityId, e.targetEntityId, t, e.event == "like"))
    host = sp.TrainingData(host_users, host_items, views, likes)
    eng = sp.SimilarProductEngine().apply()
    for algo in ({"name": "als", "params": {"rank": 8, "numIterations": 4, "lambda": 0.01, "seed": 3}},
                 {"name": "likealgo", "params": {"rank": 8, "numIterations": 4, "lambda": 0.01, "seed": 3}}):
        a, b = _fit(eng, algo, sp.TrainingData(columns=td.columns), host, sc)
        assert a.itemStringIntMap.toMap() == b.itemStringIntMap.toMap()
        assert list(a.itemStringIntMap.toMap()) == list(b.itemStringIntMap.toMap())
        assert np.array_equal(a.mf.productFeatures, b.mf.productFeatures) and np.array_equal(a.mf.userFeatures,
                                                                                          b.mf.userFeatures)
        assert a.items == b.items
    a, b = _fit(eng, {"name": "cooccurrence", "params": {"n": 10}}, sp.TrainingData(columns=td.columns), host, sc)
    assert a.itemStringIntMap.toMap() == b.itemStringIntMap.toMap() and a.items == b.items
    assert np.array_equal(a.top_items, b.top_items) and np.array_equal(a.top_counts, b.top_counts)
    assert np.array_equal(a.top_n, b.top_n)
    # the lazily built lists equal the host's
    assert td.users.keys() == host.users.keys() and td.items == host.items
    assert td.viewEvents == host.viewEvents and td.likeEvents == host.likeEvents


@pytest.mark.parametrize("implicit", [False, True])
def test_ecommerce_columns_equal_host(native, tmp_path, monkeypatch, implicit):
    from pio_b200 import workflow as w
    from pio_b200.templates import ecommerce as ec
    monkeypatch.setenv("PIO_EVENTDATA_DIR", str(tmp_path))
    s.import_events("T", _template_events(2))
    sc = w.WorkflowContext()
    td = ec.DataSource(ec.DataSourceParams(appName="T")).readTraining(sc)
    users = {k: True for k, _ in s.PEventStore.aggregateProperties("T", "user")}
    items = {k: ec.Item(pm.getOpt("categories")) for k, pm in s.PEventStore.aggregateProperties("T", "item")}
    rates, buys = [], []
    for e in s.PEventStore.find("T", entityType="user", eventNames=["rate", "buy"], targetEntityType="item"):
        t = int(e.eventTime.timestamp() * 1000)
        if e.event == "rate":
            rates.append(ec.RateEvent(e.entityId, e.targetEntityId, e.properties.get("rating", float), t))
        else:
            buys.append(ec.BuyEvent(e.entityId, e.targetEntityId, t))
    host = ec.TrainingData(users, items, rates, buys)
    ap = ec.ECommAlgorithmParams(appName="T", unseenOnly=False, seenEvents=["buy"], similarEvents=["view"], rank=8,
                                 numIterations=4, seed=3, implicitPrefs=implicit)
    a = ec.ECommAlgorithm(ap).train(sc, ec.TrainingData(columns=td.columns))
    b = ec.ECommAlgorithm(ap).train(sc, host)
    assert list(a.userStringIntMap.toMap().items()) == list(b.userStringIntMap.toMap().items())
    assert list(a.itemStringIntMap.toMap().items()) == list(b.itemStringIntMap.toMap().items())
    assert np.array_equal(a.mf.userFeatures, b.mf.userFeatures)
    assert np.array_equal(a.mf.productFeatures, b.mf.productFeatures)
    assert a.items == b.items and a.popularCount == b.popularCount
    assert td.rateEvents == host.rateEvents and td.buyEvents == host.buyEvents


def _raises(fn):
    try:
        fn()
    except Exception as e:  # noqa: BLE001
        return type(e), str(e)
    return None


def test_ecommerce_rate_without_rating_raises_as_before(native, tmp_path, monkeypatch):
    from pio_b200 import workflow as w
    from pio_b200.templates import ecommerce as ec
    monkeypatch.setenv("PIO_EVENTDATA_DIR", str(tmp_path))
    evs = _template_events(3)
    evs.append(dict(event="rate", entityType="user", entityId="u1", targetEntityType="item", targetEntityId="i1",
                    properties={"rating": "x"}, eventTime="2021-01-01T00:00:00Z"))
    evs.append(dict(event="rate", entityType="user", entityId="u1", targetEntityType="item", targetEntityId="i1",
                    eventTime="2021-01-01T00:00:00Z"))
    s.import_events("T", evs)

    def host():
        for e in s.PEventStore.find("T", entityType="user", eventNames=["rate", "buy"], targetEntityType="item"):
            if e.event == "rate":
                e.properties.get("rating", float)
    got = _raises(lambda: ec.DataSource(ec.DataSourceParams(appName="T")).readTraining(w.WorkflowContext()))
    assert got is not None and got == _raises(host)


def _classification_events(seed, extra=()):
    rng = random.Random(seed)
    t0 = dt.datetime(2021, 1, 1, tzinfo=dt.timezone.utc)
    evs = []
    for k in range(400):
        p = {"plan": rng.choice([0, 1, 2, 1.0]), "attr0": rng.choice([0, 1, 3, 2.5]), "attr1": rng.randint(0, 9),
             "attr2": rng.choice([0, 4, "7", True])}
        if k % 13 == 0:
            del p[rng.choice(list(p))]
        evs.append(dict(event="$set", entityType="user", entityId=f"u{k}", properties=p,
                        eventTime=(t0 + dt.timedelta(seconds=k)).isoformat()))
    return evs + list(extra)


def _nb_host(app):
    rows = s.PEventStore.aggregateProperties(app, "user", required=["plan", "attr0", "attr1", "attr2"])
    labels = np.array([pm.get("plan", float) for _, pm in rows], np.float64)
    feats = np.array([[pm.get("attr0", float), pm.get("attr1", float), pm.get("attr2", float)] for _, pm in rows],
                     np.float32).reshape(-1, 3)
    return labels, feats


def test_classification_columns_equal_host(native, tmp_path, monkeypatch):
    from pio_b200 import workflow as w
    from pio_b200.templates import classification as cl
    monkeypatch.setenv("PIO_EVENTDATA_DIR", str(tmp_path))
    s.import_events("C", _classification_events(4))
    sc = w.WorkflowContext()
    td = cl.DataSource(cl.DataSourceParams(appName="C")).readTraining(sc)
    labels, feats = _nb_host("C")
    assert np.array_equal(td.labels, labels) and td.labels.dtype == labels.dtype
    assert np.array_equal(td.features, feats) and td.features.dtype == feats.dtype
    a = cl.NaiveBayesAlgorithm(cl.AlgorithmParams(lambda_=1.0)).train(sc, td)
    b = cl.NaiveBayesAlgorithm(cl.AlgorithmParams(lambda_=1.0)).train(sc, cl.TrainingData(labels, feats))
    assert np.array_equal(a.pi, b.pi) and np.array_equal(a.theta, b.theta)


@pytest.mark.parametrize("bad", [{"plan": None}, {"plan": "x"}, {"attr1": None}, {"attr2": "y"}])
def test_classification_bad_value_raises_as_before(native, tmp_path, monkeypatch, bad):
    from pio_b200 import workflow as w
    from pio_b200.templates import classification as cl
    monkeypatch.setenv("PIO_EVENTDATA_DIR", str(tmp_path))
    late = dict(event="$set", entityType="user", entityId="u5", properties=bad, eventTime="2022-01-01T00:00:00Z")
    s.import_events("C", _classification_events(5, [late]))
    got = _raises(lambda: cl.DataSource(cl.DataSourceParams(appName="C")).readTraining(w.WorkflowContext()))
    assert got is not None and got == _raises(lambda: _nb_host("C"))
