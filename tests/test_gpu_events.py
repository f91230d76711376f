"""GPU tests (-m gpu) of the event scanner: pio_events_scan against the CPU driver of event_line.h, findColumns against
find on awkward files, and the recommendation template trained from event columns against training from the host
path's Rating list (BiMaps and factors bit for bit)."""
import datetime as dt
import json
import struct

import numpy as np
import pytest

import event_corpus as EC
from pio_b200 import storage as s
from pio_b200 import workflow as w
from test_event_line import driver, run_driver  # noqa: F401  (the g++ driver fixture)

pytestmark = pytest.mark.gpu


def scan_by_line(native, lines, f, sep=b"\n"):
    r = native.events_scan(sep.join(lines), **EC.native_filter_args(f))
    assert r["n_lines"] == len(lines)
    text = sep.join(lines)
    ev = {}
    for k, ln in enumerate(r["line"]):
        ev[int(ln)] = (int(r["code"][k]), int(r["flags"][k] & 1), struct.pack("<d", r["value"][k]) if r["flags"][k] & 1
                       else None, int(r["flags"][k] >> 1 & 1), int(r["time_us"][k]),
                       r["eid_bytes"][r["eid_off"][k]:r["eid_off"][k + 1]].tobytes(),
                       r["tid_bytes"][r["tid_off"][k]:r["tid_off"][k + 1]].tobytes())
    fb = {int(ln): text[b:e] for ln, b, e in zip(r["fb_line"], r["fb_begin"], r["fb_end"])}
    return ev, fb


@pytest.mark.parametrize("chunk,smem", [(None, "1"), ("4096", "1"), ("333", "1"), (None, "0"), ("4096", "0")])
def test_abi_matches_cpu_driver(native, driver, monkeypatch, chunk, smem):  # noqa: F811
    """Both parse kernels (lines staged in shared memory, or read from global memory) at several device chunk sizes."""
    monkeypatch.setenv("PIO_EVENTS_SMEM", smem)
    if chunk:
        monkeypatch.setenv("PIO_EVENTS_DEVICE_CHUNK", chunk)
    lines = EC.import_lines(3000, 41) + EC.mutate(EC.import_lines(500, 42), 8000, 43) + EC.edge_lines()
    for f in EC.FILTERS:
        ev, fb = scan_by_line(native, lines, f)
        for j, (line, (oc, code, has, bits, has_t, t_us, eid, tid)) in enumerate(zip(lines, run_driver(driver, f, lines))):
            if chunk and len(line) >= int(chunk):   # a line longer than a device chunk always goes to the host
                assert j not in ev and fb.get(j) == line, (j, line[:120])
            elif oc == EC.MATCHED:
                assert ev.get(j) == (code, has, bits if has else None, has_t, t_us, eid, tid), (j, line[:120])
            elif oc == EC.FALLBACK:
                assert j not in ev and fb.get(j) == line, (j, line[:120])
            else:
                assert j not in ev and j not in fb, (j, line[:120])


def expected_columns(app, **kw):
    evs = s.PEventStore.find(app, entityType=kw.get("entityType"), eventNames=kw.get("eventNames"),
                             targetEntityType=kw.get("targetEntityType", s._UNSET), startTime=kw.get("startTime"),
                             untilTime=kw.get("untilTime"))
    prop = kw.get("property")
    out = []
    for e in evs:
        has, v = False, 0.0
        if prop is not None and e.properties.contains(prop):
            try:
                v, has = e.properties.get(prop, float), True
            except Exception:
                pass
        out.append((-1 if kw.get("eventNames") is None else kw["eventNames"].index(e.event), has, v if has else None,
                    s.time_us(e.eventTime), e.entityId, e.targetEntityId))
    return out


def got_columns(app, **kw):
    c = s.PEventStore.findColumns(app, **kw)
    eid, tid = s.string_list(c.entityId), s.string_list(c.targetEntityId)
    return [(int(c.code[k]), bool(c.has_value[k]), float(c.value[k]) if c.has_value[k] else None, int(c.time_us[k]),
             eid[k], tid[k] if c.has_target[k] else None) for k in range(len(c))], c


def write_app(tmp_path, monkeypatch, name, raw: bytes):
    monkeypatch.setenv("PIO_EVENTDATA_DIR", str(tmp_path / "events"))
    p = s.app_file(name)
    p.parent.mkdir(parents=True, exist_ok=True)
    p.write_bytes(raw)


TEMPLATE = dict(entityType="user", eventNames=["rate", "buy"], targetEntityType="item", property="rating")


@pytest.mark.parametrize("layout", ["crlf", "cr", "no_final_newline", "blank_lines", "long_line"])
def test_find_columns_equals_find_on_awkward_files(native, tmp_path, monkeypatch, layout):
    lines = EC.import_lines(1500, 51) + EC.mutate(EC.import_lines(200, 52), 300, 53)
    # find raises on a bad line, and an event without eventTime is stamped now(), differently by each call
    lines = [x for x in lines if EC.restate(x, EC.FILTERS[1]) != ("raise",) and
             isinstance(json.loads(x.decode()).get("eventTime"), str)]
    sep = {"crlf": b"\r\n", "cr": b"\r"}.get(layout, b"\n")
    if layout == "blank_lines":
        lines = [x if k % 7 else b"  \t" for k, x in enumerate(lines)] + [b"", b""]
    if layout == "long_line":
        lines.insert(700, json.dumps({"event": "rate", "entityType": "user", "entityId": "big", "targetEntityType": "item",
                                      "targetEntityId": "x" * 9000, "properties": {"rating": 2},
                                      "eventTime": "2021-01-01T00:00:00"}).encode())
    raw = sep.join(lines) + (b"" if layout == "no_final_newline" else sep)
    write_app(tmp_path, monkeypatch, "A", raw)
    for chunk_bytes, dev_chunk in ((None, None), (997, "611"), (4096, "4096"), (2500, "8191")):
        if dev_chunk:
            monkeypatch.setenv("PIO_EVENTS_DEVICE_CHUNK", dev_chunk)
        else:
            monkeypatch.delenv("PIO_EVENTS_DEVICE_CHUNK", raising=False)
        for kw in (TEMPLATE, {}, dict(eventNames=[]), dict(entityType="user", eventNames=[], property="rating"),
                   dict(entityType="item", eventNames=["view", "$set"], targetEntityType=None, property="w",
                        startTime="1999-01-01T00:00:00Z", untilTime="2030-06-01T12:00:00.000001")):
            got, c = got_columns("A", chunk_bytes=chunk_bytes, **kw)
            assert got == expected_columns("A", **kw), (layout, chunk_bytes, kw)
            if kw.get("eventNames") == []:   # an empty name list matches nothing, however a line was parsed
                assert got == []
            assert c.n_fallback < len(lines)


def test_find_columns_two_million_events_over_many_chunks(native, tmp_path, monkeypatch):
    n = 2_000_000
    rng = np.random.default_rng(7)
    u, i, r = rng.integers(0, 50000, n), rng.integers(0, 8000, n), rng.integers(1, 6, n)
    ev = np.where(rng.random(n) < 0.3, "buy", "rate")
    lines = [f'{{"event": "{e}", "entityType": "user", "entityId": "u{a}", "targetEntityType": "item", '
             f'"targetEntityId": "i{b}", "properties": {{"rating": {c}}}, "eventTime": "2021-03-04T05:06:{k % 60:02d}.{k % 999983:06d}+02:00"}}'
             for k, (e, a, b, c) in enumerate(zip(ev.tolist(), u.tolist(), i.tolist(), r.tolist()))]
    write_app(tmp_path, monkeypatch, "Big", ("\n".join(lines) + "\n").encode())
    got, c = got_columns("Big", chunk_bytes=16 << 20, **TEMPLATE)
    assert c.n_fallback == 0 and len(got) == n
    assert got == expected_columns("Big", **TEMPLATE)


@pytest.mark.parametrize("bad", [b'{"event": "rate", "entityType": "user"', b'{"event":"rate","entityType":"user",'
                                 b'"entityId":"u","eventTime":"2021-02-30T00:00:00"}', b'[1]', b'{"entityType":"user",'
                                 b'"entityId":"u","eventTime":"2021-01-01T00:00:00"}', b'\xff\xfe'])
def test_malformed_line_raises_what_find_raises(native, tmp_path, monkeypatch, bad):
    lines = EC.import_lines(300, 61)
    lines.insert(150, bad)
    write_app(tmp_path, monkeypatch, "Bad", b"\n".join(lines) + b"\n")
    with pytest.raises(Exception) as want:
        s.PEventStore.find("Bad", entityType="user")
    with pytest.raises(Exception) as got:
        s.PEventStore.findColumns("Bad", **TEMPLATE)
    assert type(got.value) is type(want.value), (got.value, want.value)


def _rating_events(nu, ni, nnz, seed, implicit):
    rng = np.random.default_rng(seed)
    t0 = dt.datetime(2021, 1, 1, tzinfo=dt.timezone.utc)
    evs = []
    for e in range(nnz):
        u, i = f"u{rng.integers(nu)}", ("ü" if e % 97 == 0 else "i") + str(int(rng.integers(ni)))
        kind = "view" if implicit and e % 5 == 0 else "buy" if e % 3 == 0 else "rate"
        d = dict(event=kind, entityType="user", entityId=u, targetEntityType="item", targetEntityId=i,
                 eventTime=(t0 + dt.timedelta(seconds=e, microseconds=e % 1000)).isoformat())
        if kind == "rate":
            d["properties"] = {"rating": float(rng.integers(1, 11)) / 2}
        evs.append(d)
    return evs


def _host_ratings(app):
    from pio_b200.templates import recommendation as rec
    out = []
    for e in s.PEventStore.find(appName=app, entityType="user", eventNames=["rate", "buy"], targetEntityType="item"):
        out.append(rec.Rating(e.entityId, e.targetEntityId, e.properties.get("rating", float) if e.event == "rate" else 4.0))
    return out


@pytest.mark.parametrize("implicit", [False, True])
def test_recommendation_template_trains_bit_identically_from_columns(native, tmp_path, monkeypatch, implicit):
    from pio_b200.templates import recommendation as rec
    monkeypatch.setenv("PIO_EVENTDATA_DIR", str(tmp_path / "events"))
    s.import_events("R", _rating_events(300, 70, 4000, 9, implicit))
    # a line the device hands to the host, and one more rating from it
    s.import_events("R", [dict(event="rate", entityType="user", entityId="u1", targetEntityType="item",
                               targetEntityId="i1", properties={"rating": 0.30000000000000004},
                               eventTime="2021-01-01T00:00:00")])
    ds = rec.DataSource(rec.DataSourceParams(appName="R"))
    sc = w.WorkflowContext()
    td = ds.readTraining(sc)
    host = _host_ratings("R")
    assert td.columns is not None and td.ratings == host
    ap = rec.ALSAlgorithmParams(rank=8, numIterations=4, lambda_=0.05, seed=3, implicitPrefs=implicit)
    algo = rec.ALSAlgorithm(ap)
    m_cols = algo.train(sc, rec.Preparator().prepare(sc, ds.readTraining(sc)))
    m_host = algo.train(sc, rec.TrainingData(host))
    assert m_cols.userStringIntMap.toMap() == m_host.userStringIntMap.toMap()
    assert m_cols.itemStringIntMap.toMap() == m_host.itemStringIntMap.toMap()
    assert np.array_equal(m_cols.userFeatures, m_host.userFeatures)
    assert np.array_equal(m_cols.productFeatures, m_host.productFeatures)


def test_rate_event_without_rating_raises_as_before(native, tmp_path, monkeypatch):
    from pio_b200.templates import recommendation as rec
    for props, exc in (({}, s.DataMapException), ({"rating": None}, s.DataMapException), ({"rating": "x"}, ValueError)):
        monkeypatch.setenv("PIO_EVENTDATA_DIR", str(tmp_path / f"ev{len(str(props))}{exc.__name__}"))
        evs = _rating_events(20, 10, 50, 1, False)
        evs.insert(20, dict(event="rate", entityType="user", entityId="u", targetEntityType="item", targetEntityId="i",
                            properties=props, eventTime="2021-01-01T00:00:00"))
        s.import_events("R", evs)
        with pytest.raises(exc) as got:
            rec.DataSource(rec.DataSourceParams(appName="R")).readTraining(None)
        with pytest.raises(exc) as want:
            _host_ratings("R")
        assert str(got.value) == str(want.value)


def test_read_eval_folds_equal_host_folds(native, tmp_path, monkeypatch):
    from pio_b200.templates import recommendation as rec
    monkeypatch.setenv("PIO_EVENTDATA_DIR", str(tmp_path / "events"))
    s.import_events("R", _rating_events(200, 50, 3000, 4, False))
    ds = rec.DataSource(rec.DataSourceParams(appName="R", evalParams=rec.DataSourceEvalParams(kFold=5, queryNum=7)))
    folds = ds.readEval(None)
    ratings = list(enumerate(_host_ratings("R")))
    for idx, (td, _, qas) in enumerate(folds):
        assert td.ratings == [r for k, r in ratings if k % 5 != idx]
        test = [r for k, r in ratings if k % 5 == idx]
        by_user = {}
        for r in test:
            by_user.setdefault(r.user, []).append(r)
        assert qas == [(rec.Query(u, 7, set()), rec.ActualResult(rs)) for u, rs in by_user.items()]
