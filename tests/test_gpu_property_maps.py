"""GPU tests (-m gpu) of PEventStore.aggregatePropertyMaps (pio_events_scan_props + pio_events_fold_props): element by
element what aggregateProperties returns -- entity order, ids, every key in dict order with its Python type, and
firstUpdated / lastUpdated with their UTC offsets."""
import datetime as dt
import json
import random

import numpy as np
import pytest

import test_reference_specs as RS
from pio_b200 import storage as s
from test_event_keys import ENTITY_PROPS, _entity_line
from test_event_props import props_lines
from test_gpu_properties import _entity_file

pytestmark = pytest.mark.gpu


def _typed(v):
    """A JSON value with its Python types spelled out (json.dumps alone does not tell 1 from True)."""
    if isinstance(v, dict):
        return [[k, _typed(x)] for k, x in v.items()]
    if isinstance(v, list):
        return [_typed(x) for x in v]
    return [type(v).__name__, repr(v)]


def _same(app, entityType, **kw):
    want = s.PEventStore.aggregateProperties(app, entityType, **{k: v for k, v in kw.items() if k != "chunk_bytes"})
    got = s.PEventStore.aggregatePropertyMaps(app, entityType, **kw)
    assert len(got) == len(want)
    for (gk, gp), (wk, wp) in zip(got, want):
        assert gk == wk
        assert json.dumps(_typed(gp.fields)) == json.dumps(_typed(wp.fields)), (gk, gp, wp)
        assert list(gp.fields) == list(wp.fields)
        for a, b in ((gp.firstUpdated, wp.firstUpdated), (gp.lastUpdated, wp.lastUpdated)):
            assert a == b and a.utcoffset() == b.utcoffset() and a.isoformat() == b.isoformat(), (gk, a, b)
        assert gp == wp
    return got


def test_reference_spec_fixtures(native, tmp_path, monkeypatch):
    monkeypatch.setenv("PIO_EVENTDATA_DIR", str(tmp_path))
    for name, evs in (("two", [RS.u1e5, RS.u2e2, RS.u1e3, RS.u1e1, RS.u2e3, RS.u2e1, RS.u1e4, RS.u1e2]),
                      ("del", [RS.u1e5, RS.u2e2, RS.u1e3, RS.u1ed, RS.u1e1, RS.u2e3, RS.u2e1, RS.u1e4, RS.u1e2]),
                      ("del2", [RS.u1e4, RS.u1e2, RS.u1ed, RS.u1e3, RS.u1e1, RS.u1e5])):
        s.import_events(name, evs)
        _same(name, "user")
        _same(name, "user", required=["e"])


def _offset_file(n_ent, n_ev, seed):
    """Entity events with pre-1970 times and equal instants written in different UTC offsets, duplicate keys, many
    value types, and events of other kinds and types mixed in."""
    rng = random.Random(seed)
    base = [dt.datetime(1969, 12, 31, 23, 59, 59, tzinfo=dt.timezone.utc), dt.datetime(2021, 1, 1, tzinfo=dt.timezone.utc)]
    lines = []
    for _ in range(n_ev):
        t = rng.choice(base) + dt.timedelta(seconds=rng.choice([-2, 0, 0, 1]), microseconds=rng.choice([0, 0, 7]))
        tz = dt.timezone(dt.timedelta(hours=rng.choice([0, 5, -8]), minutes=rng.choice([0, 30])))
        keys = rng.choices(["a", "b", "c", "é", "éx", "k"], k=rng.randint(0, 4))
        vals = [json.dumps(rng.choice([None, 1, 1.0, -0.0, True, "s", [1, {"n": None}], {}, 10 ** 20, 1e300]))
                for _ in keys]
        props = "{" + ",".join(f"{json.dumps(k) if rng.random() < 0.5 else json.dumps(k, ensure_ascii=False)}:{v}"
                               for k, v in zip(keys, vals)) + "}"
        name = rng.choice(["$set"] * 4 + ["$unset", "$delete", "view"])
        eid = rng.randrange(n_ent)
        eid_json = str(eid) if rng.random() < 0.2 else json.dumps(str(eid))   # 7 and "7" are one entity
        props_part = rng.choice([f'"properties":{props},', f'"properties":{props},', '"properties":null,', ""])
        lines.append(f'{{"event":"{name}","entityType":"{rng.choice(["item"] * 4 + ["user"])}","entityId":{eid_json},'
                     f'{props_part}"eventTime":"{t.astimezone(tz).isoformat()}"}}')
    return lines


def test_seeded_offsets_fallbacks_and_windows(native, tmp_path, monkeypatch):
    monkeypatch.setenv("PIO_EVENTDATA_DIR", str(tmp_path))
    lines = _offset_file(300, 20000, 3)
    lines[5] = lines[5] + " \x0c"                       # outside the device grammar: parsed on the host
    lines[9] = lines[9].replace('"eventTime"', '"x":NaN,"eventTime"', 1)
    lines.insert(20, "")
    lines.insert(30, "   ")
    (tmp_path / "O.jsonl").write_bytes(("\r\n".join(lines[:100]) + "\n" + "\n".join(lines[100:]) + "\n").encode())
    got = _same("O", "item")
    assert len(got) > 50
    _same("O", "user")
    _same("O", "item", required=["a", "é"])
    _same("O", "item", startTime="1969-12-31T23:59:59Z", untilTime="2021-01-01T05:30:00.000007+05:30")
    _same("O", "item", chunk_bytes=1 << 12)


@pytest.mark.parametrize("chunk,smem", [("700", "1"), ("4096", "0"), (None, "0")])
def test_device_chunks_and_smem(native, tmp_path, monkeypatch, chunk, smem):
    monkeypatch.setenv("PIO_EVENTDATA_DIR", str(tmp_path))
    monkeypatch.setenv("PIO_EVENTS_SMEM", smem)
    if chunk:
        monkeypatch.setenv("PIO_EVENTS_DEVICE_CHUNK", chunk)   # the line with 1 200 keys falls back on size
    lines = [x.decode() for x in props_lines()] + _offset_file(100, 3000, 4)
    (tmp_path / "C.jsonl").write_text("\n".join(lines) + "\n")
    _same("C", "item")


def test_hash_collisions_and_many_keys(native, tmp_path, monkeypatch):
    monkeypatch.setenv("PIO_EVENTDATA_DIR", str(tmp_path))
    rng = random.Random(9)
    lines = _entity_file(2000, 30000, 6)
    for j in range(3000):   # thousands of distinct keys
        props = {f"key{rng.randrange(5000)}": rng.choice([1, "v", None, [j]]) for _ in range(rng.randint(1, 5))}
        lines.append(json.dumps(dict(event=rng.choice(["$set", "$set", "$unset"]), entityType="item",
                                     entityId=f"e{rng.randrange(2000)}", properties=props,
                                     eventTime=f"2021-01-0{rng.randint(1, 9)}T00:00:00Z")))
    (tmp_path / "H.jsonl").write_text("\n".join(lines) + "\n")
    got = _same("H", "item")
    assert len({k for _, pm in got for k in pm.fields}) > 2000
    monkeypatch.setenv("PIO_IDS_HASH_BITS", "3")
    _same("H", "item")
    _same("H", "user")


def test_channels_and_entity_lines(native, tmp_path, monkeypatch):
    monkeypatch.setenv("PIO_EVENTDATA_DIR", str(tmp_path))
    lines = [x.decode() for x in props_lines() if b'"$delete"' not in x]   # every entity keeps its map
    (tmp_path / "A.ch.jsonl").write_text("\n".join(lines) + "\n")
    (tmp_path / "A.jsonl").write_text("\n".join(lines[:10]) + "\n")
    assert len(_same("A", "item", channelName="ch")) > 10
    _same("A", "item")


def _raises(fn):
    try:
        fn()
    except Exception as e:  # noqa: BLE001
        return type(e), str(e)
    return None


def test_bad_lines_and_missing_app_raise_as_the_host_path(native, tmp_path, monkeypatch):
    monkeypatch.setenv("PIO_EVENTDATA_DIR", str(tmp_path))
    good = [_entity_line("$set", p, eid=f"e{k}").decode() for k, p in enumerate(ENTITY_PROPS)]
    for bad in ('{"event":"$set","entityType":"item"}', "{not json", '{"event":"$set","entityType":"item",'
                '"entityId":"x","eventTime":"2021-13-01T00:00:00Z"}'):
        (tmp_path / "B.jsonl").write_text("\n".join(good[:5] + [bad] + good[5:] + ["[1"]) + "\n")
        want = _raises(lambda: s.PEventStore.aggregateProperties("B", "item"))
        assert want is not None and _raises(lambda: s.PEventStore.aggregatePropertyMaps("B", "item")) == want
    want = _raises(lambda: s.PEventStore.aggregateProperties("missing", "item"))
    assert want[0] is FileNotFoundError and _raises(lambda: s.PEventStore.aggregatePropertyMaps("missing", "item")) == want


def test_bad_arguments_are_refused(native):
    import ctypes as C
    L = native.lib()
    text = np.frombuffer(_entity_line("$set", '{"a":1}'), np.uint8)
    n = text.shape[0]
    z = lambda k, t=np.int64: np.zeros(k, t)  # noqa: E731
    i64 = [z(n + 2) for _ in range(10)]
    cnt = [C.c_int64(0) for _ in range(5)]

    def scan(prop, rec_cap, null_keys=False):
        f, keep = native._events_filter(None, None, 0, None, prop, None, None)
        return L.pio_events_scan_props(C.c_int(0), text.ctypes.data_as(C.c_void_p), C.c_int64(n), C.byref(f),
                                       C.c_int64(n), *[C.c_void_p(a.ctypes.data) for a in i64[:9]],
                                       C.c_void_p(z(n, np.int16).ctypes.data), C.c_void_p(i64[9].ctypes.data),
                                       C.c_int64(rec_cap), C.c_void_p(z(n, np.uint8).ctypes.data),
                                       None if null_keys else C.c_void_p(z(n + 2).ctypes.data),
                                       C.c_void_p(z(n, np.uint8).ctypes.data), C.c_void_p(z(n + 2).ctypes.data),
                                       C.byref(cnt[0]), C.byref(cnt[1]), C.c_int64(0), None, None, None,
                                       C.byref(cnt[2]), C.byref(cnt[3]))
    assert scan(None, n // 4 + 1) == 0 and cnt[1].value == 1
    assert scan("a", n // 4 + 1) == native.ERR_ARG            # filter->property set
    assert scan(None, n // 4) == native.ERR_ARG               # rec_capacity below the bound
    assert scan(None, n // 4 + 1, null_keys=True) == native.ERR_ARG
    eid = (np.frombuffer(b"ab", np.uint8), np.array([0, 1, 2], np.int64))
    keys = (np.frombuffer(b"k", np.uint8), np.array([0, 1], np.int64))
    for code, prop in (([0, 3], [0, 1, 1]), ([0, -1], [0, 1, 1]), ([0, 1], [0, 1, 0]), ([0, 1], [1, 1, 2])):
        with pytest.raises(native.NativeError) as e:
            native.events_fold_props(eid, np.array(code, np.int32), np.zeros(2, np.int64), np.array(prop, np.int64),
                                     keys)
        assert e.value.code == native.ERR_ARG, (code, prop)
