"""GPU tests (-m gpu) of the event index (LEventStore.entityIndex, native.EventsIndex): every answer of
EntityEventIndex.find is compared with LEventStore.findByEntity on the same file -- the events' to_json() and the UTC
offset of each eventTime -- over awkward files, forced hash collisions, appends on both sides of the delta merge,
rewrites, a missing file, a batched lookup, and the ecommerce template's predict."""
import datetime as dt
import json
import random
import re

import numpy as np
import pytest

import event_corpus as EC
from pio_b200 import native
from pio_b200 import storage as s
from pio_b200 import workflow as w

pytestmark = pytest.mark.gpu

APP = "Ix"
DIVISOR = int(re.search(r"#define PIO_EVENTS_INDEX_MERGE_DIVISOR (\d+)",
                        (native.REPO_ROOT / "include" / "pio_als.h").read_text()).group(1))
LIMITS = [None, 0, 1, 10, -1]
VIEWS = [
    dict(entityType="user", eventNames=["rate", "buy"], targetEntityType="item"),
    dict(entityType="user", eventNames=None),
    dict(entityType="item", eventNames=["view", "$set"], targetEntityType=None),
    dict(entityType="ü", eventNames=["rate", "räte", "😀"], targetEntityType="日本"),
    dict(entityType="user", eventNames=[]),
]


@pytest.fixture
def app(tmp_path, monkeypatch):
    monkeypatch.setenv("PIO_EVENTDATA_DIR", str(tmp_path / "events"))
    p = s.app_file(APP)
    p.parent.mkdir(parents=True)
    return p


def dump(evs):
    return [(e.to_json(), e.eventTime.utcoffset()) for e in evs]


def ref(view, eid, limit=None):
    return dump(s.LEventStore.findByEntity(APP, view["entityType"], eid, eventNames=view["eventNames"],
                                           targetEntityType=view.get("targetEntityType", s._UNSET), limit=limit))


def grouped(view):
    """findByEntity of every entity at once: find's events of the view by entityId, latest first (stable)."""
    out = {}
    for e in s.PEventStore.find(APP, entityType=view["entityType"], eventNames=view["eventNames"],
                                targetEntityType=view.get("targetEntityType", s._UNSET)):
        out.setdefault(e.entityId, []).append(e)
    return {k: dump(sorted(v, key=lambda e: e.eventTime, reverse=True)) for k, v in out.items()}


def check(ix, view, ids, sample):
    """ids: every id against the grouped reference (one batched lookup per limit); sample: each against findByEntity."""
    allv = grouped(view)
    for limit in LIMITS:
        got = ix.find_many(ids, limit)
        for eid, g in zip(ids, got):
            want = allv.get(eid, [])
            assert dump(g) == (want if limit is None or limit < 0 else want[:limit]), (view, eid, limit)
        for eid in sample:
            assert dump(ix.find(eid, limit)) == ref(view, eid, limit), (view, eid, limit)


def _good(line: bytes) -> bool:
    """Lines find accepts, with a fixed eventTime (an absent one is the time of the call)."""
    try:
        d = json.loads(line.decode("utf-8").strip())
        s.Event.from_json(d)
        return isinstance(d.get("eventTime"), str)
    except Exception:
        return False


def extra_lines():
    ev = lambda eid, t, **kw: json.dumps(dict(dict(event="rate", entityType="user", entityId=eid,  # noqa: E731
                                                   targetEntityType="item", targetEntityId="i1", eventTime=t), **kw))
    L = [ev("tie", "2021-01-01T00:00:00Z", properties={"k": 1}), ev("tie", "2021-01-01T01:00:00+01:00"),
         ev("tie", "2020-12-31T23:00:00-01:00", eventId="e3"), ev("tie", "2021-01-01T00:00:00.000001Z"),
         ev("old", "1950-06-01T00:00:00Z"), ev("old", "0001-01-01T00:00:00"), ev("old", "1969-12-31T23:59:59.999999Z"),
         ev(77, "2021-01-01T00:00:00Z"), ev("77", "2021-01-01T00:00:00Z"), ev("a\"b\\c", "2022-01-01T00:00:00Z"),
         ev("😀🙂", "2022-01-01T00:00:00Z"), ev("\U0001F600", "2022-01-01T00:00:00Z", properties={"rating": 0.1 + 0.2}),
         ev("tie", "2021-01-01T00:00:00Z", properties={"rating": 0.30000000000000004}),
         # duplicated keys and a time without seconds: find takes them, the device scanner leaves them to the host
         '{"event":"rate","entityType":"user","entityId":"x","entityId":"tie","targetEntityType":"item",'
         '"eventTime":"2021-01-01T00:00:00Z"}',
         '{"event":"buy","entityType":"user","entityId":"tie","targetEntityType":"item","eventTime":"2021-01-01T00:00"}']
    return [x.encode() for x in L]


def corpus(n, seed):
    return [x for x in EC.import_lines(n, seed) + EC.edge_lines() if _good(x)] + extra_lines()


def write_mixed(path, lines, seed):
    """Lines with "\\n", "\\r\\n" and lone "\\r" terminators, blank lines, and a last line without a terminator."""
    rng = random.Random(seed)
    out = bytearray()
    for k, x in enumerate(lines):
        out += x
        if k < len(lines) - 1:
            out += rng.choice([b"\n", b"\n", b"\r\n", b"\r"]) + (b"\n  \t\n" if rng.random() < 0.05 else b"")
    path.write_bytes(bytes(out))


def ids_of(lines):
    ids = {s.Event.from_json(json.loads(x.decode("utf-8").strip())).entityId for x in lines}
    return sorted(ids) + ["nobody", "", "tie "]


def test_every_entity_of_a_seeded_corpus(native, app):
    lines = corpus(1500, 7)
    write_mixed(app, lines, 1)
    ids = ids_of(lines)
    sample = [i for i in ids if not i.lstrip("-").isdigit()] + ids[:5]
    r = native.events_scan(app.read_bytes(), entity_type="user", event_names=["rate", "buy"],
                           target_mode=native.EVENTS_TARGET_EQUALS, target_entity_type="item")
    assert len(r["fb_line"]) > 0                  # some lines of the view are parsed on the host
    for view in VIEWS:
        ix = s.LEventStore.entityIndex(APP, **view)
        check(ix, view, ids, sample)
        ix.close()


def test_forced_hash_collisions(native, app, monkeypatch):
    monkeypatch.setenv("PIO_IDS_HASH_BITS", "3")
    lines = corpus(800, 8)
    write_mixed(app, lines, 2)
    ids = ids_of(lines)
    for view in VIEWS[:2]:
        ix = s.LEventStore.entityIndex(APP, **view)
        check(ix, view, ids, ids[:12])
        ix.close()


def _events(n, seed, n_users=60, t0=dt.datetime(2021, 1, 1, tzinfo=dt.timezone.utc)):
    rng = np.random.default_rng(seed)
    return [dict(event=str(rng.choice(["rate", "buy", "view"])), entityType="user", entityId=f"u{rng.integers(n_users)}",
                 targetEntityType="item", targetEntityId=f"i{rng.integers(50)}",
                 eventTime=(t0 + dt.timedelta(seconds=int(rng.integers(0, 500)))).isoformat()) for _ in range(n)]


def test_appends_delta_merge_tail_and_bad_lines(native, app):
    view = VIEWS[0]
    ids = [f"u{k}" for k in range(62)]
    s.import_events(APP, _events(4000, 1))
    ix = s.LEventStore.entityIndex(APP, **view)
    check(ix, view, ids, ids[:3])
    st = ix.stats()
    main, merges = st["n_main"], st["n_merges"]
    assert st["n_delta"] == 0 and main > 0
    # a small append: lookups read a non-empty delta run
    s.import_events(APP, _events(20, 2))
    check(ix, view, ids, ids[:3])
    st = ix.stats()
    assert 0 < st["n_delta"] and st["n_main"] == main and st["n_merges"] == merges
    # an append past the merge threshold: lookups read the merged main run
    s.import_events(APP, _events(2 * (main // DIVISOR) + 100, 3, n_users=62))
    check(ix, view, ids, ids[:3])
    st = ix.stats()
    assert st["n_delta"] == 0 and st["n_merges"] == merges + 1 and st["n_main"] > main
    # an unterminated line, completed later
    line = json.dumps(dict(event="buy", entityType="user", entityId="u1", targetEntityType="item",
                           targetEntityId="i9", eventTime="2021-01-01T00:00:00Z")).encode()
    with open(app, "ab") as f:
        f.write(line[:40])
    for limit in LIMITS:   # find raises on the half line, and so does the index
        with pytest.raises(Exception) as a:
            ref(view, "u1", limit)
        with pytest.raises(Exception) as b:
            ix.find("u1", limit)
        assert type(a.value) is type(b.value) and str(a.value) == str(b.value)
    with open(app, "ab") as f:
        f.write(line[40:] + b"\r" + line.replace(b"i9", b"i8"))   # one more line ended by a lone CR, then none
    check(ix, view, ids, ["u1", "u2"])
    with open(app, "ab") as f:
        f.write(b"\n")
    check(ix, view, ids, ["u1", "u2"])
    # a bad line appended later raises what find raises, on every find
    with open(app, "ab") as f:
        f.write(b'{"event":"rate","entityType":"user"}\n')
    s.import_events(APP, _events(10, 4))
    for _ in range(2):
        for eid in ("u1", "nobody"):
            with pytest.raises(ValueError) as a:
                ref(view, eid)
            with pytest.raises(ValueError) as b:
                ix.find(eid)
            assert str(a.value) == str(b.value)
    ix.close()


def test_bad_line_already_in_the_file(native, app):
    s.import_events(APP, _events(300, 5))
    with open(app, "ab") as f:
        f.write(b'{"event":"rate","entityType":"user","entityId":"u1","eventTime":"2021-13-01T00:00:00"}\n')
        f.write(b"not json\n")
    s.import_events(APP, _events(300, 6))
    ix = s.LEventStore.entityIndex(APP, **VIEWS[0])
    for eid in ("u1", "u2", "nobody"):
        with pytest.raises(ValueError) as a:
            ref(VIEWS[0], eid)
        with pytest.raises(ValueError) as b:
            ix.find(eid)
        assert str(a.value) == str(b.value)
    ix.close()


def test_rewrites_and_a_missing_file(native, app):
    view = VIEWS[0]
    ids = [f"u{k}" for k in range(62)]
    ix = s.LEventStore.entityIndex(APP, **view)
    for _ in range(2):
        with pytest.raises(FileNotFoundError) as a:
            ref(view, "u1")
        with pytest.raises(FileNotFoundError) as b:
            ix.find("u1")
        assert str(a.value) == str(b.value)
    s.import_events(APP, _events(2000, 7))             # the file appears
    check(ix, view, ids, ids[:3])
    for n, seed in ((500, 8), (3000, 9), (3000, 10)):   # shorter, longer, and the same length with other events
        s.delete_app_data(APP)
        s.import_events(APP, _events(n, seed))
        check(ix, view, ids, ids[:3])
    s.delete_app_data(APP)
    with pytest.raises(FileNotFoundError):
        ix.find("u1")
    assert ix.stats() == {}                            # dropped
    s.import_events(APP, _events(100, 11))
    check(ix, view, ids, ids[:3])
    ix.close()


def test_batched_lookup_of_thousands_of_ids(native, app):
    view = VIEWS[0]
    evs = _events(30000, 12, n_users=4000)
    s.import_events(APP, evs)
    ids = [f"u{k}" for k in range(4100)]
    ix = s.LEventStore.entityIndex(APP, **view)
    allv = grouped(view)
    for limit in (None, 3):
        got = ix.find_many(ids, limit)
        assert len(got) == len(ids)
        for eid, g in zip(ids, got):
            want = allv.get(eid, [])
            assert dump(g) == (want if limit is None else want[:limit])
        for eid, g in list(zip(ids, got))[::200]:
            assert dump(g) == ref(view, eid, limit)
    ix.close()


def test_ecommerce_predict_through_the_indexes(native, app, tmp_path, monkeypatch):
    from pio_b200.templates import ecommerce as ec
    monkeypatch.setenv("PIO_MODELDATA_DIR", str(tmp_path / "models"))
    nu, ni = 80, 40
    t0 = dt.datetime(2021, 1, 1, tzinfo=dt.timezone.utc)
    rng = np.random.default_rng(13)
    sets = [dict(event="$set", entityType="user", entityId=f"u{k}", eventTime=t0.isoformat()) for k in range(nu)]
    sets += [dict(event="$set", entityType="item", entityId=f"i{k}", eventTime=t0.isoformat(),
                  properties={"categories": ["c%d" % (k % 3)]}) for k in range(ni)]
    evs = [dict(event=str(rng.choice(["rate", "buy", "view"])), entityType="user", entityId=f"u{rng.integers(nu)}",
                targetEntityType="item", targetEntityId=f"i{rng.integers(ni)}", properties={"rating": 3.0},
                eventTime=(t0 + dt.timedelta(seconds=int(rng.integers(0, 10000)))).isoformat()) for _ in range(2000)]
    s.import_events(APP, sets + evs)
    eng = ec.ECommerceRecommendationEngine().apply()
    ep = eng.jValueToEngineParams({"datasource": {"params": {"appName": APP}},
                                   "algorithms": [{"name": "ecomm", "params": {
                                       "appName": APP, "unseenOnly": True, "seenEvents": ["buy", "view"],
                                       "similarEvents": ["view"], "rank": 8, "numIterations": 4, "lambda": 0.05,
                                       "seed": 3}}]})
    sc = w.WorkflowContext()
    m = eng.prepareDeploy(sc, ep, "ix", eng.train(sc, ep, "ix"))[0]
    ap = ep.algorithmParamsList[0][1]

    class HostLookups(ec.ECommAlgorithm):   # the three lookups as findByEntity on the file
        def genBlackList(self, query):
            seen = {e.targetEntityId for e in s.LEventStore.findByEntity(
                APP, "user", query.user, eventNames=self.ap.seenEvents, targetEntityType="item")}
            unavailable = set()
            try:
                cons = s.LEventStore.findByEntity(APP, "constraint", "unavailableItems", eventNames=["$set"], limit=1)
                if cons:
                    unavailable = set(cons[0].properties.get("items"))
            except FileNotFoundError:
                pass
            return set(query.blackList or ()) | seen | unavailable

        def getRecentItems(self, query):
            return {e.targetEntityId for e in s.LEventStore.findByEntity(
                APP, "user", query.user, eventNames=self.ap.similarEvents, targetEntityType="item", limit=10)}

        def weightedItems(self):
            try:
                cons = s.LEventStore.findByEntity(APP, "constraint", "weightedItems", eventNames=["$set"], limit=1)
            except FileNotFoundError:
                return []
            return list(cons[0].properties.get("weights") or []) if cons else []

    algo, host = ec.ECommAlgorithm(ap), HostLookups(ap)
    users = [f"u{k}" for k in range(0, nu, 7)] + ["newcomer", "stranger"]

    def agree():
        for u in users:
            for q in (ec.Query(user=u, num=5), ec.Query(user=u, num=8, categories={"c1"}),
                      ec.Query(user=u, num=4, blackList={"i1", "i2"})):
                assert algo.predict(m, q) == host.predict(m, q), (u, q)

    agree()
    s.import_events(APP, [dict(event="view", entityType="user", entityId="newcomer", targetEntityType="item",
                               targetEntityId=f"i{k}", eventTime=(t0 + dt.timedelta(days=2, seconds=k)).isoformat())
                          for k in (3, 5, 7)])
    agree()
    s.import_events(APP, [dict(event="$set", entityType="constraint", entityId="unavailableItems",
                               eventTime=(t0 + dt.timedelta(days=3)).isoformat(), properties={"items": ["i3", "i4"]}),
                          dict(event="$set", entityType="constraint", entityId="weightedItems",
                               eventTime=(t0 + dt.timedelta(days=3)).isoformat(),
                               properties={"weights": [{"items": ["i5", "i6"], "weight": 3.0},
                                                       {"items": ["i7"], "weight": 0.0}]})])
    agree()
    s.import_events(APP, [dict(event="view", entityType="user", entityId=u, targetEntityType="item", targetEntityId="i9",
                               eventTime=(t0 + dt.timedelta(days=4)).isoformat()) for u in users])
    agree()
    assert algo.predict(m, ec.Query(user="newcomer", num=5)).itemScores
