"""GPU tests (-m gpu) of the lead scoring template (templates/leadscoring.py): sessions built on the device equal the
restatement tests/leadscoring_ref.py, bad events fail training, and the doc's engine.json runs end to end through
CreateWorkflow, deploy, a query and BatchPredict, with predictions equal to the restated forest's."""
import datetime as dt
import json

import numpy as np
import pytest

from pio_b200 import native
from pio_b200 import storage as s
from pio_b200 import workflow as w
from tests import forest_reg_ref as rr
from tests import leadscoring_ref as ref

pytestmark = pytest.mark.gpu

T0 = dt.datetime(2021, 3, 1, tzinfo=dt.timezone.utc)
DOC_ALGO = {"numClasses": 3, "numTrees": 5, "featureSubsetStrategy": "auto", "impurity": "variance", "maxDepth": 4,
            "maxBins": 100, "seed": 12345}


def lead_events(seed, n_sessions=300):
    """Views and buys of seeded sessions, shuffled across the file, with equal landing times, buys at the landing
    time, missing referrers / browsers and views of other target types."""
    rng = np.random.default_rng(seed)
    evs = []
    for k in range(n_sessions):
        sid = f"s{k}"
        base = T0 + dt.timedelta(seconds=int(rng.integers(0, 10 ** 6)))
        for v in range(int(rng.integers(1, 4))):
            props = {"sessionId": sid}
            if rng.random() < 0.8:
                props["referrerId"] = f"ref{int(rng.integers(0, 6))}.com"
            if rng.random() < 0.8:
                props["browser"] = ["Chrome", "Firefox", "Safari"][int(rng.integers(0, 3))]
            when = base + dt.timedelta(milliseconds=int(rng.integers(0, 3)), microseconds=int(rng.integers(0, 999)))
            evs.append(dict(event="view", entityType="user", entityId=f"u{k % 50}", targetEntityType="page",
                            targetEntityId=f"example.com/page{int(rng.integers(0, 12))}", eventTime=when.isoformat(),
                            properties=props))
        for b in range(int(rng.integers(0, 3))):
            when = base + dt.timedelta(milliseconds=int(rng.integers(0, 4)))
            evs.append(dict(event="buy", entityType="user", entityId=f"u{k % 50}", targetEntityType="item",
                            targetEntityId=f"i{b}", eventTime=when.isoformat(), properties={"sessionId": sid}))
    order = rng.permutation(len(evs))
    evs = [evs[i] for i in order]
    evs.append(dict(event="view", entityType="user", entityId="u1", targetEntityType="item", targetEntityId="x",
                    eventTime=T0.isoformat(), properties={}))          # not a page view: not read
    return evs


def restated_sessions(evs):
    rows = [{"event": e["event"], "t_ms": s.time_us(s._parse_time(e["eventTime"])) // 1000,
             "target": e["targetEntityId"], "properties": e.get("properties", {})}
            for e in evs if (e["event"], e["targetEntityType"]) in (("view", "page"), ("buy", "item"))]
    return ref.sessions(rows)


def test_device_sessions_equal_restatement(tmp_path, monkeypatch):
    monkeypatch.setenv("PIO_EVENTDATA_DIR", str(tmp_path / "events"))
    from pio_b200.templates import leadscoring as ls
    evs = lead_events(1)
    s.import_events("LS", evs)
    td = ls.DataSource(ls.DataSourceParams("LS")).readTraining(w.WorkflowContext())
    want = restated_sessions(evs)
    assert [(x.landingPageId, x.referrerId, x.browser, x.buy) for x in td.session] == [r[1:] for r in want]
    assert any(r[4] for r in want) and not all(r[4] for r in want)


def test_sessions_kernel_rules():
    # session 0: views at 5, 3, 3 (last of the equal ones lands), buy at 3 (not after); session 1: buy after
    sess = np.array([0, 0, 1, 0, 0, 1, 1])
    is_buy = np.array([0, 0, 0, 0, 1, 1, 0])
    t = np.array([5, 3, 7, 3, 3, 8, 7])
    landing, buy = native.lead_sessions(sess, is_buy, t, 2)
    assert landing.tolist() == [3, 6] and buy.tolist() == [False, True]
    landing, _ = native.lead_sessions(np.array([0, 1]), np.array([0, 1]), np.array([0, 0]), 2)
    assert landing.tolist() == [0, -1]
    with pytest.raises(native.NativeError):
        native.lead_sessions(np.array([0, 2]), np.array([0, 0]), np.array([0, 0]), 2)


@pytest.mark.parametrize("bad,msg", [("no_session", "Cannot get sessionId"), ("buy_only", "has buy events but no view")])
def test_bad_sessions_fail_training(tmp_path, monkeypatch, bad, msg):
    monkeypatch.setenv("PIO_EVENTDATA_DIR", str(tmp_path / "events"))
    from pio_b200.templates import leadscoring as ls
    evs = lead_events(2, 20)
    if bad == "no_session":
        evs.append(dict(event="view", entityType="user", entityId="u", targetEntityType="page", targetEntityId="p",
                        eventTime=T0.isoformat(), properties={"browser": "x"}))
    else:
        evs.append(dict(event="buy", entityType="user", entityId="u", targetEntityType="item", targetEntityId="i",
                        eventTime=T0.isoformat(), properties={"sessionId": "lonely"}))
    s.import_events("LSB", evs)
    with pytest.raises(ValueError, match=msg):
        ls.DataSource(ls.DataSourceParams("LSB")).readTraining(w.WorkflowContext())


def test_template_end_to_end(tmp_path, monkeypatch):
    monkeypatch.setenv("PIO_EVENTDATA_DIR", str(tmp_path / "events"))
    monkeypatch.setenv("PIO_MODELDATA_DIR", str(tmp_path / "models"))
    evs = lead_events(3, 500)
    s.import_events("MyApp1", evs)
    variant = tmp_path / "engine.json"
    variant.write_text(json.dumps({
        "id": "default", "description": "Default settings",
        "engineFactory": "pio_b200.templates.leadscoring.LeadScoringEngine",
        "datasource": {"params": {"appName": "MyApp1"}},
        "algorithms": [{"name": "randomforest", "params": DOC_ALGO}]}))
    inst = w.CreateWorkflow.main(["--engine-id", "ls", "--engine-version", "1", "--engine-variant", f"file:{variant}"])
    assert inst.status == "COMPLETED"
    labels, feats, maps = ref.prepare(restated_sessions(evs))
    cat = {k: len(maps[f]) for k, f in enumerate(ref.FEATURES)}
    forest = rr.train(labels, np.array(feats), 5, "auto", "variance", 4, 100, seed=12345, categorical=cat)
    queries = [{"landingPageId": "example.com/page9", "referrerId": "ref1.com", "browser": "Firefox"},
               {"landingPageId": "nowhere", "referrerId": "", "browser": "Chrome"},
               {"landingPageId": "example.com/page0", "referrerId": "ref5.com", "browser": "Safari"}]
    want = rr.predict(forest, np.array([ref.query_features(maps, q["landingPageId"], q["referrerId"], q["browser"])
                                        for q in queries]))
    server = w.deploy(inst.id)
    got = [server.query(q) for q in queries]
    assert got == [{"score": float(v)} for v in want]
    (tmp_path / "in.json").write_text("\n".join(json.dumps(q) for q in queries) + "\n")
    out = tmp_path / "out.json"
    assert w.BatchPredict.main(["--input", str(tmp_path / "in.json"), "--output", str(out),
                                "--engine-instance-id", inst.id]) == len(queries)
    lines = [json.loads(x) for x in out.read_text().splitlines()]
    assert [x["prediction"] for x in lines] == got and [x["query"] for x in lines] == queries
