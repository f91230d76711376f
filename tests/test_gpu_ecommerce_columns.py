"""GPU: the ecommerce engine's batches, trained from a seeded shop event file of a few thousand items with many cold
users and weights of 0, -1 and 50: predictMany equals predict query by query with all three branches taken, also when a
NaN weight sends the popularity rows to the host rule and when the weights change between calls; predictManyColumns
holds what predictMany returns; and batchpredict writes the same bytes on the column path as on the object path."""
import datetime as dt
import json

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

N_USERS, N_ITEMS, N_NEW = 300, 3000, 40


def _shop_events(seed=21):
    t0 = dt.datetime(2021, 1, 1, tzinfo=dt.timezone.utc)
    at = lambda s: (t0 + dt.timedelta(seconds=int(s))).isoformat()   # noqa: E731
    rng = np.random.default_rng(seed)
    evs = [dict(event="$set", entityType="user", entityId=f"u{k}", eventTime=at(0)) for k in range(N_USERS + 200)]
    evs += [dict(event="$set", entityType="item", entityId=f"i{k}", eventTime=at(0),
                 properties={"categories": ["c%d" % (k % 5)] + (["c9"] if k % 7 == 0 else [])}) for k in range(N_ITEMS)]
    for _ in range(6000):     # users u300 .. u499 are known to the model but own no factor: cold
        evs.append(dict(event="rate", entityType="user", entityId=f"u{rng.integers(N_USERS)}", targetEntityType="item",
                        targetEntityId=f"i{rng.integers(N_ITEMS)}", properties={"rating": float(rng.integers(1, 6))},
                        eventTime=at(rng.integers(0, 100000))))
    for e in range(1500):     # buys of few items: most items score 0, so the popularity rule is mostly ties
        evs.append(dict(event="buy", entityType="user", entityId=f"u{rng.integers(N_USERS)}", targetEntityType="item",
                        targetEntityId=f"i{rng.integers(400)}", eventTime=at(e)))
    for k in range(N_NEW):    # users the model does not know, with recent views: the predictSimilar branch
        for _ in range(3):
            evs.append(dict(event="view", entityType="user", entityId=f"new{k}", targetEntityType="item",
                            targetEntityId=f"i{rng.integers(N_ITEMS)}", eventTime=at(200000 + k)))
    evs.append(dict(event="$set", entityType="constraint", entityId="unavailableItems", eventTime=at(300000),
                    properties={"items": ["i3", "i4", "i999999"]}))
    evs.append(dict(event="$set", entityType="constraint", entityId="weightedItems", eventTime=at(300000),
                    properties={"weights": [{"items": [f"i{k}" for k in range(0, 600, 5)], "weight": 0.0},
                                            {"items": [f"i{k}" for k in range(1, 3000, 4)], "weight": -1.0},
                                            {"items": [f"i{k}" for k in range(2, 400, 9)], "weight": 50.0}]}))
    return evs


def _variant():
    return {"id": "default", "engineFactory": "pio_b200.templates.ecommerce.ECommerceRecommendationEngine",
            "datasource": {"params": {"appName": "Shop"}},
            "algorithms": [{"name": "ecomm", "params": {
                "appName": "Shop", "unseenOnly": True, "seenEvents": ["buy"], "similarEvents": ["view"], "rank": 8,
                "numIterations": 4, "lambda": 0.05, "seed": 3}}]}


def _pick(rng, lo, hi):
    xs = [f"i{x}" for x in rng.integers(0, N_ITEMS, rng.integers(lo, hi))]
    return xs + (["nope"] if rng.random() < 0.3 else [])


def _queries(rng, n):
    from pio_b200.templates import ecommerce as ec
    cats = [None, None, None, {"c0"}, {"c1", "c9"}, {"zz"}, set()]
    qs = []
    for j in range(n):
        kind = int(rng.choice([0, 1, 2, 2, 3, 3]))    # known, recent views, cold known to the model, cold unknown
        user = [f"u{rng.integers(0, N_USERS)}", f"new{rng.integers(0, N_NEW)}", f"u{rng.integers(N_USERS, N_USERS + 200)}",
                f"ghost{j}"][kind]
        num = int(rng.choice([0, 1, 4, 10, 33, 70, 5000]))
        if num == 0 and kind < 3:   # predict takes num < 1 only from users of the popularity rule
            num = 1
        qs.append(ec.Query(user=user, num=num,
                           categories=cats[rng.integers(0, len(cats))],
                           whiteList=None if rng.random() < 0.8 else set(_pick(rng, 0, 60)),
                           blackList=None if rng.random() < 0.5 else set(_pick(rng, 0, 40))))
    return qs


def _exact(p):
    """A PredictedResult as (item, repr(score)) pairs: -0.0 and NaN compare as themselves."""
    return [(s.item, repr(s.score)) for s in p.itemScores]


@pytest.fixture(scope="module")
def shop(tmp_path_factory):
    from pio_b200 import storage as s
    from pio_b200 import workflow as w
    tmp = tmp_path_factory.mktemp("shop")
    mp = pytest.MonkeyPatch()
    mp.setenv("PIO_EVENTDATA_DIR", str(tmp / "events"))
    mp.setenv("PIO_MODELDATA_DIR", str(tmp / "models"))
    s.import_events("Shop", _shop_events())
    variant = tmp / "engine.json"
    variant.write_text(json.dumps(_variant()))
    inst = w.CreateWorkflow.main(["--engine-id", "shop", "--engine-version", "1", "--engine-variant", str(variant)])
    yield tmp, inst, w.deploy(inst.id)
    mp.undo()


def _branches(model, qs):
    out = {"known": 0, "similar": 0, "default": 0}
    for q in qs:
        u = model.userStringIntMap.get(q.user)
        out["known" if u is not None and model.mf.userHas[u] else "similar" if q.user.startswith("new") else
            "default"] += 1
    return out


def test_predict_many_equals_predict(shop):
    _, _, server = shop
    algo, model = server.algorithms[0], server.models[0]
    qs = _queries(np.random.default_rng(22), 500)
    many = algo.predictMany(model, qs)
    each = [algo.predict(model, q) for q in qs]
    assert [_exact(p) for p in many] == [_exact(p) for p in each]
    assert all(_branches(model, qs).values())
    default = [p for q, p in zip(qs, each) if q.user.startswith("ghost") and q.num > 0]
    assert any(len(p.itemScores) > 100 for p in default)                     # a num past the candidates
    scores = [s.score for p in default for s in p.itemScores]
    assert any(s > 0 for s in scores) and any(s < 0 for s in scores)
    assert any(s == 0 and np.signbit(s) for s in scores)                     # 0 buys x weight -1: -0.0
    assert any(s == 0 and not np.signbit(s) for s in scores)
    assert model.__dict__.get("_popular_model") is not None
    assert algo.predictMany(model, []) == []


def test_nan_weight_and_changed_weights(shop, monkeypatch):
    _, _, server = shop
    algo, model = server.algorithms[0], server.models[0]
    from pio_b200.templates import ecommerce as ec
    qs = [q for q in _queries(np.random.default_rng(23), 300) if q.user.startswith("ghost")]
    qs.append(ec.Query(user="ghost-all", num=N_ITEMS + 1))                        # every item, NaN scores included
    groups = algo.weightedItems()
    for changed in (groups + [{"items": ["i7", "i8"], "weight": float("nan")}],       # a NaN weight: the host rule
                    groups + [{"items": ["i2999"], "weight": float("inf")}],          # 0 buys x inf: NaN
                    groups + [{"items": [f"i{k}" for k in range(20, 40)], "weight": 3.0}]):   # new weights: a new model
        monkeypatch.setattr(algo, "weightedItems", lambda g=changed: g)
        before = model.__dict__.get("_popular_model")
        many = algo.predictMany(model, qs)
        assert [_exact(p) for p in many] == [_exact(algo.predict(model, q)) for q in qs]
        after = model.__dict__.get("_popular_model")
        nan = any(g["weight"] != g["weight"] or g["weight"] == float("inf") for g in changed)
        assert (after is before) == nan
        if nan:
            assert any(s.score != s.score for p in many for s in p.itemScores)


def test_predict_many_columns_hold_predict_many(shop):
    from pio_b200 import native
    _, _, server = shop
    algo, model = server.algorithms[0], server.models[0]
    qs = _queries(np.random.default_rng(24), 400)
    many = algo.predictMany(model, qs)
    cols = algo.predictManyColumns(model, qs)
    assert isinstance(cols, native.ScoredColumns) and cols.scores.dtype == np.float64
    assert set(cols.objects) == {j for j, q in enumerate(qs) if q.num < 1}
    assert cols.objects
    for j, p in enumerate(many):
        if j in cols.objects:
            assert _exact(cols.objects[j]) == _exact(p)
            continue
        n = int(cols.count[j])
        got = [(cols.names[i], repr(s)) for i, s in zip(cols.items[j, :n].tolist(), cols.scores[j, :n].tolist())]
        assert got == _exact(p)
        assert (cols.items[j, n:] == -1).all() and (cols.scores[j, n:] == 0).all()
    assert algo.predictManyColumns(model, qs).names is cols.names                     # cached on the model


def test_batch_predict_column_path_writes_the_object_path_bytes(shop, monkeypatch):
    from pio_b200 import workflow as w
    from pio_b200.workflow import to_json
    tmp, inst, server = shop
    assert w.BatchPredict.columnar(server)
    qs = _queries(np.random.default_rng(25), 400)
    (tmp / "in.json").write_text("\n".join(json.dumps(to_json(q)) for q in qs) + "\n")
    args = ["--input", str(tmp / "in.json"), "--engine-instance-id", inst.id, "--query-chunk", "64"]
    assert w.BatchPredict.main(args + ["--output", str(tmp / "columns.json")]) == len(qs)
    monkeypatch.setattr(w.BatchPredict, "columnar", staticmethod(lambda server: False))
    assert w.BatchPredict.main(args + ["--output", str(tmp / "objects.json")]) == len(qs)
    columns, objects = (tmp / "columns.json").read_bytes(), (tmp / "objects.json").read_bytes()
    assert columns == objects and b"-0.0" in columns
