"""GPU: predictMany of the recommendation and similarproduct templates equals their predict, query by query, over seeded
queries that mix every filter field, unknown users and items, and differing `num`."""
import numpy as np
import pytest

pytestmark = pytest.mark.gpu

N_USERS, N_ITEMS, RANK = 60, 500, 10
CATS = ["c0", "c1", "c2", "c3"]


@pytest.fixture(scope="module")
def mf():
    from pio_b200 import native
    from pio_b200.mllib import MatrixFactorizationModel
    native.build()
    rng = np.random.default_rng(3)
    uf = rng.standard_normal((N_USERS, RANK)).astype(np.float32)
    itf = rng.standard_normal((N_ITEMS, RANK)).astype(np.float32)
    uh, ih = np.ones(N_USERS, np.uint8), np.ones(N_ITEMS, np.uint8)
    uh[[4, 9]] = 0
    ih[rng.choice(N_ITEMS, 25, replace=False)] = 0
    uf[uh == 0] = 0
    itf[ih == 0] = 0
    h = native.NativeALS.from_factors(uf, itf, uh, ih)
    yield MatrixFactorizationModel(RANK, uf, itf, uh, ih, h)
    h.close()


def _pick(rng, pool, lo, hi, unknown):
    xs = [str(x) for x in rng.choice(pool, rng.integers(lo, hi), replace=False)]
    return xs + ([unknown] if rng.random() < 0.3 else [])


def test_recommendation_predict_many_equals_predict(mf):
    from pio_b200.storage import BiMap
    from pio_b200.templates import recommendation as rec
    model = rec.ALSModel(mf, BiMap({f"u{u}": u for u in range(N_USERS)}), BiMap({f"i{i}": i for i in range(N_ITEMS)}))
    algo = rec.ALSAlgorithm(rec.ALSAlgorithmParams(rank=RANK, numIterations=1, lambda_=0.01, seed=1))
    rng = np.random.default_rng(4)
    items = [f"i{i}" for i in range(N_ITEMS)]
    qs = []
    for j in range(300):
        user = f"u{rng.integers(0, N_USERS + 5)}"            # some users are unknown, two own no factor
        black = None if j % 4 == 0 else [] if j % 4 == 1 else _pick(rng, items, 1, 40, "nope")
        qs.append(rec.Query(user=user, num=int(rng.choice([1, 4, 10, 40])), blackList=black))
    many = algo.predictMany(model, qs)
    assert many == [algo.predict(model, q) for q in qs]
    assert any(p.itemScores for p in many) and any(not p.itemScores for p in many)
    algo.predictMany(model, qs)
    assert "filtered" in mf._handle().stats()["last_score_path"]
    assert algo.predictMany(model, []) == [] and algo.predictMany(model, [rec.Query(user="ghost", num=3)]) == [rec.PredictedResult([])]


@pytest.mark.parametrize("algo_name", ["ALSAlgorithm", "LikeAlgorithm"])
def test_similarproduct_predict_many_equals_predict(mf, algo_name):
    from pio_b200.storage import BiMap
    from pio_b200.templates import similarproduct as sp
    rng = np.random.default_rng(6)
    props = {}
    for i in range(N_ITEMS):
        r = rng.random()
        if r >= 0.05:
            props[i] = sp.Item(categories=None if r < 0.15 else list(rng.choice(CATS, rng.integers(1, 3), replace=False)))
    model = sp.ALSModel(mf, BiMap({f"i{i}": i for i in range(N_ITEMS)}), props)
    algo = getattr(sp, algo_name)(sp.ALSAlgorithmParams(rank=RANK, numIterations=1, lambda_=0.01, seed=1))
    items = [f"i{i}" for i in range(N_ITEMS)]
    cat_rules = [None, None, ["c0"], ["c1", "c3"], ["zz"], []]
    qs = []
    for j in range(300):
        q_items = _pick(rng, items, 1, 5, "nope") if j % 11 else ["nope", "nada"]
        qs.append(sp.Query(items=q_items, num=int(rng.choice([1, 5, 10, 40])),
                           categories=cat_rules[rng.integers(0, len(cat_rules))],
                           categoryBlackList=cat_rules[rng.integers(0, len(cat_rules))],
                           whiteList=None if rng.random() < 0.7 else _pick(rng, items, 0, 80, "nope"),
                           blackList=None if rng.random() < 0.5 else _pick(rng, items, 0, 30, "nope")))
    many = algo.predictMany(model, qs)
    assert many == [algo.predict(model, q) for q in qs]
    assert any(p.itemScores for p in many) and any(not p.itemScores for p in many)
    algo.predictMany(model, qs)
    assert {"filtered", "listed"} <= mf._handle().stats()["last_score_path"]


# ---- templates trained from a seeded event file, and the batchpredict workflow ------------------------------------------
def _shop_events(nu=120, ni=60, seed=5):
    import datetime as dt
    t0 = dt.datetime(2021, 1, 1, tzinfo=dt.timezone.utc)
    rng = np.random.default_rng(seed)
    evs = [dict(event="$set", entityType="user", entityId=f"u{k}", eventTime=t0.isoformat()) for k in range(nu)]
    evs += [dict(event="$set", entityType="item", entityId=f"i{k}", eventTime=t0.isoformat(),
                 properties={"categories": ["c%d" % (k % 3)] + (["c9"] if k % 7 == 0 else [])}) for k in range(ni)]
    for e in range(3000):
        evs.append(dict(event="rate", entityType="user", entityId=f"u{rng.integers(nu)}", targetEntityType="item",
                        targetEntityId=f"i{rng.integers(ni)}", properties={"rating": float(rng.integers(1, 6))},
                        eventTime=(t0 + dt.timedelta(seconds=int(rng.integers(0, 100000)))).isoformat()))
    for e in range(400):
        evs.append(dict(event="buy", entityType="user", entityId=f"u{rng.integers(nu)}", targetEntityType="item",
                        targetEntityId=f"i{rng.integers(ni)}", eventTime=(t0 + dt.timedelta(seconds=e)).isoformat()))
    for k in range(12):       # users the model does not know, with recent views: the predictSimilar branch
        for _ in range(3):
            evs.append(dict(event="view", entityType="user", entityId=f"new{k}", targetEntityType="item",
                            targetEntityId=f"i{rng.integers(ni)}", eventTime=(t0 + dt.timedelta(days=2, seconds=k)).isoformat()))
    evs.append(dict(event="$set", entityType="constraint", entityId="unavailableItems",
                    eventTime=(t0 + dt.timedelta(days=3)).isoformat(), properties={"items": ["i3", "i4", "i999"]}))
    evs.append(dict(event="$set", entityType="constraint", entityId="weightedItems",
                    eventTime=(t0 + dt.timedelta(days=3)).isoformat(),
                    properties={"weights": [{"items": ["i5", "i6"], "weight": 0.0}, {"items": ["i7"], "weight": 50.0},
                                            {"items": ["i8"], "weight": -1.0}]}))
    return evs


def _ecomm_variant(unseen_only):
    return {"id": "default", "engineFactory": "pio_b200.templates.ecommerce.ECommerceRecommendationEngine",
            "datasource": {"params": {"appName": "Shop"}},
            "algorithms": [{"name": "ecomm", "params": {
                "appName": "Shop", "unseenOnly": unseen_only, "seenEvents": ["buy"], "similarEvents": ["view"], "rank": 8,
                "numIterations": 4, "lambda": 0.05, "seed": 3}}]}


def _ecomm_queries(rng, n):
    from pio_b200.templates import ecommerce as ec
    items = [f"i{k}" for k in range(60)]
    cats = [None, None, {"c0"}, {"c1", "c9"}, {"zz"}, set()]
    qs = []
    for j in range(n):
        user = [f"u{rng.integers(0, 120)}", f"new{rng.integers(0, 12)}", f"ghost{j}"][int(rng.choice([0, 0, 0, 1, 2]))]
        qs.append(ec.Query(user=user, num=int(rng.choice([1, 4, 10, 70])), categories=cats[rng.integers(0, len(cats))],
                           whiteList=None if rng.random() < 0.7 else set(_pick(rng, items, 0, 30, "nope")),
                           blackList=None if rng.random() < 0.5 else set(_pick(rng, items, 0, 20, "nope"))))
    return qs


@pytest.mark.parametrize("unseen_only", [True, False])
def test_ecommerce_predict_many_equals_predict(tmp_path, monkeypatch, unseen_only):
    import json
    from pio_b200 import storage as s
    from pio_b200 import workflow as w
    monkeypatch.setenv("PIO_EVENTDATA_DIR", str(tmp_path / "events"))
    monkeypatch.setenv("PIO_MODELDATA_DIR", str(tmp_path / "models"))
    s.import_events("Shop", _shop_events())
    variant = tmp_path / "engine.json"
    variant.write_text(json.dumps(_ecomm_variant(unseen_only)))
    inst = w.CreateWorkflow.main(["--engine-id", "shop", "--engine-version", "1", "--engine-variant", str(variant)])
    server = w.deploy(inst.id)
    algo, model = server.algorithms[0], server.models[0]
    qs = _ecomm_queries(np.random.default_rng(9), 300)
    many = algo.predictMany(model, qs)
    each = [algo.predict(model, q) for q in qs]
    assert many == each
    branch = {"known": 0, "similar": 0, "default": 0}
    for q, p in zip(qs, each):
        branch["known" if q.user.startswith("u") else "similar" if q.user.startswith("new") else "default"] += 1
    assert all(branch.values()), branch                                   # all three branches were taken
    assert any(p.itemScores for q, p in zip(qs, each) if q.user.startswith("new"))
    for p in each:                                                        # unavailableItems and zero weights hold
        assert not {"i3", "i4"} & {x.item for x in p.itemScores}
    # a batch of known users only, then the path of the last device call
    algo.predictMany(model, [q for q in qs if q.user.startswith("u")])
    assert {"filtered", "listed"} & model.mf._handle().stats()["last_score_path"]


def test_batch_predict_writes_what_the_deployed_engine_answers(tmp_path, monkeypatch):
    import json
    from pio_b200 import storage as s
    from pio_b200 import workflow as w
    from pio_b200.workflow import to_json
    monkeypatch.setenv("PIO_EVENTDATA_DIR", str(tmp_path / "events"))
    monkeypatch.setenv("PIO_MODELDATA_DIR", str(tmp_path / "models"))
    s.import_events("Shop", _shop_events())
    variant = tmp_path / "engine.json"
    variant.write_text(json.dumps(_ecomm_variant(True)))
    inst = w.CreateWorkflow.main(["--engine-id", "shop", "--engine-version", "1", "--engine-variant", str(variant)])
    qjs = [to_json(q) for q in _ecomm_queries(np.random.default_rng(10), 120)]
    qjs[3] = {"user": "u1", "num": 4}                                     # optional fields left out
    lines = []
    for j, qj in enumerate(qjs):
        lines.append(json.dumps(qj))
        if j % 9 == 0:
            lines += ["", "   \t "]
    (tmp_path / "in.json").write_text("\n".join(lines) + "\n\n")
    out = tmp_path / "out.json"
    for args in (["--engine-instance-id", inst.id, "--query-partitions", "4", "--query-chunk", "50"],
                 ["--engine-id", "shop", "--engine-version", "1"]):
        n = w.BatchPredict.main(["--input", str(tmp_path / "in.json"), "--output", str(out)] + args)
        written = out.read_text().splitlines()
        assert n == len(qjs) == len(written)
        server = w.deploy(inst.id)
        for qj, line in zip(qjs, written):
            rec = json.loads(line)
            assert set(rec) == {"query", "prediction"} and ": " not in line
            assert rec["query"]["user"] == qj["user"] and rec["query"]["num"] == qj["num"]
            assert rec["prediction"] == server.query(qj)
