"""GPU tests (-m gpu) of pio_als_rank_lists and the product ranking template (templates/productranking.py).

The device ranking equals the restatement tests/productranking_ref.rank_lists byte for byte -- positions, score bytes
and ranked flags -- at list lengths around the warp and the tile, on the radix path, at every padded rank, on trained
(degree-permuted), loaded and imported handles, with unknown ids, factor-less rows, ties, NaN and infinities, and at
budgets that split a batch into parts.  The doc's engine.json runs end to end through CreateWorkflow, deploy, predict,
predictMany and BatchPredict."""
import ctypes as C
import datetime as dt
import json

import numpy as np
import pytest

from pio_b200 import native
from pio_b200 import storage as s
from pio_b200 import workflow as w
from pio_b200.mllib import ALS
from tests import productranking_ref as ref

pytestmark = pytest.mark.gpu

T = ref.TILE
LENGTHS = (0, 1, 31, 32, 33, T - 1, T, T + 1, 1 << 17)


def _bits(a):
    return np.asarray(a, np.float64).view(np.uint64)


def _batch(rng, n_users, n_items, lengths, unknown=0.1):
    """users and lists of the given lengths, with a share of unknown and out-of-range ids and repeats"""
    users = rng.integers(0, n_users, len(lengths)).astype(np.int32)
    bad_u = rng.random(len(lengths)) < unknown
    users[bad_u] = rng.choice([-1, n_users, n_users + 7, -(1 << 31)], int(bad_u.sum()))
    ptr = np.concatenate([[0], np.cumsum(lengths)]).astype(np.int64)
    items = rng.integers(0, n_items, int(ptr[-1])).astype(np.int32)
    bad_i = rng.random(items.shape[0]) < unknown
    items[bad_i] = rng.choice([-1, n_items, (1 << 31) - 1], int(bad_i.sum()))
    return users, ptr, items


def _check(h, factors, users, ptr, items):
    uf, itf, uh, ih = factors
    pos, sc, ranked = h.rank_lists(users, ptr, items)
    wp, ws, wr = ref.rank_lists(uf, uh, itf, ih, users, ptr, items)
    assert np.array_equal(ranked, wr)
    assert np.array_equal(pos, wp)
    assert np.array_equal(_bits(sc), _bits(ws))
    return pos, sc, ranked


def _imported(rng, nu, ni, rank, has=0.9, levels=None):
    """random factors (a few levels when `levels`: ties everywhere), some rows without a factor"""
    if levels:
        uf = (rng.integers(-levels, levels + 1, (nu, rank)) * 0.25).astype(np.float32)
        itf = (rng.integers(-levels, levels + 1, (ni, rank)) * 0.5).astype(np.float32)
    else:
        uf = rng.standard_normal((nu, rank)).astype(np.float32)
        itf = rng.standard_normal((ni, rank)).astype(np.float32)
    uh = (rng.random(nu) < has).astype(np.uint8)
    ih = (rng.random(ni) < has).astype(np.uint8)
    return native.NativeALS.from_factors(uf, itf, uh, ih), (uf, itf, uh, ih)


def test_list_lengths_and_both_paths():
    rng = np.random.default_rng(1)
    h, f = _imported(rng, 300, 5000, 64)
    for n in LENGTHS:
        users, ptr, items = _batch(rng, 300, 5000, [n] * 3)
        _check(h, f, users, ptr, items)
    users, ptr, items = _batch(rng, 300, 5000, list(LENGTHS) * 2 + [7] * 500)
    _check(h, f, users, ptr, items)
    st = native.rank_lists_stats()
    assert st["radix_queries"] == 2 * 2 and st["tile_queries"] == 2 * 6 + 500 and st["parts"] == 1
    assert st["entries"] == int(ptr[-1]) and st["device_ms"] > 0
    h.close()


@pytest.mark.parametrize("rank", [1, 10, 32, 64, 65, 128])
def test_ranks(rank):
    rng = np.random.default_rng(rank)
    h, f = _imported(rng, 200, 3000, rank)
    users, ptr, items = _batch(rng, 200, 3000, [0, 1, 5, 33, T - 1, T + 1, 200, 3 * T] + [40] * 100)
    _check(h, f, users, ptr, items)
    h.close()


def test_tie_heavy_factors():
    rng = np.random.default_rng(2)
    h, f = _imported(rng, 50, 400, 4, has=0.7, levels=1)
    users, ptr, items = _batch(rng, 50, 400, [int(x) for x in rng.integers(0, 3 * T, 40)], unknown=0.2)
    pos, sc, _ = _check(h, f, users, ptr, items)
    assert (np.diff(sc) == 0).mean() > 0.5        # the order of most entries is decided by the position
    h.close()


def test_all_unknown_and_factorless():
    rng = np.random.default_rng(3)
    h, f = _imported(rng, 20, 100, 8, has=0.5)
    uh, ih = f[2], f[3]
    no_u, u = int(np.flatnonzero(uh == 0)[0]), int(np.flatnonzero(uh)[0])
    no_i = np.flatnonzero(ih == 0).astype(np.int32)
    lists = [(u, [-1, 100, 5000]), (u, no_i.tolist()), (no_u, list(range(100))), (99, [0, 1]), (u, []),
             (u, np.tile(no_i, T // len(no_i) + 2).tolist())]
    users = np.array([x for x, _ in lists], np.int32)
    ptr = np.concatenate([[0], np.cumsum([len(x) for _, x in lists])]).astype(np.int64)
    items = np.array([i for _, x in lists for i in x], np.int32)
    pos, sc, ranked = _check(h, f, users, ptr, items)
    assert not ranked.any() and not sc.any()
    assert np.array_equal(pos, np.concatenate([np.arange(len(x)) for _, x in lists]).astype(np.int32))
    h.close()


def test_nan_and_infinities_from_imported_factors():
    rng = np.random.default_rng(4)
    uf = rng.standard_normal((30, 16)).astype(np.float32)
    itf = rng.standard_normal((500, 16)).astype(np.float32)
    uf[::5, 3] = np.inf
    uf[1::7, 0] = -np.inf
    itf[::3, 3] = 0.0                        # inf * 0: NaN
    itf[::11, 0] = -np.inf
    itf[::13, 5] = np.nan
    uh, ih = np.ones(30, np.uint8), np.ones(500, np.uint8)
    h = native.NativeALS.from_factors(uf, itf, uh, ih)
    users, ptr, items = _batch(rng, 30, 500, [0, 9, 100, T, T + 3, 4 * T], unknown=0.05)
    _, sc, _ = _check(h, (uf, itf, uh, ih), users, ptr, items)
    assert np.isnan(sc).any() and np.isposinf(sc).any() and np.isneginf(sc).any()
    h.close()


def _trained(rng, nu=400, ni=250, rank=10):
    """a trained handle whose rows are degree-permuted; the last users and items have no rating"""
    u = rng.integers(0, nu - 20, 6000).astype(np.int32)
    i = np.minimum(rng.zipf(1.5, 6000), ni - 10).astype(np.int32) - 1
    m = ALS.trainImplicit((u, i, np.ones(6000, np.float32)), rank=rank, iterations=3, lambda_=0.01, seed=7,
                          dedup="sum", n_users=nu, n_products=ni)
    return m


def test_trained_and_loaded_handles(tmp_path):
    rng = np.random.default_rng(5)
    m = _trained(rng)
    f = (m.userFeatures, m.productFeatures, m.userHas, m.productHas)
    assert not m.userHas.all() and not m.productHas.all()
    users, ptr, items = _batch(rng, 400, 250, [0, 3, 250, T + 5, 17] * 20)
    want = _check(m._handle(), f, users, ptr, items)
    m.save(str(tmp_path / "m.pioals"))
    h = native.NativeALS.load(str(tmp_path / "m.pioals"))
    got = h.rank_lists(users, ptr, items)
    assert all(np.array_equal(np.asarray(a).view(np.uint8), np.asarray(b).view(np.uint8)) for a, b in zip(got, want))
    h.close()


def test_recommend_cross_check():
    rng = np.random.default_rng(6)
    m = _trained(rng)
    h = m._handle()
    k = 20
    for u in np.flatnonzero(m.userHas)[:5]:
        lst = np.flatnonzero(m.productHas).astype(np.int32)
        pos, sc, ranked = h.rank_lists(np.array([u], np.int32), np.array([0, lst.shape[0]], np.int64), lst)
        items, scores, cnt = h.recommend(np.array([u], np.int32), k)
        assert ranked[0] and cnt[0] == k
        assert np.array_equal(lst[pos[:k]], items[0]) and np.array_equal(sc[:k].astype(np.float32), scores[0])


@pytest.mark.parametrize("budget,parts", [(100, 1), (200, 2), (300, 3)])
def test_budget_parts(monkeypatch, budget, parts):
    rng = np.random.default_rng(7)
    h, f = _imported(rng, 100, 1000, 32)
    lens = [100] * 12 + [5000, 0, 3]
    monkeypatch.setenv("PIO_RANK_LISTS_BUDGET", str(budget))
    users, ptr, items = _batch(rng, 100, 1000, lens)
    _check(h, f, users, ptr, items)
    st = native.rank_lists_stats()
    assert st["parts"] == len(ref.plan(ptr, budget)) and st["max_part_entries"] == 5000
    # every part of the twelve 100-entry queries holds `parts` queries
    assert [p["q1"] - p["q0"] for p in ref.plan(ptr, budget)][:12 // parts] == [parts] * (12 // parts)
    h.close()


def test_argument_rejections_before_device_work():
    rng = np.random.default_rng(8)
    h, _ = _imported(rng, 10, 10, 4)
    L = native.lib()
    u = np.zeros(2, np.int32)
    it = np.zeros(4, np.int32)
    pos, sc, rk = np.zeros(4, np.int32), np.zeros(4), np.zeros(2, np.uint8)
    before = h.stats()["kernel_launches"]

    def call(users, n, ptr, items, p=pos, s_=sc, r=rk, handle=None):
        return L.pio_als_rank_lists(h._h if handle is None else handle, native._addr(users), n, native._addr(ptr),
                                    native._addr(items), native._addr(p), native._addr(s_), native._addr(r))
    good = np.array([0, 2, 4], np.int64)
    assert call(u, -1, good, it) == native.ERR_ARG
    assert call(u, 2, np.array([1, 2, 4], np.int64), it) == native.ERR_ARG
    assert call(u, 2, np.array([0, 3, 2], np.int64), it) == native.ERR_ARG
    assert call(u, 2, np.array([0, 1 << 31, (1 << 31) + 1], np.int64), it) == native.ERR_ARG
    assert call(u, 2, good, it, p=None) == native.ERR_ARG
    assert call(u, 2, good, it, s_=None) == native.ERR_ARG
    assert call(u, 2, good, it, r=None) == native.ERR_ARG
    assert call(u, 2, good, it, handle=C.c_void_p()) == native.ERR_ARG
    assert h.stats()["kernel_launches"] == before
    assert call(u, 0, np.zeros(1, np.int64), it) == 0
    assert call(u, 2, good, it) == 0
    h.close()


# ---- the template end to end ------------------------------------------------------------------------------------------
DOC_ALGO = {"rank": 10, "numIterations": 20, "lambda": 0.01, "seed": 3}


def _events(seed, nu=60, ni=40):
    rng = np.random.default_rng(seed)
    t0 = dt.datetime(2021, 1, 1, tzinfo=dt.timezone.utc)
    at = lambda k: (t0 + dt.timedelta(seconds=k)).isoformat()   # noqa: E731
    evs = [dict(event="$set", entityType="user", entityId=f"u{k}", eventTime=at(0)) for k in range(nu)]
    evs += [dict(event="$set", entityType="item", entityId=f"i{k}", eventTime=at(0),
                 properties={"categories": ["c"]}) for k in range(ni)]
    for e in range(1500):    # repeated pairs; items i35.. are set but never viewed
        evs.append(dict(event="view", entityType="user", entityId=f"u{rng.integers(nu)}", targetEntityType="item",
                        targetEntityId=f"i{rng.integers(ni - 5)}", eventTime=at(e + 1)))
    evs.append(dict(event="view", entityType="user", entityId="ghost", targetEntityType="item", targetEntityId="i1",
                    eventTime=at(2000)))       # a user without $set
    evs.append(dict(event="view", entityType="user", entityId="u1", targetEntityType="item", targetEntityId="phantom",
                    eventTime=at(2001)))       # an item without $set
    return evs


def test_template_end_to_end(tmp_path, monkeypatch):
    monkeypatch.setenv("PIO_EVENTDATA_DIR", str(tmp_path / "events"))
    monkeypatch.setenv("PIO_MODELDATA_DIR", str(tmp_path / "models"))
    from pio_b200.templates import productranking as pr
    evs = _events(9)
    s.import_events("MyApp1", evs)
    variant = tmp_path / "engine.json"
    variant.write_text(json.dumps({
        "id": "default", "description": "Default settings",
        "engineFactory": "pio_b200.templates.productranking.ProductRankingEngine",
        "datasource": {"params": {"appName": "MyApp1"}},
        "algorithms": [{"name": "als", "params": DOC_ALGO}]}))
    inst = w.CreateWorkflow.main(["--engine-id", "pr", "--engine-version", "1", "--engine-variant", f"file:{variant}"])
    assert inst.status == "COMPLETED"
    server = w.deploy(inst.id)
    model = server.models[0]
    um, im = model.userStringIntMap, model.itemStringIntMap
    # the restated ratings: views of known users and items, summed per pair
    pairs = {}
    for e in evs:
        if e["event"] == "view" and um.get(e["entityId"]) is not None and im.get(e["targetEntityId"]) is not None:
            key = (um(e["entityId"]), im(e["targetEntityId"]))
            pairs[key] = pairs.get(key, 0) + 1
    u = np.array([k[0] for k in pairs], np.int32)
    i = np.array([k[1] for k in pairs], np.int32)
    r = np.array(list(pairs.values()), np.float32)
    direct = ALS.trainImplicit((u, i, r), rank=10, iterations=20, lambda_=0.01, blocks=-1, alpha=1.0, seed=3,
                               n_users=um.size, n_products=im.size)
    mf = model.mf
    assert um.size == 60 and im.size == 40 and not mf.productHas[im("i39")]
    assert np.array_equal(mf.userFeatures, direct.userFeatures) and np.array_equal(mf.productFeatures,
                                                                                  direct.productFeatures)
    f = (mf.userFeatures, mf.productFeatures, mf.userHas, mf.productHas)
    queries = [{"user": "u2", "items": ["i1", "i3", "i10", "i2", "i5", "i31", "i9"]},
               {"user": "u2", "items": ["i1", "i3", "i1", "nope", "i39", "i0"]},
               {"user": "ghost", "items": ["i1", "i2"]},
               {"user": "u3", "items": ["i39", "nope"]},
               {"user": "u4", "items": []}]
    want = []
    for q in queries:
        ids = [im.getOrElse(x, -1) for x in q["items"]]
        pos, sc, orig = ref.predict_literal(*[f[k] for k in (0, 2, 1, 3)], um.getOrElse(q["user"], -1), ids)
        want.append({"itemScores": [{"item": q["items"][p], "score": v} for p, v in zip(pos, sc)],
                     "isOriginal": orig})
    got = [server.query(q) for q in queries]
    assert got == want
    assert [g["isOriginal"] for g in got] == [False, False, True, True, True]
    algo = server.algorithms[0]
    qs = [pr.Query(**q) for q in queries] * 3
    assert algo.predictMany(model, qs) == [algo.predict(model, q) for q in qs]
    (tmp_path / "in.json").write_text("\n".join(json.dumps(q) for q in queries) + "\n")
    out = tmp_path / "out.json"
    assert w.BatchPredict.main(["--input", str(tmp_path / "in.json"), "--output", str(out),
                                "--engine-instance-id", inst.id]) == len(queries)
    lines = out.read_text().splitlines()
    assert lines == [json.dumps({"query": q, "prediction": w.to_json(algo.predict(model, pr.Query(**q)))},
                                separators=(",", ":")) for q in queries]
