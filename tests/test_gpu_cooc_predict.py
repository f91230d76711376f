"""GPU: pio_cooc_predict_filtered equals the restatement (cooc_predict_ref.py) exactly at its boundaries -- empty batches
and queries, items without a list, the first and last item ids, empty white lists, shared set rows, ties, sums past
2^31 and 2^32, topk around the candidate count, and parts of one, two and three queries -- with stats() showing the part
counts reached; CooccurrenceAlgorithm.predictMany equals predict on a model trained from an event file; and batchpredict
over an engine with als and cooccurrence writes what the deployed engine answers."""
import datetime as dt
import json
import pickle

import numpy as np
import pytest

import cooc_predict_ref as ref

pytestmark = pytest.mark.gpu

N_ITEMS, TOPN = 400, 16


@pytest.fixture(scope="module")
def arrays():
    rng = np.random.default_rng(11)
    ti = np.full((N_ITEMS, TOPN), -1, np.int32)
    tc = np.zeros((N_ITEMS, TOPN), np.int32)
    tn = rng.integers(0, TOPN + 1, N_ITEMS).astype(np.int32)
    tn[[5, 6, 7]] = 0                                    # items with an empty list
    tn[[0, N_ITEMS - 1]] = TOPN
    for i in range(N_ITEMS):
        ti[i, :tn[i]] = rng.permutation(np.delete(np.arange(N_ITEMS), i))[:tn[i]]
        tc[i, :tn[i]] = np.sort(rng.integers(1, 4, tn[i]))[::-1]   # small counts: many ties
    ti[1, :3], tn[1] = [0, N_ITEMS - 1, 2], max(tn[1], 3)            # ids 0 and n_items - 1 as candidates
    return ti, tc, tn


@pytest.fixture(scope="module")
def model(native, arrays):
    m = native.CoocModel(*arrays)
    yield m
    m.close()


def check(native, m, arrays, qls, topk, qf=None, **filt):
    got = m.predict_filtered(qls, topk, qf)
    want = ref.predict(*arrays, qls, topk, **filt)
    for g, w in zip(got, want):
        assert g.dtype == w.dtype and np.array_equal(g, w)
    return got


def test_empty_batch_and_empty_queries(native, model, arrays):
    oi, os_, oc = check(native, model, arrays, [], 5)
    assert oi.shape == (0, 5) and model.stats()["last_parts"] == 0
    oi, os_, oc = check(native, model, arrays, [[], [-1, N_ITEMS, 10 ** 6], [5, 6, 7, 5], []], 5)
    st = model.stats()
    assert not oc.any() and st["last_parts"] == 1 and st["last_expanded"] == 0 and st["last_rows"] == 0


def test_item_range_and_repeats(native, model, arrays):
    qls = [[0], [N_ITEMS - 1], [1], [1, 1, 1, -3], [0, N_ITEMS - 1, 1], [2, 3, 4, 8, 9, 10, 11, 12]]
    oi, os_, oc = check(native, model, arrays, qls, 40)
    assert {0, N_ITEMS - 1} <= set(oi[2].tolist())
    assert model.stats()["last_expanded"] == sum(ref.expansion(arrays[2], np.unique(q[q >= 0]))
                                                 for q in map(np.array, qls))


@pytest.mark.parametrize("topk", [1, "exact", 200])
def test_topk_around_the_candidate_count(native, model, arrays, topk):
    qls = [[3, 4], [9], [20, 21, 22, 23]]
    if topk == "exact":
        _, _, oc = ref.predict(*arrays, qls[:1], 1000)
        topk = int(oc[0])
    oi, os_, oc = check(native, model, arrays, qls, topk)
    assert topk == 1 or any(np.diff(os_[2, :oc[2]]) == 0)   # tied scores, ordered by item


def test_filters(native, model, arrays):
    rng = np.random.default_rng(12)
    n = 60
    qls = [rng.choice(N_ITEMS, rng.integers(1, 6), replace=False).tolist() + ([N_ITEMS + 3] if j % 5 == 0 else [])
           for j in range(n)]
    ex = [None if j % 3 == 0 else rng.choice(N_ITEMS, rng.integers(0, 30)).tolist() + [-1] for j in range(n)]
    wl = [None if j % 4 else [] if j % 8 == 0 else rng.choice(N_ITEMS, rng.integers(1, 150)).tolist() for j in range(n)]
    sets = (rng.random((3, N_ITEMS)) < 0.4).astype(np.uint8)
    six = np.array([[-1, 0, 1, 2][j % 4] for j in range(n)], np.int32)   # rows shared by several queries
    qf = native.QueryFilter(n, ex, wl, six, sets)
    oi, os_, oc = check(native, model, arrays, qls, 12, qf, exclude=ex, white=wl, set_ix=six, item_sets=sets)
    assert oc.any() and not oc[[j for j in range(n) if j % 8 == 0]].any()   # an empty white list: nothing
    qf = native.QueryFilter(n, white=[None] * n)                             # no query has a white list
    check(native, model, arrays, qls, 12, qf)


def test_sums_past_two_to_the_32(native):
    big = 2 ** 31 - 1
    ti = np.array([[3, 4, 5], [3, 4, 5], [3, 5, -1], [0, 1, 2], [0, 1, 2], [0, 1, 2]], np.int32)
    tc = np.array([[big, big, 7], [big, big - 1, 7], [big, 1, 0], [1, 2, 3], [3, 2, 1], [big, 0, 0]], np.int32)
    tn = np.array([3, 3, 2, 3, 3, 1], np.int32)
    m = native.CoocModel(ti, tc, tn)
    try:
        oi, os_, oc = check(native, m, (ti, tc, tn), [[0, 1, 2], [0, 1], [3, 4, 5], [5]], 4)
        assert os_[0, 0] == 3 * big > 2 ** 32 and os_[0, 1] == 2 * big - 1 > 2 ** 31
    finally:
        m.close()


@pytest.mark.parametrize("budget", [1, 40, 75, 10 ** 9])
def test_parts(native, model, arrays, monkeypatch, budget):
    rng = np.random.default_rng(13)
    tn = arrays[2]
    qls = []
    while len(qls) < 30:
        q = rng.choice(N_ITEMS, 3, replace=False)
        if (tn[q] > 0).all() and tn[q].sum() <= 40:     # every query expands to 3 .. 40 entries
            qls.append(q.tolist())
    qls[7] = [0, N_ITEMS - 1, 1, 2, 3]                  # one query over the 40 and 75 budgets
    monkeypatch.setenv("PIO_COOC_PREDICT_BUDGET", str(budget))
    check(native, model, arrays, qls, 10)
    first = ref.parts(tn, qls, budget)
    sizes = np.diff(first + [len(qls)])
    st = model.stats()
    assert st["last_parts"] == len(first) and st["last_max_part_queries"] == sizes.max() and st["last_budget"] == budget
    assert {1: {1}, 40: {1, 2}, 75: {2, 3}, 10 ** 9: {30}}[budget] <= set(sizes.tolist())
    assert budget != 40 or sizes[first.index(7)] == 1   # query 7 expands to 56: a part of its own


def test_rejected_query_leaves_no_part(native):
    topn = 1 << 16
    m = native.CoocModel(np.ones((2, topn), np.int32), np.ones((2, topn), np.int32), np.array([topn, 0], np.int32))
    try:
        with pytest.raises(native.NativeError) as e:
            m.predict_filtered([[1], [0] * topn], 3)
        assert e.value.code == native.ERR_ARG and m.stats()["last_parts"] == 0
        oi, os_, oc = m.predict_filtered([[0, 0, 0]], 3)
        assert oi[0].tolist() == [1, -1, -1] and os_[0].tolist() == [topn, 0, 0] and m.stats()["last_parts"] == 1
    finally:
        m.close()


# ---- the template, trained from an event file ----------------------------------------------------------------------------
def _events(nu=150, ni=70, seed=4):
    t0 = dt.datetime(2021, 1, 1, tzinfo=dt.timezone.utc)
    rng = np.random.default_rng(seed)
    evs = [dict(event="$set", entityType="user", entityId=f"u{k}", eventTime=t0.isoformat()) for k in range(nu)]
    for k in range(ni + 4):                              # four items nobody views; every fifth without categories
        props = {} if k % 5 == 4 else {"categories": ["c%d" % (k % 3)] + (["c9"] if k % 7 == 0 else [])}
        evs.append(dict(event="$set", entityType="item", entityId=f"i{k}", eventTime=t0.isoformat(), properties=props))
    for e in range(2500):
        evs.append(dict(event=["view", "view", "like", "dislike"][e % 4], entityType="user",
                        entityId=f"u{rng.integers(nu)}", targetEntityType="item",
                        targetEntityId=f"i{min(int(rng.random() ** 2 * ni), ni - 1)}",
                        eventTime=(t0 + dt.timedelta(seconds=e)).isoformat()))
    return evs


def _variant():
    return {"id": "default", "engineFactory": "pio_b200.templates.similarproduct.SimilarProductEngine",
            "datasource": {"params": {"appName": "Sim"}},
            "algorithms": [{"name": "als", "params": {"rank": 8, "numIterations": 4, "lambda": 0.01, "seed": 3}},
                           {"name": "cooccurrence", "params": {"n": 12}}]}


def _queries(rng, n):
    from pio_b200.templates import similarproduct as sp
    items = [f"i{k}" for k in range(74)]
    cats = [None, None, {"c0"}, {"c1", "c9"}, {"zz"}, set()]

    def pick(lo, hi):
        return [str(x) for x in rng.choice(items, rng.integers(lo, hi), replace=False)] + (
            ["nope"] if rng.random() < 0.3 else [])
    qs = []
    for j in range(n):
        q_items = pick(1, 5) if j % 11 else ["nope", "nada"]
        qs.append(sp.Query(items=q_items + q_items[:1] * (j % 6 == 0), num=int(rng.choice([1, 4, 10, 70])),
                           categories=cats[rng.integers(0, len(cats))],
                           categoryBlackList=cats[rng.integers(0, len(cats))],
                           whiteList=None if rng.random() < 0.7 else set(pick(0, 30)),
                           blackList=None if rng.random() < 0.5 else set(pick(0, 20))))
    qs.append(sp.Query(items=["i1"], num=0))
    qs.append(sp.Query(items=["i1", "i2"], num=-2))
    return qs


def test_num_far_above_the_item_count(engine):
    """One query with a num no batch could hold rows for: the call is cut at the item count, which no query's candidates
    exceed, and the answers are predict's."""
    from pio_b200 import workflow as w
    from pio_b200.templates import similarproduct as sp
    server = w.deploy(engine.id)
    k = [type(a) for a in server.algorithms].index(sp.CooccurrenceAlgorithm)
    algo, model = server.algorithms[k], server.models[k]
    qs = _queries(np.random.default_rng(9), 40)[:-2] + [sp.Query(items=["i1", "i3"], num=10 ** 9)]
    many = algo.predictMany(model, qs)
    assert many == [algo.predict(model, q) for q in qs] and many[-1].itemScores


@pytest.fixture
def engine(tmp_path, monkeypatch):
    from pio_b200 import storage as s
    from pio_b200 import workflow as w
    monkeypatch.setenv("PIO_EVENTDATA_DIR", str(tmp_path / "events"))
    monkeypatch.setenv("PIO_MODELDATA_DIR", str(tmp_path / "models"))
    s.import_events("Sim", _events())
    variant = tmp_path / "engine.json"
    variant.write_text(json.dumps(_variant()))
    return w.CreateWorkflow.main(["--engine-id", "sim", "--engine-version", "1", "--engine-variant", str(variant)])


def test_predict_many_equals_predict(engine):
    from pio_b200 import workflow as w
    from pio_b200.templates import similarproduct as sp
    server = w.deploy(engine.id)
    k = [type(a) for a in server.algorithms].index(sp.CooccurrenceAlgorithm)
    algo, model = server.algorithms[k], server.models[k]
    qs = _queries(np.random.default_rng(7), 300)
    many = algo.predictMany(model, qs)
    assert many == [algo.predict(model, q) for q in qs]
    assert sum(bool(p.itemScores) for p in many) > 100 and any(not p.itemScores for p in many)
    st = model.device_model().stats()
    assert st["last_parts"] == 1 and st["last_rows"] > 0
    assert algo.predictMany(model, []) == []
    # the pickle keeps the arrays only; a model read back builds its own device copy
    blob = pickle.dumps(model)
    back = pickle.loads(blob)
    assert "_device_model" not in back.__dict__ and "_category_index" not in back.__dict__
    assert algo.predictMany(back, qs) == many


def test_batch_predict_writes_what_the_deployed_engine_answers(engine, tmp_path):
    from pio_b200 import workflow as w
    from pio_b200.workflow import to_json
    qjs = [to_json(q) for q in _queries(np.random.default_rng(8), 150)[:-2]]
    (tmp_path / "in.json").write_text("\n".join(json.dumps(q) for q in qjs) + "\n")
    out = tmp_path / "out.json"
    n = w.BatchPredict.main(["--input", str(tmp_path / "in.json"), "--output", str(out), "--engine-instance-id",
                             engine.id, "--query-chunk", "40"])
    written = out.read_text().splitlines()
    assert n == len(qjs) == len(written)
    server = w.deploy(engine.id)
    for qj, line in zip(qjs, written):
        assert json.loads(line)["prediction"] == server.query(qj)
