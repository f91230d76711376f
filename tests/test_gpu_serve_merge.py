"""GPU: pio_serve_zscore_merge equals the restatement (serve_merge_ref.py) bit for bit -- list lengths across the pairwise
sum's 8 / 128 / split thresholds and the warp, batches across the radix tile, topk across the take kernel's block, and
parts of one, two and three queries -- and rejects bad input before any device work; the similarproduct engine served
through predictManyColumns + serveManyColumns answers what serve answers over predict, also with a model whose item
numbering differs; and batchpredict on the column path writes the object path's bytes."""
import datetime as dt
import json

import numpy as np
import pytest

import serve_merge_ref as ref

pytestmark = pytest.mark.gpu


def batch(rng, Q, widths, n_items, fill=None, tie_every=0):
    items, scores, counts = [], [], []
    for a, w in enumerate(widths):
        it = np.full((Q, w), -1, np.int32)
        sc = np.zeros((Q, w))
        cn = (rng.integers(0, w + 1, Q) if fill is None else np.full(Q, min(fill, w))).astype(np.int32)
        for j in range(Q):
            c = int(cn[j])
            it[j, :c] = rng.choice(n_items, c, replace=c > n_items)
            v = rng.standard_normal(c) * 10.0 ** rng.integers(-3, 4)
            sc[j, :c] = v.round(1) if tie_every and j % tie_every == 0 else v
            if a == 2:
                sc[j, :c] = np.sort(rng.integers(1, 30, c))[::-1]   # co-occurrence-like integer sums
        items.append(it)
        scores.append(sc)
        counts.append(cn)
    return items, scores, counts


def check(native, items, scores, counts, num, topk, n_items):
    got = native.serve_zscore_merge(items, scores, counts, num, topk, n_items)
    want = ref.merge(items, scores, counts, num, topk)
    assert np.array_equal(got[0], want[0]) and np.array_equal(got[2], want[2])
    assert got[1].tobytes() == want[1].tobytes()
    return got


@pytest.mark.parametrize("n", [1, 2, 7, 8, 9, 31, 32, 33, 127, 128, 129, 136, 255, 256, 257, 1024, 1031, 2100])
def test_list_lengths(native, n):
    """Full lists of n entries: the pairwise sum's plain loop, blocked and split forms, and the per-list warp."""
    rng = np.random.default_rng(n)
    Q = 6
    items, scores, counts = batch(rng, Q, [n, n, n], 5000, fill=n)
    num = np.array([1, 2, 5, n, 3 * n, 10 ** 9])[:Q]
    check(native, items, scores, counts, num, min(3 * n, 4000), 5000)


@pytest.mark.parametrize("Q,widths,n_items,topk", [
    (1, [1], 1, 1), (3, [0, 4], 3, 5), (127, [20, 20, 20], 40, 60), (128, [20, 20, 20], 40, 127),
    (129, [20, 20, 20], 40, 128), (300, [15, 30, 15], 1000, 129), (700, [10, 3, 8], 7, 21),
    (1500, [40, 40, 40], 2 ** 20, 40), (4097, [1, 1, 1], 2, 3)])
def test_batches(native, Q, widths, n_items, topk):
    """Batch sizes across the stats block, the radix tile (4096 entries) and the take kernel's 128 threads; items shared
    by two and three algorithms (small numberings), exact ties, and the first and last ids."""
    rng = np.random.default_rng(Q)
    items, scores, counts = batch(rng, Q, widths, n_items, tie_every=3)
    if widths[0]:
        items[0][0, 0] = 0
        items[0][-1, 0] = n_items - 1
        counts[0][[0, -1]] = np.maximum(counts[0][[0, -1]], 1)
    num = rng.choice([1, 2, 4, 10, 100], Q)
    _, _, oc = check(native, items, scores, counts, num, topk, n_items)
    st = native.serve_merge_stats()
    assert st["parts"] == 1 and st["entries"] == sum(int(c.sum()) for c in counts) and st["rows"] >= oc.sum()


def test_signed_zeros_and_equal_scores(native):
    items = [np.array([[0, 1, 2], [0, 1, 2], [3, 4, 0]], np.int32), np.array([[2, 0], [1, 2], [4, 3]], np.int32)]
    scores = [np.array([[-0.0, 0.0, -0.0], [5.0, 5.0, 5.0], [1.0, 2.0, 3.0]]), np.array([[-0.0, -0.0], [7.0, 7.0],
                                                                                         [2.0, 1.0]])]
    counts = [np.array([3, 3, 3], np.int32), np.array([2, 2, 2], np.int32)]
    for num in ([1, 1, 1], [3, 3, 3], [1, 2, 5]):
        check(native, items, scores, counts, np.array(num), 5, 5)


@pytest.mark.parametrize("budget,sizes", [(1, {1}), (40, {1, 2, 3}), (60, {3}), (10 ** 9, {30})])
def test_parts(native, monkeypatch, budget, sizes):
    rng = np.random.default_rng(budget % 97)
    Q = 30
    widths = [12, 12, 12]
    items, scores, counts = batch(rng, Q, widths, 50, fill=11)
    for c in counts:
        c[:] = rng.integers(3, 7, Q)           # 9 .. 18 entries per query
    counts[0][7], counts[1][7], counts[2][7] = 11, 11, 11   # 33: over the budget of 40 with any neighbour
    num = rng.choice([1, 3, 20], Q)
    base = native.serve_zscore_merge(items, scores, counts, num, 20, 50)
    monkeypatch.setenv("PIO_SERVE_MERGE_BUDGET", str(budget))
    got = check(native, items, scores, counts, num, 20, 50)
    for g, b in zip(got, base):
        assert g.tobytes() == b.tobytes()
    first = ref.parts(counts, budget)
    part_sizes = np.diff(first + [Q])
    st = native.serve_merge_stats()
    assert st["parts"] == len(first) and st["max_part_queries"] == part_sizes.max() and st["budget"] == budget
    assert sizes <= set(part_sizes.tolist())


def test_rejections_before_device_work(native):
    rng = np.random.default_rng(2)
    items, scores, counts = batch(rng, 4, [5, 5], 10, fill=3)
    num = np.array([2, 2, 2, 2])

    def rejected(its, scs, cns, nm, topk=5, n_items=10):
        native.serve_zscore_merge(items, scores, counts, num, 5, 10)          # a good call first: its stats are reset
        assert native.serve_merge_stats()["parts"] == 1
        with pytest.raises(native.NativeError) as e:
            native.serve_zscore_merge(its, scs, cns, nm, topk, n_items)
        assert e.value.code == native.ERR_ARG and native.serve_merge_stats()["parts"] == 0

    def edit(arrs, a, j, t, v):
        out = [x.copy() for x in arrs]
        if t is None:
            out[a][j] = v
        else:
            out[a][j, t] = v
        return out

    rejected(items, scores, edit(counts, 1, 2, None, 6), num)                 # count above the width
    rejected(items, scores, edit(counts, 0, 0, None, -1), num)                # negative count
    rejected(edit(items, 0, 3, 2, -1), scores, counts, num)                   # id below the numbering
    rejected(edit(items, 1, 1, 0, 10), scores, counts, num)                   # id past the numbering
    rejected(items, edit(scores, 0, 1, 1, np.nan), counts, num)               # non-finite scores
    rejected(items, edit(scores, 1, 3, 2, np.inf), counts, num)
    rejected(items, edit(scores, 1, 3, 0, -np.inf), counts, num)
    rejected([], [], [], num)                                                 # no algorithm
    rejected(items, scores, counts, np.array([2, 0, 2, 2]))                   # num below 1
    rejected(items, scores, counts, np.array([2, 2, 2, -5]))
    rejected(items, scores, counts, num, topk=0)
    rejected(items, scores, counts, num, n_items=0)
    # entries past a list's count are not read: ids, NaN or inf there are accepted
    ok = edit(edit(items, 0, 0, 4, -7), 0, 0, 3, 99)
    check(native, ok, edit(scores, 0, 0, 4, np.nan), counts, num, 5, 10)
    with pytest.raises(ValueError):
        native.serve_zscore_merge(items, scores, counts[:1], num, 5, 10)


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


def _queries(rng, n, low_num=False):
    from pio_b200.templates import similarproduct as sp
    items = [f"i{k}" for k in range(74)]
    cats = [None, None, {"c0"}, {"c1", "c9"}, {"zz"}, set()]

    def pick(lo, hi):
        return [str(x) for x in rng.choice(items, rng.integers(lo, hi), replace=False)] + (
            ["nope"] if rng.random() < 0.3 else [])
    qs = []
    for j in range(n):
        q_items = pick(1, 5) if j % 11 else ["nope", "nada"]
        qs.append(sp.Query(items=q_items, num=int(rng.choice([1, 2, 4, 10, 70])),
                           categories=cats[rng.integers(0, len(cats))],
                           categoryBlackList=cats[rng.integers(0, len(cats))],
                           whiteList=None if rng.random() < 0.7 else set(pick(0, 30)),
                           blackList=None if rng.random() < 0.5 else set(pick(0, 20))))
    qs.append(sp.Query(items=["i3", "i4"], num=500))
    if low_num:   # ALS scoring rejects num < 1 in predict itself, so only an engine without it can answer these
        qs += [sp.Query(items=["i1"], num=0), sp.Query(items=["i1", "i2"], num=-2), sp.Query(items=["nope"], num=-1)]
    return qs


@pytest.fixture(scope="module")
def engine(tmp_path_factory):
    from pio_b200 import storage as s
    from pio_b200 import workflow as w
    tmp = tmp_path_factory.mktemp("sim")
    mp = pytest.MonkeyPatch()
    mp.setenv("PIO_EVENTDATA_DIR", str(tmp / "events"))
    mp.setenv("PIO_MODELDATA_DIR", str(tmp / "models"))
    s.import_events("Sim", _events())
    variant = tmp / "engine.json"
    variant.write_text(json.dumps({
        "id": "default", "engineFactory": "pio_b200.templates.similarproduct.SimilarProductEngine",
        "datasource": {"params": {"appName": "Sim"}},
        "algorithms": [{"name": "als", "params": {"rank": 8, "numIterations": 4, "lambda": 0.01, "seed": 3}},
                       {"name": "likealgo", "params": {"rank": 8, "numIterations": 4, "lambda": 0.01, "seed": 5}},
                       {"name": "cooccurrence", "params": {"n": 12}}]}))
    inst = w.CreateWorkflow.main(["--engine-id", "sim", "--engine-version", "1", "--engine-variant", str(variant)])
    yield inst, tmp
    mp.undo()


def served(server, qs, algorithms=None, models=None):
    algorithms, models = algorithms or server.algorithms, models or server.models
    cols = server.serving.serveManyColumns(qs, [a.predictManyColumns(m, qs) for a, m in zip(algorithms, models)])
    out = []
    for j in range(len(qs)):
        if j in cols.objects:
            out.append([(x.item, x.score) for x in cols.objects[j].itemScores])
        else:
            n = cols.count[j]
            out.append([(cols.names[i], v) for i, v in zip(cols.items[j, :n].tolist(), cols.scores[j, :n].tolist())])
    return out, cols


def expected(server, qs, algorithms=None, models=None):
    algorithms, models = algorithms or server.algorithms, models or server.models
    return [[(x.item, x.score) for x in server.serving.serve(q, [a.predict(m, q) for a, m in
                                                                  zip(algorithms, models)]).itemScores] for q in qs]


def same(got, want):
    assert len(got) == len(want)
    for g, w in zip(got, want):
        assert [i for i, _ in g] == [i for i, _ in w]
        assert [np.float64(v).tobytes() for _, v in g] == [np.float64(v).tobytes() for _, v in w]


def test_columns_serve_what_serve_answers(engine, monkeypatch):
    from pio_b200 import workflow as w
    inst, tmp = engine
    monkeypatch.setenv("PIO_MODELDATA_DIR", str(tmp / "models"))
    server = w.deploy(inst.id)
    assert [type(a).__name__ for a in server.algorithms] == ["ALSAlgorithm", "LikeAlgorithm", "CooccurrenceAlgorithm"]
    qs = _queries(np.random.default_rng(7), 400)
    got, cols = served(server, qs)
    same(got, expected(server, qs))
    assert not cols.objects and sum(bool(g) for g in got) > 200 and any(not g for g in got)
    assert any(q.num == 1 and g for q, g in zip(qs, got)) and got[-1]
    # the co-occurrence model alone answers num < 1: those queries are marked and go through serve
    qs = _queries(np.random.default_rng(6), 100, low_num=True)
    a, m = server.algorithms[2:], server.models[2:]
    got, cols = served(server, qs, a, m)
    same(got, expected(server, qs, a, m))
    n = len(qs)
    assert set(cols.objects) == {n - 3, n - 2, n - 1} and got[n - 2]
    assert server.serving._numbering([a.predictManyColumns(m, qs[:1]).names
                                      for a, m in zip(server.algorithms, server.models)])[1] == [None] * 3


def test_remap_of_a_model_with_another_numbering(engine, monkeypatch):
    """A co-occurrence model whose ids are a permutation of the others', with one more item: the serving numbers the
    union and gathers that model's ids into it."""
    from pio_b200 import workflow as w
    from pio_b200.storage import BiMap
    from pio_b200.templates import similarproduct as sp
    inst, tmp = engine
    monkeypatch.setenv("PIO_MODELDATA_DIR", str(tmp / "models"))
    server = w.deploy(inst.id)
    cm = server.models[2]
    n = len(cm.top_n)
    perm = np.random.default_rng(3).permutation(n + 1)[:n]     # old id -> new id, in [0, n]; one id left free
    ti = np.full((n + 1, cm.top_items.shape[1]), -1, np.int32)
    tc = np.zeros_like(ti)
    tn = np.zeros(n + 1, np.int32)
    ti[perm] = np.where(cm.top_items >= 0, perm[np.maximum(cm.top_items, 0)], -1)
    tc[perm], tn[perm] = cm.top_counts, cm.top_n
    names = {s: int(perm[i]) for s, i in cm.itemStringIntMap.toSeq()}
    names["extra-item"] = int(np.setdiff1d(np.arange(n + 1), perm)[0])
    other = sp.CooccurrenceModel(ti, tc, tn, BiMap(names), {int(perm[i]): v for i, v in cm.items.items()}, cm.device)
    qs = _queries(np.random.default_rng(8), 300)
    algorithms, models = server.algorithms, server.models[:2] + [other]
    got, cols = served(server, qs, algorithms, models)
    _, remaps = server.serving._item_numbering[1:]
    same(got, expected(server, qs, algorithms, models))
    assert remaps[0] is None and remaps[1] is None and remaps[2] is not None and len(cols.names) == n + 1


def test_batch_predict_writes_the_object_paths_bytes(engine, monkeypatch, tmp_path):
    from pio_b200 import workflow as w
    from pio_b200.workflow import to_json
    inst, tmp = engine
    monkeypatch.setenv("PIO_MODELDATA_DIR", str(tmp / "models"))
    qjs = [to_json(q) for q in _queries(np.random.default_rng(9), 300)]
    (tmp_path / "in.json").write_text("\n".join(json.dumps(q) for q in qjs) + "\n")
    out = tmp_path / "out.json"
    n = w.BatchPredict.main(["--input", str(out.with_name("in.json")), "--output", str(out), "--engine-instance-id",
                             inst.id, "--query-chunk", "70"])
    server = w.deploy(inst.id)
    assert n == len(qjs) and w.BatchPredict.columnar(server)
    queries = w.BatchPredict.read_queries(tmp_path / "in.json", server.algorithms[0].queryClass())
    want = "".join(json.dumps(rec, separators=(",", ":")) + "\n" for rec in w.BatchPredict.run(server, queries, 70))
    assert out.read_bytes() == want.encode()
