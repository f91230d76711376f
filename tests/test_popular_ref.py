"""CPU: popular_ref.py, the restatement the GPU tests compare pio_popular_predict_filtered with, equals the default branch
of ECommAlgorithm.predict (users with no factor and no recent items); its part split on hand-made cases; and the
arguments pio_popular_model_create / pio_popular_predict_filtered reject before any device work."""
import ctypes as C
import math

import numpy as np
import pytest

import popular_ref as ref
from pio_b200.mllib import MatrixFactorizationModel
from pio_b200.storage import BiMap
from pio_b200.templates import ecommerce as ec

CATS = ["c0", "c1", "c2", "c3"]


class _NoEvents:
    """An event index that finds nothing: no seen items, no recent items, no constraint entity."""

    def find(self, *args, **kwargs):
        return []

    def find_many(self, keys, **kwargs):
        return [[] for _ in keys]


def seeded_model(rng, n_items=150, n_users=20):
    """A model whose users own no factor, with buy counts that tie (many items bought by nobody)."""
    mf = MatrixFactorizationModel(4, np.zeros((n_users, 4), np.float32), np.zeros((n_items, 4), np.float32),
                                  np.zeros(n_users, np.uint8), np.ones(n_items, np.uint8))
    popular = {int(i): int(rng.integers(1, 5)) for i in rng.choice(n_items, n_items // 3, replace=False)}
    items = {}
    for i in range(n_items):
        r = rng.random()
        if r < 0.1:
            continue                                  # an item the model has no properties for
        items[i] = ec.Item(categories=None if r < 0.2 else [] if r < 0.25 else
                           list(rng.choice(CATS, rng.integers(1, 3), replace=False)))
    return ec.ECommModel(mf, BiMap({f"u{u}": u for u in range(n_users)}), BiMap({f"i{i}": i for i in range(n_items)}),
                         items, popular)


def seeded_algo(monkeypatch, groups):
    algo = ec.ECommAlgorithm(ec.ECommAlgorithmParams(appName="Shop", unseenOnly=True, seenEvents=["buy"],
                                                     similarEvents=["view"], rank=4, numIterations=1))
    monkeypatch.setattr(algo, "_index", lambda view: _NoEvents())
    monkeypatch.setattr(algo, "weightedItems", lambda: groups)
    return algo


def _pick(rng, n_items, lo, hi):
    xs = [f"i{x}" for x in rng.choice(n_items, rng.integers(lo, hi))]   # repeats allowed
    return xs + (["nope"] if rng.random() < 0.3 else [])


def seeded_queries(rng, n_items, count):
    cat_rules = [None, None, {"c0"}, {"c1", "c3"}, {"zz"}, set()]
    return [ec.Query(user=f"u{rng.integers(0, 25)}", num=int(rng.choice([1, 3, 10, 60, 400])),
                     categories=cat_rules[rng.integers(0, len(cat_rules))],
                     whiteList=None if rng.random() < 0.7 else set(_pick(rng, n_items, 0, 40)),
                     blackList=None if rng.random() < 0.5 else set(_pick(rng, n_items, 0, 30)))
            for _ in range(count)]


def query_arrays(model, qs):
    """What the device call is handed for each query: exclusion list, white list, set row or -1, and the set rows (one per
    distinct `categories`; an item is set when it has no categories or none of the query's)."""
    ids = lambda xs: [i for i in (model.itemStringIntMap.get(x) for x in xs) if i is not None]   # noqa: E731
    n = len(model.mf.productHas)
    rows, row_of, ex, wl, six = [], {}, [], [], []
    for q in qs:
        s = -1
        if q.categories is not None:
            key = frozenset(q.categories)
            if key not in row_of:
                row_of[key] = len(rows)
                rows.append(np.array([not (i in model.items and model.items[i].categories is not None and
                                           set(model.items[i].categories) & set(q.categories)) for i in range(n)],
                                     np.uint8))
            s = row_of[key]
        ex.append(ids(q.blackList or ()))
        wl.append(None if q.whiteList is None else ids(q.whiteList))
        six.append(s)
    return ex, wl, np.array(six, np.int32), (np.stack(rows) if rows else np.zeros((0, n), np.uint8))


def _exact(pairs):
    """(item, score) pairs with the sign of a zero kept: -0.0 == 0.0 in Python."""
    return [(i, repr(float(s))) for i, s in pairs]


WEIGHT_GROUPS = [
    [],
    [{"items": ["i1", "i2", "i3"], "weight": 0.0}, {"items": ["i4", "i5"], "weight": -1.0},
     {"items": ["i6", "i7", "i8"], "weight": 50.0}],
    [{"items": [f"i{k}" for k in range(0, 150, 3)], "weight": -1.0}, {"items": ["i9"], "weight": 2.5}],
]


@pytest.mark.parametrize("seed", [1, 2, 3])
def test_restatement_equals_predict_default_branch(monkeypatch, seed):
    rng = np.random.default_rng(seed)
    model = seeded_model(rng)
    groups = WEIGHT_GROUPS[seed - 1]
    algo = seeded_algo(monkeypatch, groups)
    w = algo._weights(model)
    scores = model.popularity() if w is None else model.popularity() * w
    qs = seeded_queries(rng, len(model.mf.productHas), 200)
    ex, wl, six, sets = query_arrays(model, qs)
    topk = max(q.num for q in qs)
    oi, os_, oc = ref.predict(scores, len(qs), topk, ex, wl, six, sets)
    ties = over = neg_zero = 0
    for j, q in enumerate(qs):
        want = algo.predict(model, q)
        n = min(int(oc[j]), q.num)
        got = [(model.itemIntStringMap(int(oi[j, t])), os_[j, t]) for t in range(n)]
        assert _exact(got) == _exact((s.item, s.score) for s in want.itemScores), j
        ties += int(np.any(np.diff(os_[j, :n]) == 0))
        over += int(q.num > oc[j])
        neg_zero += int(any(math.copysign(1.0, s) < 0 and s == 0 for s in os_[j, :n]))
    assert ties and over and any(oc == 0) and sets.shape[0] > 2
    assert neg_zero or seed != 2                      # 0 buys x weight -1 is -0.0, and it is returned as such


def test_infinite_and_signed_zero_scores(monkeypatch):
    rng = np.random.default_rng(4)
    model = seeded_model(rng, n_items=40)
    model.popularCount = {0: 3, 1: 3, 2: 1, 5: 2}
    groups = [{"items": ["i0"], "weight": float("inf")}, {"items": ["i1"], "weight": float("-inf")},
              {"items": ["i3", "i4"], "weight": -1.0}, {"items": ["i2"], "weight": -0.5}]
    algo = seeded_algo(monkeypatch, groups)
    scores = model.popularity() * algo._weights(model)
    assert not np.isnan(scores).any()
    oi, os_, oc = ref.predict(scores, 1, 40)
    want = algo.predict(model, ec.Query(user="u1", num=40))
    got = [(model.itemIntStringMap(int(i)), s) for i, s in zip(oi[0, :oc[0]], os_[0, :oc[0]])]
    assert _exact(got) == _exact((s.item, s.score) for s in want.itemScores)
    assert oi[0, 0] == 0 and oi[0, oc[0] - 1] == 1 and os_[0, 0] == math.inf
    zeros = [int(i) for i, s in zip(oi[0], os_[0]) if s == 0]
    assert zeros == sorted(zeros) and {3, 4} <= set(zeros)   # -0.0 and +0.0 tie, by item index


def test_part_split():
    ex = [[1, 2], None, [], [5] * 6, [7]]
    wl = [None, [1, 2, 3], [], [1], None]
    assert [ref.entries(2, ex, wl, j) for j in range(5)] == [4, 5, 2, 9, 3]
    assert ref.parts(5, 2, 1 << 40, ex, wl) == [0]
    assert ref.parts(5, 2, 9, ex, wl) == [0, 2, 3, 4]        # 4 + 5 | 2 | 9 | 3
    assert ref.parts(5, 2, 11, ex, wl) == [0, 3, 4]          # 4 + 5 + 2 | 9 | 3
    assert ref.parts(5, 2, 12, ex, wl) == [0, 3]             # 4 + 5 + 2 | 9 + 3
    assert ref.parts(5, 2, 1, ex, wl) == [0, 1, 2, 3, 4]     # a part holds at least one query
    assert ref.parts(4, 3, 6) == [0, 2]                      # output slots alone: two queries of 3
    assert ref.parts(0, 3, 10) == []


# ---- the ABI: rejected before any device work (device 4096 does not exist, so only a check made before the device is
# touched can report an argument error) ------------------------------------------------------------------------------------
NO_DEVICE = 4096


def test_model_scores_rejected(native):
    for bad, msg in (([1.0, float("nan"), 2.0], "item 1"), ([float("nan")], "item 0")):
        with pytest.raises(native.NativeError) as e:
            native.PopularModel(np.array(bad), device=NO_DEVICE)
        assert e.value.code == native.ERR_ARG and msg in str(e.value) and "NaN" in str(e.value)
    with pytest.raises(native.NativeError) as e:
        native.PopularModel(np.zeros(0), device=NO_DEVICE)                 # n_items < 1
    assert e.value.code == native.ERR_ARG
    native.PopularModel(np.array([math.inf, -math.inf, -0.0, 0.0, -3.0]), device=NO_DEVICE).close()


def _raw_predict(native, m, n, topk=3, f=None, outs=True):
    k = max(n, 1) * max(topk, 1)
    oi, os_, oc = np.zeros(k, np.int32), np.zeros(k, np.float64), np.zeros(max(n, 1), np.int32)
    return native.lib().pio_popular_predict_filtered(m._h, n, topk, None if f is None else C.addressof(f),
                                                     oi.ctypes.data if outs else None, os_.ctypes.data,
                                                     oc.ctypes.data)


def test_predict_arguments_rejected(native):
    m = native.PopularModel(np.array([3.0, 1.0, 2.0]), device=NO_DEVICE)
    assert _raw_predict(native, m, 2) == native.ERR_CUDA                  # a good call reaches the device
    assert _raw_predict(native, m, 0) == 0                                # nothing to score
    assert _raw_predict(native, m, 2, topk=0) == native.ERR_ARG
    assert _raw_predict(native, m, -1) == native.ERR_ARG
    assert _raw_predict(native, m, 2, outs=False) == native.ERR_ARG       # a NULL output
    bad_filters = [native.QueryFilter(2, set_ix=[0, 1], item_sets=np.zeros((1, 3), np.uint8)),
                   native.QueryFilter(2, set_ix=[-2, -1], item_sets=np.zeros((1, 3), np.uint8)),
                   native.QueryFilter(2, set_ix=[0, -1])]
    for qf in bad_filters:
        assert _raw_predict(native, m, 2, f=qf.struct(2, 3)) == native.ERR_ARG
    for name in ("ex", "wl"):
        for ptr in ([0, 2, 1], [-1, 0, 1]):
            qf = native.QueryFilter(2, exclude=[[1], [2]], white=[[1], [2]])
            setattr(qf, f"{name}_ptr", np.array(ptr, np.int64))
            assert _raw_predict(native, m, 2, f=qf.struct(2, 3)) == native.ERR_ARG
        qf = native.QueryFilter(2, exclude=[[1], [2]], white=[[1], [2]])
        setattr(qf, f"{name}_items", None)                                 # entries named, no items
        assert _raw_predict(native, m, 2, f=qf.struct(2, 3)) == native.ERR_ARG
    ok = native.QueryFilter(2, exclude=[[1, 1, 7], None], white=[None, [-4]], set_ix=[0, -1],
                            item_sets=np.zeros((1, 3), np.uint8))
    assert _raw_predict(native, m, 2, f=ok.struct(2, 3)) == native.ERR_CUDA
    with pytest.raises(native.NativeError) as e:
        m.predict_filtered(2, 3, native.QueryFilter(2, set_ix=[3, 0], item_sets=np.zeros((1, 3), np.uint8)))
    assert e.value.code == native.ERR_ARG and "set_ix" in str(e.value)
    st = m.stats()
    assert st["last_parts"] == 0 and st["kernel_launches"] == 0
    m.close()


def test_query_over_the_part_numbering_is_rejected(native):
    m = native.PopularModel(np.ones(4), device=NO_DEVICE)
    qf = native.QueryFilter(2, exclude=[[1], [2]])
    items = qf.ex_items
    for last, rc in (((1 << 32) - 2, native.ERR_ARG), ((1 << 32) - 3, native.ERR_CUDA)):
        qf.ex_ptr = np.array([0, 1, last], np.int64)   # query 1's last - 1 entries plus 3 slots: 2^32, then 2^32 - 1
        qf.ex_items = items                             # never read: the call stops before the device
        assert _raw_predict(native, m, 2, topk=3, f=qf.struct(2, 4)) == rc
    m.close()
