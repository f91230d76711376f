"""CPU: cooc_predict_ref.py, the restatement the GPU tests compare pio_cooc_predict_filtered with, equals
CooccurrenceAlgorithm.predict; its part split on hand-made cases; and the arguments pio_cooc_model_create /
pio_cooc_predict_filtered reject before any device work."""
import ctypes as C

import numpy as np
import pytest

import cooc_predict_ref as ref
from pio_b200.storage import BiMap
from pio_b200.templates import similarproduct as sp

CATS = ["c0", "c1", "c2", "c3"]


def seeded_model(rng, n_items=120, n=12, count_hi=6):
    """A model as training leaves it: per item up to n distinct other items, counts >= 1 (small, so scores tie)."""
    ti = np.full((n_items, n), -1, np.int32)
    tc = np.zeros((n_items, n), np.int32)
    tn = rng.integers(0, n + 1, n_items).astype(np.int32)
    tn[:3] = [0, n, 1]
    for i in range(n_items):
        others = rng.permutation(np.delete(np.arange(n_items), i))[:tn[i]]
        ti[i, :tn[i]] = others
        tc[i, :tn[i]] = np.sort(rng.integers(1, count_hi, tn[i]))[::-1]
    items = {}
    for i in range(n_items):
        r = rng.random()
        if r < 0.1:
            continue                                  # an item the model has no properties for
        items[i] = sp.Item(categories=None if r < 0.2 else [] if r < 0.25 else
                           list(rng.choice(CATS, rng.integers(1, 3), replace=False)))
    return sp.CooccurrenceModel(ti, tc, tn, BiMap({f"i{i}": i for i in range(n_items)}), items)


def _pick(rng, n_items, lo, hi):
    xs = [f"i{x}" for x in rng.choice(n_items, rng.integers(lo, hi), replace=False)]
    return xs + (["nope"] if rng.random() < 0.3 else [])


def seeded_queries(rng, n_items, count):
    cat_rules = [None, None, {"c0"}, {"c1", "c3"}, {"zz"}, set()]
    qs = []
    for j in range(count):
        q_items = _pick(rng, n_items, 1, 5) if j % 13 else ["nope", "nada"]
        if j % 7 == 0:
            q_items = q_items + q_items[:1]            # a repeated query item
        qs.append(sp.Query(items=q_items, num=int(rng.choice([1, 3, 10, 200])),
                           categories=cat_rules[rng.integers(0, len(cat_rules))],
                           categoryBlackList=cat_rules[rng.integers(0, len(cat_rules))],
                           whiteList=None if rng.random() < 0.7 else set(_pick(rng, n_items, 0, 40)),
                           blackList=None if rng.random() < 0.5 else set(_pick(rng, n_items, 0, 20))))
    return qs


def query_arrays(model, qs):
    """What predictMany hands the library for each query: (known ids, exclusion list, white list, set row or -1) and the
    set rows (one per distinct `categories`)."""
    ids = lambda xs: [i for i in (model.itemStringIntMap.get(x) for x in xs) if i is not None]   # noqa: E731
    ix = sp.CategoryIndex(len(model.top_n), model.items)
    rows, row_of, out = [], {}, []
    for q in qs:
        s = -1
        if q.categories is not None:
            key = frozenset(q.categories)
            if key not in row_of:
                row_of[key] = len(rows)
                rows.append(ix.excluded(q.categories, None))
            s = row_of[key]
        out.append((ids(q.items), None if q.blackList is None else ids(q.blackList),
                    None if q.whiteList is None else ids(q.whiteList), s))
    return out, (np.stack(rows) if rows else np.zeros((0, len(model.top_n)), np.uint8))


@pytest.mark.parametrize("seed", [1, 2, 3])
def test_restatement_equals_predict(seed):
    rng = np.random.default_rng(seed)
    model = seeded_model(rng)
    qs = seeded_queries(rng, len(model.top_n), 250)
    algo = sp.CooccurrenceAlgorithm(sp.CooccurrenceAlgorithmParams(n=12))
    arrs, sets = query_arrays(model, qs)
    ql, ex, wl, six = zip(*arrs)
    num = max(q.num for q in qs)
    oi, os_, oc = ref.predict(model.top_items, model.top_counts, model.top_n, ql, num, ex, wl, np.array(six), sets)
    ties = over = 0
    for j, q in enumerate(qs):
        want = algo.predict(model, q)
        n = min(int(oc[j]), q.num)
        got = [sp.ItemScore(model.itemIntStringMap(int(oi[j, t])), float(os_[j, t])) for t in range(n)]
        assert got == want.itemScores, j
        ties += int(np.any(np.diff(os_[j, :oc[j]]) == 0))
        over += int(q.num > oc[j] > 0)
    assert ties and over and any(oc == 0) and sets.shape[0] > 2


def test_category_black_list_is_no_rule():
    rng = np.random.default_rng(9)
    model = seeded_model(rng)
    algo = sp.CooccurrenceAlgorithm(sp.CooccurrenceAlgorithmParams(n=12))
    base = sp.Query(items=["i1", "i5"], num=50)
    for black in ({"c0"}, set(CATS), set()):
        q = sp.Query(items=base.items, num=50, categoryBlackList=black)
        assert algo.predict(model, q) == algo.predict(model, base)


def test_scores_above_two_to_the_32_stay_exact():
    big = 2 ** 31 - 1
    ti = np.array([[2, 3], [2, 3], [0, 1], [0, 1]], np.int32)
    tc = np.array([[big, 5], [big, big], [1, 1], [2, 2]], np.int32)
    tn = np.array([2, 2, 2, 2], np.int32)
    oi, os_, oc = ref.predict(ti, tc, tn, [[0, 1], [0, 1, 0, 7, -3]], 3)
    assert oi[0].tolist() == [2, 3, -1] and os_[0].tolist() == [2 * big, big + 5, 0] and oc.tolist() == [2, 2]
    assert np.array_equal(oi[1], oi[0]) and np.array_equal(os_[1], os_[0])


def test_part_split():
    tn = np.array([5, 0, 3, 7], np.int32)
    qs = [[0], [1], [2, 2], [3, 0], [], [9, -1], [3]]
    assert [ref.expansion(tn, q) for q in qs] == [5, 0, 6, 12, 0, 0, 7]
    assert ref.parts(tn, qs, 1 << 40) == [0]
    assert ref.parts(tn, qs, 11) == [0, 3, 4]        # 11, 12 (one query over the budget), 0 + 0 + 7
    assert ref.parts(tn, qs, 12) == [0, 3, 6]        # 11, 12 + 0 + 0, 7
    assert ref.parts(tn, qs, 1) == [0, 1, 2, 3, 4, 6]   # a part holds at least one query; empty ones join
    assert ref.parts(tn, qs, 0) == [0, 1, 2, 3, 4, 6]
    assert ref.parts(tn, [], 10) == []
    with pytest.raises(ValueError):
        ref.parts(np.array([1 << 16], np.int64), [[0] * (1 << 16)], 10)


# ---- the ABI: rejected before any device work (device 4096 does not exist, so only a check made before the device is
# touched can report an argument error) ------------------------------------------------------------------------------------
NO_DEVICE = 4096


def _model_arrays():
    ti = np.array([[1, 2, -1], [0, -1, -1], [0, 1, -1]], np.int32)
    tc = np.array([[4, 2, 0], [4, 0, 0], [2, 1, 0]], np.int32)
    return ti, tc, np.array([2, 1, 2], np.int32)


@pytest.mark.parametrize("edit,msg", [
    (lambda ti, tc, tn: tn.__setitem__(1, 4), "item 1: top_n 4"),
    (lambda ti, tc, tn: tn.__setitem__(2, -1), "item 2: top_n -1"),
    (lambda ti, tc, tn: ti.__setitem__((2, 1), 3), "item 2, slot 1: item 3"),
    (lambda ti, tc, tn: ti.__setitem__((0, 0), -1), "item 0, slot 0: item -1"),
    (lambda ti, tc, tn: tc.__setitem__((1, 0), -7), "item 1, slot 0: count -7"),
])
def test_model_arrays_rejected(native, edit, msg):
    ti, tc, tn = _model_arrays()
    edit(ti, tc, tn)
    with pytest.raises(native.NativeError) as e:
        native.CoocModel(ti, tc, tn, device=NO_DEVICE)
    assert e.value.code == native.ERR_ARG and msg in str(e.value)
    ti, tc, tn = _model_arrays()
    ti[1, 2], tc[0, 2] = 77, -5                      # entries past top_n are padding, never read
    native.CoocModel(ti, tc, tn, device=NO_DEVICE).close()


def _raw_predict(native, m, ptr, items, n, topk=3, f=None):
    oi, os_, oc = np.zeros(max(n, 1) * topk, np.int32), np.zeros(max(n, 1) * topk, np.int64), np.zeros(max(n, 1), np.int32)
    return native.lib().pio_cooc_predict_filtered(m._h, None if ptr is None else ptr.ctypes.data,
                                                  None if items is None else items.ctypes.data, n, topk,
                                                  None if f is None else C.addressof(f), oi.ctypes.data,
                                                  os_.ctypes.data, oc.ctypes.data)


def test_predict_arguments_rejected(native):
    m = native.CoocModel(*_model_arrays(), device=NO_DEVICE)
    items = np.array([0, 1, 2], np.int32)
    good = np.array([0, 2, 3], np.int64)
    assert _raw_predict(native, m, good, items, 2) == native.ERR_CUDA     # a good call reaches the device
    assert _raw_predict(native, m, good, items, 0) == 0                  # nothing to score
    for ptr in ([0, 3, 2], [-1, 0, 3]):
        assert _raw_predict(native, m, np.array(ptr, np.int64), items, 2) == native.ERR_ARG
    assert _raw_predict(native, m, good, None, 2) == native.ERR_ARG      # entries named, no items
    assert _raw_predict(native, m, good, items, 2, topk=0) == native.ERR_ARG
    assert _raw_predict(native, m, good, items, -1) == native.ERR_ARG
    assert _raw_predict(native, m, None, items, 2) == native.ERR_ARG
    bad_filters = [native.QueryFilter(2, set_ix=[0, 1], item_sets=np.zeros((1, 3), np.uint8)),
                   native.QueryFilter(2, set_ix=[-2, -1], item_sets=np.zeros((1, 3), np.uint8)),
                   native.QueryFilter(2, set_ix=[0, -1])]
    for qf in bad_filters:
        assert _raw_predict(native, m, good, items, 2, f=qf.struct(2, 3)) == native.ERR_ARG
    for name in ("ex", "wl"):
        qf = native.QueryFilter(2, exclude=[[1], [2]], white=[[1], [2]])
        setattr(qf, f"{name}_ptr", np.array([0, 2, 1], np.int64))
        assert _raw_predict(native, m, good, items, 2, f=qf.struct(2, 3)) == native.ERR_ARG
    ok = native.QueryFilter(2, exclude=[[1], None], white=[None, []], set_ix=[0, -1], item_sets=np.zeros((1, 3), np.uint8))
    assert _raw_predict(native, m, good, items, 2, f=ok.struct(2, 3)) == native.ERR_CUDA
    with pytest.raises(native.NativeError) as e:
        m.predict_filtered([[0], [5]], 3, native.QueryFilter(2, set_ix=[3, 0], item_sets=np.zeros((1, 3), np.uint8)))
    assert e.value.code == native.ERR_ARG and "set_ix" in str(e.value)
    st = m.stats()
    assert st["last_parts"] == 0 and st["kernel_launches"] == 0
    m.close()


def test_query_over_the_scan_is_rejected(native):
    topn = 1 << 16
    ti = np.ones((2, topn), np.int32)
    tc = np.ones((2, topn), np.int32)
    m = native.CoocModel(ti, tc, np.array([topn, 0], np.int32), device=NO_DEVICE)
    with pytest.raises(native.NativeError) as e:
        m.predict_filtered([[1], [0] * topn], 5)       # the second query lists 2^16 x 2^16 = 2^32 entries
    assert e.value.code == native.ERR_ARG and "query 1" in str(e.value)
    with pytest.raises(native.NativeError) as e:
        m.predict_filtered([[0] * (topn - 1)], 5)      # one entry fewer fits: the device is reached
    assert e.value.code == native.ERR_CUDA
    m.close()
