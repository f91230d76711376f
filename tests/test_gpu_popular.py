"""GPU: pio_popular_predict_filtered equals the restatement (popular_ref.py) bit for bit -- items, score bytes, counts --
at its boundaries: item counts around the warp and near 10^5, topk around the warp and the candidate count, all scores
equal, signed zeros, infinities and negative scores, exclusion lists with repeats and out-of-range ids, white lists that
are empty or hold repeats and excluded or set items, set rows that exclude everything, parts of one, two and three
queries, and one model reused across calls and after a rejected one; and the walk of unfiltered queries stops after
32 x ceil(topk / 32) ranked entries."""
import math

import numpy as np
import pytest

import popular_ref as ref

pytestmark = pytest.mark.gpu


def check(m, scores, n, topk, qf=None, **filt):
    got = m.predict_filtered(n, topk, qf)
    want = ref.predict(scores, n, topk, **filt)
    assert got[0].dtype == want[0].dtype and np.array_equal(got[0], want[0])
    assert got[1].dtype == np.float64 and got[1].tobytes() == want[1].tobytes()
    assert np.array_equal(got[2], want[2])
    return got


def tied_scores(rng, n):
    """Small counts times a few weights: long runs of equal scores, 0.0 and -0.0 among them."""
    counts = np.where(rng.random(n) < 0.6, 0.0, rng.integers(1, 6, n).astype(np.float64))
    return counts * rng.choice([1.0, 1.0, 0.0, -1.0, 50.0], n)


def filters(native, rng, n_items, n):
    ex = [None if j % 3 == 0 else rng.integers(-3, n_items + 3, rng.integers(0, 40)).tolist() for j in range(n)]
    wl = [None if j % 4 else [] if j % 8 == 0 else rng.integers(-2, n_items + 2, rng.integers(1, 60)).tolist()
          for j in range(n)]
    sets = (rng.random((3, n_items)) < 0.5).astype(np.uint8)
    six = np.array([[-1, 0, 1, 2][j % 4] for j in range(n)], np.int32)
    return native.QueryFilter(n, ex, wl, six, sets), dict(exclude=ex, white=wl, set_ix=six, item_sets=sets)


@pytest.mark.parametrize("n_items", [1, 31, 32, 33, 100_003])
def test_item_counts(native, n_items):
    rng = np.random.default_rng(n_items)
    scores = tied_scores(rng, n_items)
    m = native.PopularModel(scores)
    try:
        for topk in (1, 32, 33, n_items, n_items + 7):
            check(m, scores, 5, topk)
        n = 40 if n_items < 1000 else 12
        qf, filt = filters(native, rng, n_items, n)
        for topk in (1, 32, 33, n_items + 1):
            check(m, scores, n, topk, qf, **filt)
    finally:
        m.close()


def test_topk_at_the_candidate_count(native):
    rng = np.random.default_rng(7)
    scores = tied_scores(rng, 500)
    m = native.PopularModel(scores)
    qf, filt = filters(native, rng, 500, 24)
    _, _, oc = ref.predict(scores, 24, 600, **filt)
    for topk in sorted({int(c) for c in oc if c > 0}):       # each query's candidate count, exactly
        check(m, scores, 24, topk, qf, **filt)
    m.close()


def test_equal_signed_zero_infinite_and_negative_scores(native):
    scores = np.array([0.0, -0.0, math.inf, -3.5, -math.inf, 0.0, 7.0, -0.0, math.inf, -3.5, -math.inf, 1e-300,
                       -1e-300, 5e-324, -5e-324] * 5, np.float64)
    m = native.PopularModel(scores)
    oi, os_, oc = check(m, scores, 3, scores.shape[0] + 2)
    assert np.signbit(os_[0][os_[0] == 0][:oc[0]]).any()       # -0.0 comes back as -0.0
    m.close()
    same = np.full(77, 2.5)
    m = native.PopularModel(same)
    oi, _, _ = check(m, same, 2, 77)
    assert oi[0].tolist() == list(range(77))                    # every score equal: index order
    m.close()


def test_exclusion_and_white_list_edges(native):
    n_items = 100
    scores = tied_scores(np.random.default_rng(8), n_items)
    order = sorted(range(n_items), key=lambda i: (-scores[i], i))
    ex = [order[:40] + order[:5] + [-1, n_items, 10 ** 6],        # more entries than topk, repeats, out of range
          None, [], order[:3], list(range(n_items)), None]
    wl = [None, [], [order[50], order[50], order[2], -7, n_items, order[1]],   # repeats and out of range
          order[:10],                                           # held items that are excluded too
          order[:5], [order[9], order[4]]]
    sets = np.zeros((2, n_items), np.uint8)
    sets[0, :] = 1                                              # a set row that excludes everything
    sets[1, order[4]] = 1                                       # a white-listed item that is set
    six = np.array([-1, -1, -1, -1, 0, 1], np.int32)
    qf = native.QueryFilter(6, ex, wl, six, sets)
    m = native.PopularModel(scores)
    oi, os_, oc = check(m, scores, 6, 30, qf, exclude=ex, white=wl, set_ix=six, item_sets=sets)
    assert oc.tolist()[:2] == [30, 0] and oc[4] == 0 and oc[5] == 1
    st = m.stats()
    assert st["last_listed"] == sum(len(w) for w in wl if w is not None)
    m.close()


@pytest.mark.parametrize("per_part", [1, 2, 3])
def test_parts(native, monkeypatch, per_part):
    rng = np.random.default_rng(9)
    n_items, n, topk = 300, 30, 8
    scores = tied_scores(rng, n_items)
    ex = [rng.integers(0, n_items, 4).tolist() for _ in range(n)]
    wl = [None if j % 3 else rng.integers(0, n_items, 4).tolist() for j in range(n)]
    six = np.array([j % 2 - 1 for j in range(n)], np.int32)
    sets = (rng.random((1, n_items)) < 0.3).astype(np.uint8)
    qf = native.QueryFilter(n, ex, wl, six, sets)
    # a query holds 4 exclusion entries, 4 white-list entries every third query, and 8 slots: 12 or 16 entries, so a
    # budget of 16 x per_part gives parts of exactly per_part queries
    budget = 16 * per_part
    monkeypatch.setenv("PIO_POPULAR_PREDICT_BUDGET", str(budget))
    m = native.PopularModel(scores)
    check(m, scores, n, topk, qf, exclude=ex, white=wl, set_ix=six, item_sets=sets)
    first = ref.parts(n, topk, budget, ex, wl)
    sizes = np.diff(first + [n])
    st = m.stats()
    assert st["last_parts"] == len(first) and st["last_max_part_queries"] == sizes.max()
    assert set(sizes.tolist()) == {per_part}
    monkeypatch.setenv("PIO_POPULAR_PREDICT_BUDGET", "1")
    check(m, scores, n, topk, qf, exclude=ex, white=wl, set_ix=six, item_sets=sets)
    assert m.stats()["last_parts"] == n                           # at least one query per part
    m.close()


def test_walk_bound_without_filters(native):
    n_items = 100_003
    scores = tied_scores(np.random.default_rng(10), n_items)
    m = native.PopularModel(scores)
    for topk in (1, 31, 32, 33, 64, 65, 1000):
        n = 7
        check(m, scores, n, topk)
        assert m.stats()["last_walked"] <= n * 32 * math.ceil(topk / 32)
    wl = [[1, 2], [3], None]
    check(m, scores, 3, 5, native.QueryFilter(3, white=wl), white=wl)
    assert m.stats()["last_walked"] <= 32                      # only the query without a white list walks
    m.close()


def test_reuse_across_calls_and_after_a_rejected_call(native):
    rng = np.random.default_rng(11)
    scores = tied_scores(rng, 1000)
    m = native.PopularModel(scores)
    qf, filt = filters(native, rng, 1000, 20)
    check(m, scores, 20, 16, qf, **filt)
    launches = m.stats()["kernel_launches"]
    check(m, scores, 20, 16, qf, **filt)
    again = m.stats()["kernel_launches"] - launches
    assert 0 < again < launches                                    # the ranked order is made once
    with pytest.raises(native.NativeError) as e:
        m.predict_filtered(20, 0, qf)
    assert e.value.code == native.ERR_ARG
    st = m.stats()
    assert st["last_parts"] == 0 and st["kernel_launches"] == launches + again
    check(m, scores, 20, 16, qf, **filt)
    check(m, scores, 4, 1000)
    oi, os_, oc = m.predict_filtered(0, 5)
    assert oi.shape == (0, 5) and m.stats()["last_parts"] == 0
    m.close()
