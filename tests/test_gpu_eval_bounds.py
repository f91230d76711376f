"""GPU tests (-m gpu): the device k-fold split and rank counts (eval_folds.cuh, pio_eval_folds_*) held exactly to
tests/eval_ref.py at their boundaries: fold sizes, the four maps and every fold's rank counts, for n around the scan and
sort tiles and at 2 M ratings, k_fold from 1 (no training set) to past n (empty test folds), queries with thousands of
test items (the rank-count lane loops and a deep binary search), query counts at multiples of the CTA's eight warps,
(query, item) sort keys past 32 bits, top-N widths around a warp, and NaN / inf / tied ratings.  Each case asserts the
facts that make it a boundary case."""
import ctypes as C

import numpy as np
import pytest

import eval_ref
import ingest_ref
from pio_b200 import native as nat
from pio_b200.evaluation import EvalColumns
from pio_b200.templates import recommendation as rec

pytestmark = pytest.mark.gpu

RC_WARPS = 8


def predictions(rng, fold, num, ends=True):
    """A top-N result of the fold: per query its own training-known test items first (so hits happen), random fold-local
    items after them, and fold-local items 0 and n_items - 1; counts 0 .. num."""
    nq, ni = fold["query_user"].shape[0], fold["item"].shape[0]
    if ni == 0:
        return np.zeros((nq, num), np.int32), np.zeros(nq, np.int32)
    items = rng.integers(0, ni, (nq, num)).astype(np.int32)
    if ends and num > 1:
        items[::2, -1], items[1::2, -1] = ni - 1, 0
        items[::3, 0] = ni - 1
    loc = np.full(int(max(fold["item"].max(), fold["test_item"].max(initial=0))) + 1, -1, np.int64)
    loc[fold["item"]] = np.arange(ni)
    t = np.flatnonzero(loc[fold["test_item"]] >= 0)
    q = fold["test_q"][t]
    o = np.argsort(q, kind="stable")
    t, q = t[o], q[o]
    start = np.searchsorted(q, q, side="left")
    p = np.arange(q.shape[0]) - start                 # position of the test rating inside its query
    keep = (p < num - 1) & (p % 2 == 0)               # every other one: some hits, some misses
    items[q[keep], p[keep]] = loc[fold["test_item"][t[keep]]]
    count = rng.integers(0, num + 1, nq).astype(np.int32)
    count[:2] = [0, num][:nq]
    return items, count


def check_split(gu, gi, ratings, k_fold, folds=None):
    """Sizes and maps of every fold against eval_ref.split; returns (ref folds, device folds)."""
    ref = eval_ref.split(gu, gi, ratings, k_fold)
    folds = folds or nat.EvalFolds(gu, gi, ratings, k_fold)
    for f in range(k_fold):
        r = ref[f]
        assert folds.sizes(f) == (r["user"].shape[0], r["item"].shape[0], r["train_user"].shape[0],
                                  r["query_user"].shape[0]), f
        m = folds.maps(f)
        for key in ("user", "item", "query_user", "query_train_user"):
            assert np.array_equal(m[key], r[key]), (f, key)
    return ref, folds


def check_counts(res, fold, items, count, ks, thresholds):
    for k in ks:
        for thr in thresholds:
            got = res.rank_counts(k, thr)
            want = eval_ref.rank_counts(fold, items, count, k, thr)
            for name, g, w in zip(("hits", "npos", "nraw"), got, want):
                assert np.array_equal(g, w), (name, k, thr)


def assert_empty_folds_give_nothing(folds, ref, k_fold, n):
    empty = [f for f in range(k_fold) if f >= n]
    for f in empty:
        assert ref[f]["query_user"].shape[0] == 0 and folds.sizes(f)[3] == 0
        res = folds.add_result(f, np.zeros((0, 3), np.int32), np.zeros(0, np.int32))
        assert all(x.shape == (0,) for x in res.rank_counts(5, 1.0))
        res.close()
    return empty


# ---- n and k_fold ---------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("n", [1, 2, 2047, 2048, 2049, 4095, 4096, 4097])
@pytest.mark.parametrize("kf", ["1", "2", "31", "n-1", "n", "n+3", "1000"])
def test_n_and_k_fold(n, kf):
    k_fold = {"1": 1, "2": 2, "31": 31, "n-1": n - 1, "n": n, "n+3": n + 3, "1000": 1000}[kf]
    if k_fold < 1:
        pytest.skip("k_fold n - 1 = 0 at n = 1")
    rng = np.random.default_rng(n * 31 + k_fold)
    gu = rng.integers(0, max(2, n // 7), n)
    gi = rng.integers(0, max(2, n // 3), n)
    ratings = rng.choice(np.array([1.0, 2.0, 3.0, 4.0, 4.5, 5.0]), n)
    ref, folds = check_split(gu, gi, ratings, k_fold)
    empty = assert_empty_folds_give_nothing(folds, ref, k_fold, n)
    assert (len(empty) > 0) == (k_fold > n)
    for f in sorted({0, k_fold - 1, min(n, k_fold) - 1}):
        if f in empty:
            continue
        items, count = predictions(rng, ref[f], 10)
        res = folds.add_result(f, items, count)
        check_counts(res, ref[f], items, count, (1, 9, 10, 15, 1000), (1.0, 4.0, 4.5, 6.0))
    if k_fold == 1:
        assert folds.sizes(0)[:3] == (0, 0, 0)
        als = nat.NativeALS(4, 1, 1, seed=1, init_mode=nat.INIT_HASH)
        with pytest.raises(nat.NativeError) as e:
            folds.set_ratings(0, als)
        assert e.value.code == nat.ERR_ARG
        als.close()
    folds.close()


# ---- query shapes ---------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("num", [33, 100])
def test_one_user_with_thousands_of_test_items(num):
    """One user's 30 000 ratings over 12 000 items beside 4 000 light users: in fold 0 it has > 15 000 test ratings over
    thousands of distinct items, so every lane loop of rank_counts_kernel runs many strides and the binary search runs
    over thousands of slots."""
    rng = np.random.default_rng(num)
    heavy = np.zeros(30000, np.int64)
    hi = rng.integers(0, 12000, 30000)
    lu, li = rng.integers(1, 4001, 8000), rng.integers(0, 12000, 8000)
    gu, gi = np.concatenate([heavy, lu]), np.concatenate([hi, li])
    o = rng.permutation(gu.shape[0])
    gu, gi = gu[o], gi[o]
    ratings = rng.choice(np.array([1.0, 2.0, 3.0, 4.0, 5.0]), gu.shape[0])
    ref, folds = check_split(gu, gi, ratings, 2)
    for f in range(2):
        r = ref[f]
        q0 = int(np.flatnonzero(r["query_user"] == 0)[0])
        mine = r["test_q"] == q0
        assert mine.sum() > 14000 and np.unique(r["test_item"][mine]).shape[0] > 5000
        items, count = predictions(rng, r, num)
        count[q0] = num
        res = folds.add_result(f, items, count)
        check_counts(res, r, items, count, (1, num - 1, num, num + 5, 1000), (1.0, 3.0, 5.0, 5.5))
        if num > 64:
            assert res.rank_counts(1000, 1.0)[0][q0] > 32   # hits from more than one stride of the kk loop
    folds.close()


def test_every_user_has_exactly_one_test_rating():
    k_fold = 5
    n = 5 * 3001
    gu = np.arange(n) // k_fold                          # user u rates positions 5u .. 5u + 4: one in every fold
    rng = np.random.default_rng(2)
    gi = rng.integers(0, 900, n)
    ratings = rng.choice(np.array([1.0, 3.0, 5.0]), n)
    ref, folds = check_split(gu, gi, ratings, k_fold)
    for f in (0, 4):
        r = ref[f]
        assert r["query_user"].shape[0] == 3001 and np.array_equal(np.bincount(r["test_q"]), np.ones(3001))
        items, count = predictions(rng, r, 31)
        res = folds.add_result(f, items, count)
        check_counts(res, r, items, count, (1, 30, 31, 36, 1000), (1.0, 3.0, 4.0))
    folds.close()


@pytest.mark.parametrize("nq", [7, 8, 9, 15, 16, 17, 1023, 1024, 1025])
def test_query_counts_around_the_cta(nq):
    """Fold 0 has exactly nq queries: the last CTA of rank_counts_kernel is full, one warp short or one warp over."""
    rng = np.random.default_rng(nq)
    k_fold = 3
    n = 3 * (nq * 4)
    gu = np.empty(n, np.int64)
    gu[0::3] = rng.permutation(np.repeat(np.arange(nq), 4))
    gu[1::3] = rng.integers(0, nq + 50, nq * 4)
    gu[2::3] = rng.integers(0, nq + 50, nq * 4)
    gi = rng.integers(0, 200, n)
    ratings = rng.choice(np.array([1.0, 2.0, 4.0, 5.0]), n)
    ref, folds = check_split(gu, gi, ratings, k_fold)
    assert ref[0]["query_user"].shape[0] == nq and nq % RC_WARPS in (0, 1, RC_WARPS - 1)
    items, count = predictions(rng, ref[0], 32)
    res = folds.add_result(0, items, count)
    check_counts(res, ref[0], items, count, (1, 31, 32, 37), (2.0, 4.0))
    folds.close()


# ---- key widths -------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("top", [2, 256, 257, 65536, 65537, 1 << 24, (1 << 24) + 1])
@pytest.mark.parametrize("users", [100, 33000])
def test_sort_key_widths(top, users):
    """Sparse global item ids up to top - 1 (ibits 1, 8 / 9, 16 / 17, 24 / 25) and enough queries that
    ceil_log2(nq) + ibits lies on both sides of 32, up to 40."""
    rng = np.random.default_rng(top + users)
    n = 4 * users
    gu = rng.permutation(np.repeat(np.arange(users), 4))
    ids = np.unique(np.concatenate([[0, top - 1], rng.integers(0, top, 300)]))
    gi = rng.choice(ids, n)
    gi[:2] = [0, top - 1]
    ratings = rng.choice(np.array([-1.0, 0.0, 2.0, 4.0]), n)
    ref, folds = check_split(gu, gi, ratings, 2)
    ibits = ingest_ref.ceil_log2(top)
    for f in range(2):
        nq = ref[f]["query_user"].shape[0]
        width = ingest_ref.ceil_log2(nq) + ibits
        assert ibits == {2: 1, 256: 8, 257: 9, 65536: 16, 65537: 17, 1 << 24: 24, (1 << 24) + 1: 25}[top]
        if users == 33000 and top > 1 << 24:
            assert width > 32 and nq > 1 << 14
        items, count = predictions(rng, ref[f], 8)
        res = folds.add_result(f, items, count)
        check_counts(res, ref[f], items, count, (1, 8), (0.0, 2.0, 3.0))
    folds.close()


# ---- results ---------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("num", [1, 31, 32, 33, 100])
def test_result_widths_and_freed_results(num):
    rng = np.random.default_rng(num)
    n = 40000
    gu, gi = rng.integers(0, 600, n), rng.integers(0, 2500, n)
    ratings = rng.choice(np.array([1.0, 2.0, 3.0, 4.0, 5.0]), n)
    ref, folds = check_split(gu, gi, ratings, 4)
    for f in (0, 3):
        r = ref[f]
        made = []
        for _ in range(3):
            items, count = predictions(rng, r, num)
            made.append((folds.add_result(f, items, count), items, count))
        made[1][0].close()                               # freed in between: the others keep their own arrays
        items, count = predictions(rng, r, num)
        made[1] = (folds.add_result(f, items, count), items, count)
        for res, items, count in made:
            assert (count == 0).any() and (count == num).any()
            check_counts(res, r, items, count, sorted({1, max(num - 1, 1), num, num + 5, 1000}), (1.0, 3.0, 5.0))
    folds.close()


# ---- ratings ---------------------------------------------------------------------------------------------------------------
def test_special_and_duplicate_ratings():
    """Repeated (query, item) test pairs with different ratings (the largest decides), thresholds equal to rating values,
    below and above all, negative ratings, 0, +-inf, NaN alone and NaN before or after a finite rating of the pair."""
    rng = np.random.default_rng(17)
    k_fold = 2
    pairs = 3000
    pu, pi = rng.integers(0, 400, pairs), rng.integers(0, 300, pairs)
    rep = rng.integers(1, 5, pairs)
    gu, gi = np.repeat(pu, rep), np.repeat(pi, rep)
    vals = np.array([-3.0, -0.0, 0.0, 1.0, 2.5, 4.0, np.inf, -np.inf, np.nan])
    ratings = rng.choice(vals, gu.shape[0])
    first = np.concatenate([[0], np.cumsum(rep)[:-1]])
    ratings[first[::7]] = np.nan                         # NaN before a finite rating of the same pair
    o = rng.permutation(gu.shape[0])                     # NaN both before and after a pair's finite ratings
    gu, gi, ratings = gu[o], gi[o], ratings[o]
    ref, folds = check_split(gu, gi, ratings, k_fold)
    for f in range(k_fold):
        r = ref[f]
        key = r["test_q"] * 1000 + r["test_item"]
        _, inv, cnt = np.unique(key, return_inverse=True, return_counts=True)
        dup = cnt[inv] > 1
        assert dup.sum() > 100 and np.isnan(r["test_rating"][dup]).any() and np.isinf(r["test_rating"]).any()
        items, count = predictions(rng, r, 20)
        res = folds.add_result(f, items, count)
        check_counts(res, r, items, count, (1, 20, 1000), [-np.inf, -5.0, -3.0, -0.0, 0.0, 1.0, 2.5, 4.0, 5.0, np.inf])
    folds.close()


# ---- the fold's training COO goes through the ingest --------------------------------------------------------------------------
def test_fold_training_ingest_equals_the_restatement(native):
    rng = np.random.default_rng(23)
    n = 60000
    gu, gi = rng.integers(0, 3000, n), rng.integers(0, 800, n)
    ratings = rng.choice(np.array([-1.0, 0.0, 1.0, 2.5, 4.0]), n)
    ref, folds = check_split(gu, gi, ratings, 5)
    for f in (0, 4):
        r = ref[f]
        nu, ni = r["user"].shape[0], r["item"].shape[0]
        als = native.NativeALS(12, nu, ni, implicit=True, init_mode=native.INIT_HASH)
        folds.set_ratings(f, als)
        want = ingest_ref.ingest(r["train_user"], r["train_item"], r["train_rating"], nu, ni, "none", implicit=True,
                                 rank=12)
        for name in ("user", "item"):
            assert not ingest_ref.differences(als.debug_side(name), want[name][0]), (f, name)
        assert want["user"][0]["nnz"] == n - (n + 4 - f) // 5
        als.close()
    folds.close()


# ---- scale and the metrics -------------------------------------------------------------------------------------------------
def test_two_million_ratings_and_the_metric_values():
    """About 2 M ratings, k_fold 3: every fold's counts, and PrecisionAtK / PositiveCount per-query values as
    calculate_columns builds them from the device counts."""
    rng = np.random.default_rng(2024)
    n = 2_000_003
    gu = np.minimum(rng.zipf(1.4, n), 150_000) - 1
    gi = np.minimum(rng.zipf(1.3, n), 40_000) - 1
    ratings = rng.choice(np.array([1.0, 2.0, 3.0, 4.0, 5.0]), n)
    ref, folds = check_split(gu, gi, ratings, 3)
    for f in range(3):
        r = ref[f]
        items, count = predictions(rng, r, 10)
        res = folds.add_result(f, items, count)
        check_counts(res, r, items, count, (1, 10), (2.0, 4.0))
        for k, thr in ((10, 4.0), (3, 2.0)):
            hits, npos, nraw = res.rank_counts(k, thr)
            rh, rp, rr = eval_ref.rank_counts(r, items, count, k, thr)
            ok = npos > 0
            assert (hits[ok] / np.minimum(k, npos[ok]).astype(np.float64)).tolist() == \
                eval_ref.precision_values(rh, rp, k)
            assert nraw.astype(np.float64).tolist() == rr.astype(np.float64).tolist()
            cols = EvalColumns([(None, None, res)])
            want = EvalColumns([(None, None, _Ref(r, items, count))])
            for m in (rec.PrecisionAtK(k, thr), rec.PositiveCount(thr)):
                assert m.calculate_columns(None, cols) == m.calculate_columns(None, want)
    folds.close()


class _Ref:
    def __init__(self, fold, items, count):
        self.fold, self.items, self.count = fold, items, count

    def rank_counts(self, k, threshold):
        return eval_ref.rank_counts(self.fold, self.items, self.count, k, threshold)


def test_create_refuses_n_of_2_31_before_reading():
    """n = 2^31 with one-element arrays: ERR_ARG from the size check, before any array is read."""
    one_i, one_d = np.zeros(1, np.int32), np.ones(1, np.float64)
    h = C.c_void_p()
    rc = nat.lib().pio_eval_folds_create(C.c_int(0), one_i.ctypes.data_as(C.POINTER(C.c_int32)),
                                         one_i.ctypes.data_as(C.POINTER(C.c_int32)),
                                         one_d.ctypes.data_as(C.POINTER(C.c_double)), C.c_int64(1 << 31), C.c_int32(2),
                                         C.byref(h))
    assert rc == nat.ERR_ARG and not h.value
