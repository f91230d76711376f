"""GPU: filtered batch scoring (pio_als_recommend_filtered / pio_als_similar_batch_filtered), its definition taken literally.

Row j of a filtered batch must equal, bit for bit, what the unfiltered call returns for query j ALONE with the dense mask
    item_mask | item_sets[set_ix[j]] | (ex list of j) | (complement of the wl list of j, if has_wl[j])
and the same weights and flags -- and what tests/scoring_ref.py computes from that mask.  Every case also asserts
pio_als_stats.last_score_path: the scan kernels ran in their filtered instantiation ("filtered"), white-listed queries
went over their lists ("listed")."""
import numpy as np
import pytest

import scoring_ref
import test_gpu_scoring as G

pytestmark = pytest.mark.gpu

N_ITEMS = 777          # no multiple of the 64-row ring step, the 256-item tile or the 512-item CTA step
N_USERS = 90


@pytest.fixture(scope="module")
def native():
    from pio_b200 import native as n
    n.build()
    return n


def make_model(native, rank, seed, n_items=N_ITEMS, n_users=N_USERS):
    rng = np.random.default_rng(seed)
    uf = rng.standard_normal((n_users, rank)).astype(np.float32)
    itf = rng.standard_normal((n_items, rank)).astype(np.float32)
    uh = np.ones(n_users, np.uint8)
    ih = np.ones(n_items, np.uint8)
    uh[[3, 17]] = 0                                  # users without a factor
    ih[rng.choice(n_items, n_items // 20, replace=False)] = 0
    uf[uh == 0] = 0
    itf[ih == 0] = 0
    m = native.NativeALS.from_factors(uf, itf, uh, ih)
    return m, uf, itf, uh, ih


def random_filter(rng, n, n_items, top=None, white_share=0.25, n_sets=3):
    """Per-query lists mixing every shape the definition names; top[j]: ids to exclude wholesale for some queries."""
    exclude, white = [], []
    for j in range(n):
        kind = j % 7
        if kind == 0:
            ex = []
        elif kind == 1:
            ex = list(rng.integers(0, n_items, 5))
        elif kind == 2:                              # duplicates, ids below 0 and past the item range
            ex = list(rng.integers(0, n_items, 6)) * 2 + [-1, -7, n_items, n_items + 5, 2 ** 31 - 1]
        elif kind == 3:                              # longer than any tile of the item matrix
            ex = list(rng.choice(n_items, min(n_items, 600), replace=False))
        elif kind == 4 and top is not None:          # the whole unfiltered top-k goes
            ex = [int(i) for i in top[j] if i >= 0]
        else:
            ex = list(rng.integers(0, n_items, 40))
        rng.shuffle(ex)
        exclude.append(ex)
        if rng.random() < white_share:
            shape = rng.integers(0, 4)
            if shape == 0:
                wl = []
            elif shape == 1:
                wl = [int(rng.integers(0, n_items))]
            else:
                wl = list(rng.integers(0, n_items, 60)) + [-3, n_items + 1]
                if ex:
                    wl += ex[:5]                     # white list and exclusion list intersect
            white.append(wl)
        else:
            white.append(None)
    item_sets = (rng.random((n_sets, n_items)) < 0.4).astype(np.uint8)
    set_ix = rng.integers(-1, n_sets, n).astype(np.int32)
    return exclude, white, set_ix, item_sets


def dense_mask(n_items, base, exclude, white, set_ix, item_sets, j):
    m = np.zeros(n_items, np.uint8) if base is None else np.asarray(base, np.uint8).copy()
    if set_ix is not None and set_ix[j] >= 0:
        m |= item_sets[set_ix[j]]
    if exclude is not None:
        e = np.asarray(exclude[j], np.int64)
        m[e[(e >= 0) & (e < n_items)]] = 1
    if white is not None and white[j] is not None:
        allow = np.zeros(n_items, bool)
        w = np.asarray(white[j], np.int64)
        allow[w[(w >= 0) & (w < n_items)]] = True
        m[~allow] = 1
    return m


def expect_rec_path(kp, topk, blocked, any_scanned, any_listed):
    p = set()
    if any_scanned:
        p |= {"filtered", "dot_blocked" if blocked and kp <= 64 and topk <= G.DB_MAXK else "dot_batched"}
    if any_listed:
        p.add("listed")
    if topk > G.TK_MAXK:
        p.add("multi_pass")
    return p


def check_recommend(native, model, users, topk, flt, mask=None, weight=None, blocked=True, ref_every=1):
    m, uf, itf, uh, ih = model
    exclude, white, set_ix, item_sets = flt
    n, ni = len(users), itf.shape[0]
    qf = native.QueryFilter(n, exclude, white, set_ix, item_sets)
    got = m.recommend(users, topk, mask, weight, query_filter=qf)
    path = m.stats()["last_score_path"]
    listed = [white is not None and white[j] is not None for j in range(n)]
    assert path == expect_rec_path(G.kp_of(itf.shape[1]), topk, blocked, not all(listed), any(listed)), path
    for j in range(n):
        dm = dense_mask(ni, mask, exclude, white, set_ix, item_sets, j)
        want = m.recommend(users[j:j + 1], topk, dm, weight)
        G._same((got[0][j:j + 1], got[1][j:j + 1], got[2][j:j + 1]), want, ("recommend_filtered vs single", j, topk))
        if j % ref_every == 0:
            ref = scoring_ref.recommend(uf, uh, itf, ih, users[j:j + 1], topk, dm, weight)
            G._same((got[0][j:j + 1], got[1][j:j + 1], got[2][j:j + 1]), ref, ("recommend_filtered vs ref", j, topk))
    return got


def expect_sim_path(kp, queries, ih, topk, blocked, listed):
    mp = {"multi_pass"} if topk > G.TK_MAXK else set()
    p = set()
    scanned = [q for q, l in zip(queries, listed) if not l]
    if any(listed):
        p |= {"listed"} | mp
    if scanned and sum(len(q) for q in scanned) > 0:
        nv = [G._n_valid(q, ih) for q in scanned]
        if blocked and kp <= 64 and topk <= G.DB_MAXK and max(nv) <= G.DB_QW:
            p |= {"cos_blocked", "filtered"}
        elif max(sum(nv[g:g + G.SM_QG]) for g in range(0, len(nv), G.SM_QG)) <= G.SM_NV:
            p |= {"cos_multi", "filtered"} | mp
        else:                                        # S5: one query at a time, with its dense mask
            p |= set().union(*[G._s5_path(kp, q, ih, topk) for q in scanned])
    return p


def check_similar(native, model, queries, topk, flt, mask=None, weight=None, keep=False, blocked=True, ref_every=1):
    m, uf, itf, uh, ih = model
    exclude, white, set_ix, item_sets = flt
    n, ni = len(queries), itf.shape[0]
    qf = native.QueryFilter(n, exclude, white, set_ix, item_sets)
    got = m.similar_batch(queries, topk, mask, weight, keep, query_filter=qf)
    path = m.stats()["last_score_path"]
    listed = [white is not None and white[j] is not None for j in range(n)]
    assert path == expect_sim_path(G.kp_of(itf.shape[1]), queries, ih, topk, blocked, listed), path
    for j in range(n):
        dm = dense_mask(ni, mask, exclude, white, set_ix, item_sets, j)
        wi, ws, wc = m.similar(np.asarray(queries[j], np.int32), topk, dm, weight, keep)
        G._same((got[0][j], got[1][j], got[2][j]), (wi, ws, wc), ("similar_filtered vs single", j, topk))
        if j % ref_every == 0:
            ref = scoring_ref.similar(itf, ih, queries[j], topk, dm, weight, keep)
            G._same((got[0][j], got[1][j], got[2][j]), ref, ("similar_filtered vs ref", j, topk))
    return got


def weights_with_zero_ties(rng, n_items):
    w = np.ones(n_items, np.float64)
    w[rng.integers(0, n_items, n_items // 3)] = rng.choice([0.0, -0.0, 0.5, 2.0, -1.0], n_items // 3)
    return w


@pytest.mark.parametrize("rank", [10, 32, 64, 128])
@pytest.mark.parametrize("blocked", [True, False])
def test_recommend_filtered_equals_single_queries_with_the_dense_mask(native, monkeypatch, rank, blocked):
    if not blocked:
        monkeypatch.setenv("PIO_ALS_SCORE_BLOCKED", "0")
    model = make_model(native, rank, seed=rank)
    monkeypatch.delenv("PIO_ALS_SCORE_BLOCKED", raising=False)
    m, uf, itf, uh, ih = model
    rng = np.random.default_rng(100 + rank)
    base = (np.arange(N_ITEMS) % 11 == 0).astype(np.uint8)
    w = weights_with_zero_ties(rng, N_ITEMS)
    for n in (1, 16, 17, 60):
        users = rng.integers(-2, N_USERS + 2, n).astype(np.int32)     # unknown ids on both sides
        users[: min(n, 3)] = [5, 3, 17][: min(n, 3)]                   # a known user and the two without a factor
        for topk in (1, 10, 32, 33, 128, 300):
            if n == 60 and topk in (1, 128) or n in (16, 17) and topk in (10, 300):
                continue
            top = m.recommend(users, topk)[0]
            flt = random_filter(rng, n, N_ITEMS, top)
            check_recommend(native, model, users, topk, flt, blocked=blocked)
            check_recommend(native, model, users, topk, flt, mask=base, weight=w, blocked=blocked)
    m.close()


def test_recommend_filtered_list_shapes(native):
    """Each filter field alone, shared and distinct set rows, and no white list at all (the scan only)."""
    model = make_model(native, 64, seed=7)
    m = model[0]
    rng = np.random.default_rng(8)
    n, topk = 40, 10
    users = rng.integers(0, N_USERS, n).astype(np.int32)
    top = m.recommend(users, topk)[0]
    ex, wl, six, sets = random_filter(rng, n, N_ITEMS, top, white_share=0.5, n_sets=5)
    check_recommend(native, model, users, topk, (ex, None, None, None))
    check_recommend(native, model, users, topk, (None, wl, None, None))
    check_recommend(native, model, users, topk, (None, None, six, sets))
    check_recommend(native, model, users, topk, (None, None, np.zeros(n, np.int32), sets))       # one shared row
    check_recommend(native, model, users, topk, (None, None, (np.arange(n) % 5).astype(np.int32), sets))
    check_recommend(native, model, users, topk, (ex, [[] for _ in range(n)], six, sets))          # every white list empty
    check_recommend(native, model, users, topk, ([[] for _ in range(n)], [None] * n, np.full(n, -1, np.int32), sets))
    m.close()


def test_recommend_filtered_many_users(native):
    """4 100 users: ragged last group of 16, more than one wave of CTAs on the listed route."""
    model = make_model(native, 32, seed=11)
    m = model[0]
    rng = np.random.default_rng(12)
    n = 4100
    users = rng.integers(0, N_USERS, n).astype(np.int32)
    top = m.recommend(users, 10)[0]
    check_recommend(native, model, users, 10, random_filter(rng, n, N_ITEMS, top), ref_every=41)
    m.close()


@pytest.mark.parametrize("rank", [10, 32, 64, 128])
@pytest.mark.parametrize("blocked", [True, False])
def test_similar_filtered_equals_single_queries_with_the_dense_mask(native, monkeypatch, rank, blocked):
    if not blocked:
        monkeypatch.setenv("PIO_ALS_SCORE_BLOCKED", "0")
    model = make_model(native, rank, seed=50 + rank)
    monkeypatch.delenv("PIO_ALS_SCORE_BLOCKED", raising=False)
    m, uf, itf, uh, ih = model
    rng = np.random.default_rng(200 + rank)
    base = (np.arange(N_ITEMS) % 13 == 0).astype(np.uint8)
    w = weights_with_zero_ties(rng, N_ITEMS)
    off = np.flatnonzero(ih == 0)
    for n in (1, 16, 17, 60):
        queries = [list(rng.integers(0, N_ITEMS, rng.integers(1, 5))) for _ in range(n)]
        queries[0] = [int(off[0]), N_ITEMS + 3, -1]          # no valid item
        if n > 2:
            queries[1] = []
            queries[2] = [int(off[1]), int(np.flatnonzero(ih)[0])]
        for topk in (1, 10, 32, 33, 128, 300):
            if n == 60 and topk in (1, 128) or n in (16, 17) and topk in (10, 300):
                continue
            top = m.similar_batch(queries, topk)[0]
            flt = random_filter(rng, n, N_ITEMS, top)
            check_similar(native, model, queries, topk, flt, blocked=blocked)
            check_similar(native, model, queries, topk, flt, mask=base, weight=w, keep=True, blocked=blocked)
    m.close()


def test_similar_filtered_long_queries_and_many_queries(native):
    model = make_model(native, 64, seed=21)
    m, uf, itf, uh, ih = model
    rng = np.random.default_rng(22)
    # a query of 50 ids sends the scanned part to the one-query-at-a-time kernels, each with its dense mask
    queries = [list(rng.integers(0, N_ITEMS, 3)) for _ in range(9)] + [list(rng.choice(N_ITEMS, 50, replace=False))]
    top = m.similar_batch(queries, 20)[0]
    check_similar(native, model, queries, 20, random_filter(rng, len(queries), N_ITEMS, top))
    n = 4100
    queries = [list(rng.integers(0, N_ITEMS, rng.integers(1, 4))) for _ in range(n)]
    top = m.similar_batch(queries, 10)[0]
    check_similar(native, model, queries, 10, random_filter(rng, n, N_ITEMS, top), ref_every=41)
    m.close()


def test_null_filter_is_the_unfiltered_call(native):
    model = make_model(native, 64, seed=31)
    m = model[0]
    users = np.arange(40, dtype=np.int32)
    queries = [[j, j + 1] for j in range(40)]
    for qf in (native.QueryFilter(40), None):
        a = m.recommend(users, 10, query_filter=qf)
        pa = m.stats()["last_score_path"]
        b = m.recommend(users, 10)
        assert pa == m.stats()["last_score_path"] == {"dot_blocked"}
        G._same(a, b, "null filter recommend")
        a = m.similar_batch(queries, 10, query_filter=qf)
        pa = m.stats()["last_score_path"]
        b = m.similar_batch(queries, 10)
        assert pa == m.stats()["last_score_path"] == {"cos_blocked"}
        G._same(a, b, "null filter similar")
    # one user with a null filter keeps the single-query path
    m.recommend(users[:1], 10, query_filter=native.QueryFilter(1))
    assert m.stats()["last_score_path"] == {"score_one"}
    m.close()


def test_argument_errors_are_rejected_before_any_launch(native):
    model = make_model(native, 16, seed=41)
    m = model[0]
    n = 20
    users = np.arange(n, dtype=np.int32)
    queries = [[j] for j in range(n)]
    sets = np.zeros((2, N_ITEMS), np.uint8)

    def filters():
        bad_ptr = native.QueryFilter(n, [[1, 2]] * n)
        bad_ptr.ex_ptr[5] = bad_ptr.ex_ptr[6] + 1
        yield bad_ptr
        bad_wl = native.QueryFilter(n, None, [[1]] * n)
        bad_wl.wl_ptr[n] = bad_wl.wl_ptr[n - 1] - 1
        yield bad_wl
        no_items = native.QueryFilter(n, [[1, 2]] * n)
        no_items.ex_items = None
        yield no_items
        no_wl_items = native.QueryFilter(n, None, [[1]] * n)
        no_wl_items.wl_items = None
        yield no_wl_items
        yield native.QueryFilter(n, None, None, np.full(n, 2, np.int32), sets)       # row past n_sets
        yield native.QueryFilter(n, None, None, np.full(n, -2, np.int32), sets)
        no_sets = native.QueryFilter(n, None, None, np.zeros(n, np.int32), sets)
        no_sets.item_sets = None
        yield no_sets
        neg = native.QueryFilter(n, [[1]] * n)
        neg.n_sets = -1
        yield neg

    for qf in filters():
        for call in (lambda: m.recommend(users, 5, query_filter=qf), lambda: m.similar_batch(queries, 5, query_filter=qf)):
            before = m.stats()["kernel_launches"]
            with pytest.raises(native.NativeError) as e:
                call()
            assert e.value.code == native.ERR_ARG and "query filter" in str(e.value)
            st = m.stats()
            assert st["kernel_launches"] == before and st["last_score_path"] == set()
    m.close()


def test_second_launch_chunk_of_listed_and_scanned_queries(native):
    """More query groups than one launch takes (32 768): the listed route has one group per query, so 33 000 white-listed
    users need a second launch, whose queries are numbered from the chunk's first one; the scanned route reaches its
    second launch above 524 288 users."""
    model = make_model(native, 10, seed=61, n_items=150)
    m, uf, itf, uh, ih = model
    rng = np.random.default_rng(62)
    for n, white_all in ((G.GROUP_CHUNK + 232, True), (G.GROUP_CHUNK * G.SB_QB + 40, False)):
        users = rng.integers(0, N_USERS, n).astype(np.int32)
        ex = rng.integers(0, 150, (n, 3))
        wl = rng.integers(0, 150, (n, 6)) if white_all else None
        qf = native.QueryFilter(n)
        qf.ex_ptr, qf.ex_items = np.arange(n + 1, dtype=np.int64) * 3, np.ascontiguousarray(ex.reshape(-1), np.int32)
        if white_all:
            qf.has_wl = np.ones(n, np.uint8)
            qf.wl_ptr, qf.wl_items = np.arange(n + 1, dtype=np.int64) * 6, np.ascontiguousarray(wl.reshape(-1), np.int32)
        got = m.recommend(users, 5, query_filter=qf)
        assert m.stats()["last_score_path"] == ({"listed"} if white_all else {"dot_blocked", "filtered"})
        for j in list(range(0, n, 997)) + list(range(n - 300, n, 7)):          # rows of both launches
            dm = np.zeros(150, np.uint8)
            if white_all:
                dm[:] = 1
                dm[wl[j]] = 0
            dm[ex[j]] = 1
            want = m.recommend(users[j:j + 1], 5, dm)
            G._same((got[0][j:j + 1], got[1][j:j + 1], got[2][j:j + 1]), want, ("chunked", n, j))
    m.close()


def test_null_filter_pointer_through_the_filtered_symbols(native):
    model = make_model(native, 32, seed=71)
    m = model[0]
    L = native.lib()
    users = np.arange(30, dtype=np.int32)
    want = m.recommend(users, 7)
    oi, os_, oc = np.full((30, 7), -1, np.int32), np.zeros((30, 7), np.float32), np.zeros(30, np.int32)
    assert L.pio_als_recommend_filtered(m._h, users.ctypes.data, 30, 7, None, None, None, oi.ctypes.data, os_.ctypes.data,
                                        oc.ctypes.data) == 0
    G._same((oi, os_, oc), want, "recommend_filtered(f = NULL)")
    queries = [[j, j + 2] for j in range(30)]
    want = m.similar_batch(queries, 7)
    ptr = np.arange(31, dtype=np.int64) * 2
    flat = np.ascontiguousarray(np.asarray(queries, np.int32).reshape(-1))
    assert L.pio_als_similar_batch_filtered(m._h, ptr.ctypes.data, flat.ctypes.data, 30, 7, None, None, 0, None,
                                            oi.ctypes.data, os_.ctypes.data, oc.ctypes.data) == 0
    G._same((oi, os_, oc), want, "similar_batch_filtered(f = NULL)")
    m.close()
