"""GPU: the filtered batch calls (pio_als_recommend_filtered / pio_als_similar_batch_filtered) against tests/filtered_ref.py,
bit for bit, at the boundaries where their kernels can go wrong.

tests/test_gpu_filtered.py checks the definition on imported handles (internal row == external id), random factors and
one item count.  Here every case but one runs on a handle whose internal order is NOT the external one (`permuted`, the
trained handles of test_gpu_scoring and its `controlled` tie handle), so a kernel that indexes a filter, a set bit or a
factor row by the wrong numbering fails.  Every case compares ids, scores (as bits) and counts with filtered_ref and
asserts pio_als_stats.last_score_path, so it provably ran the path it names.  Sections:

  a  equal scores and signed zeros cut at the topk boundary by exclusions, white lists and set rows
  b  the padded-rank ladder on trained handles, every route
  c  item counts around the 32-bit set word, the scan tiles and the CTA step; set bits only in the last partial word
  d  dispatch edges under a filter: user counts, topk, DB_QW / SM_NV / SM_QIDS, the S5 split, an all-empty batch
  e  the listed route: white-list lengths around the warp and LS_THREADS, duplicates across those entries, its passes
  f  a filter leaving exactly 128 / 256 candidates on the scan route
  g  the grid split of the similar side: cos_blocked bins, cos_multi groups, listed cosine queries
  h  a tie over 300 007 items that survives a filter
The constants and ladders below are checked against the sources by tests/test_filtered_ref.py."""
import numpy as np
import pytest

import filtered_ref as FR
import scoring_ref
import test_gpu_filtered as F
import test_gpu_scoring as G

pytestmark = pytest.mark.gpu

LS_THREADS, WARP, SET_WORD = 256, 32, 32
WL_LENGTHS = [0, 1, 31, 32, 33, 255, 256, 257, 513]   # white-list entries of one listed query
WL_DUPS = [31, 255]                                    # a duplicate at sorted entries (d, d + 1): lanes 31 / 32, steps
SET_ITEMS = [31, 32, 33, 63, 64, 65]                   # item counts around the 32-bit set word
TIE_TOPKS = [1, 10, 32, 33, 128, 129, 256, 257]
ZERO_TOPKS = TIE_TOPKS + [1000]
REC_USERS = [1, 16, 17]
REC_TOPKS = [32, 33, 128, 129]
QUERY_VALID = [8, 9]                                   # valid vectors of one batch query: S3 up to DB_QW
GROUP_VECTORS = [40, 41]                               # valid vectors of an 8-query group: S4 up to SM_NV
QUERY_IDS = [64, 65, 70]                               # ids of one S4 query: shared memory up to SM_QIDS
S5_VALID = [56, 57]                                    # one S5 query at KP 64, topk 20: cos_batched / cos_fallback
EXHAUST = [128, 256]                                   # candidates left by the filter
EXHAUST_TOPKS = [128, 129, 256, 257]
LISTED_SPLIT = G.GROUP_CHUNK + 232                     # white-listed queries: one group each
OVERFLOW_ITEMS, OVERFLOW_RANKS, OVERFLOW_TOPKS = 300_007, [8, 24, 40], [77, 128, 129]


# ---- handles -----------------------------------------------------------------------------------------------------------
def assert_permuted(m):
    """the handle's internal order differs from the external one on the item side (and on the user side if it has
    more than one user)"""
    for side in ("item", "user"):
        d = m.debug_side(side)
        if d["n"] > 1:
            assert not np.array_equal(d["perm"], np.arange(d["n"])), side


def permuted(native, uf, itf, uh=None, ih=None, seed=0):
    """A handle scoring exactly these factors in a non-identity internal order: set_ratings with degrees rising with the
    id (the degree-descending internal order runs against the external one), then set_init, as
    test_gpu_scoring.controlled() does.  Rows without a factor get no rating."""
    nu, k = uf.shape
    ni = itf.shape[0]
    uh = np.ones(nu, np.uint8) if uh is None else np.asarray(uh, np.uint8)
    ih = np.ones(ni, np.uint8) if ih is None else np.asarray(ih, np.uint8)
    uf = np.where(uh[:, None] == 1, uf, 0).astype(np.float32)
    itf = np.where(ih[:, None] == 1, itf, 0).astype(np.float32)
    rng = np.random.default_rng(seed)
    au, ai = np.flatnonzero(uh), np.flatnonzero(ih)
    di = 1 + (np.arange(ai.size) * 3) // ai.size
    du = 1 + (np.arange(au.size) * 3) // au.size
    item = np.concatenate([np.repeat(ai, di), rng.choice(ai, int(du.sum()))])
    user = np.concatenate([rng.choice(au, int(di.sum())), np.repeat(au, du)])
    m = native.NativeALS(k, nu, ni, lam=0.01)
    m.set_ratings(user, item, rng.random(item.shape[0]).astype(np.float32) + 0.5)
    m.set_init(uf, itf)
    guf, gitf, guh, gih = m.get_factors()
    assert np.array_equal(guh, uh) and np.array_equal(gih, ih)
    assert np.array_equal(guf, uf) and np.array_equal(gitf, itf)       # the factors come back unchanged
    assert_permuted(m)
    return G.Scorer(m, uf, itf, uh, ih)


def random_model(native, n_items, rank, seed, n_users=40, ties=True):
    rng = np.random.default_rng(seed)
    itf = rng.standard_normal((n_items, rank)).astype(np.float32)
    if ties:
        itf[1::7] = itf[0]
    ih = (rng.random(n_items) > 0.1).astype(np.uint8)
    ih[0] = ih[-1] = 1
    uf = rng.standard_normal((n_users, rank)).astype(np.float32)
    uf[0] = 0.0                                     # the all-ties user
    uh = np.ones(n_users, np.uint8)
    uh[[3, 7]] = 0
    return permuted(native, uf, itf, uh, ih, seed), rng


# ---- checks ------------------------------------------------------------------------------------------------------------
def _sub(flt, rows):
    ex, wl, six, sets = flt
    return (None if ex is None else [ex[j] for j in rows], None if wl is None else [wl[j] for j in rows],
            None if six is None else np.asarray(six)[rows], sets)


def _listed(wl, n):
    return [wl is not None and wl[j] is not None for j in range(n)]


def check_rec(native, s, users, topk, flt, mask=None, weight=None, rows=None, names=(), qf=None):
    """recommend with the filter flt = (exclude, white, set_ix, item_sets): the path, then rows (all) against the ref"""
    users = np.asarray(users, np.int32)
    n = users.shape[0]
    qf = native.QueryFilter(n, *flt) if qf is None else qf
    got = s.m.recommend(users, topk, mask, weight, query_filter=qf)
    p = s.path()
    listed = _listed(flt[1], n)
    want = F.expect_rec_path(s.kp, topk, True, not all(listed), any(listed))
    what = ("recommend", s.kp, n, topk, mask is not None, weight is not None)
    assert p == want and set(names) <= p, (what, p, want, names)
    rows = np.arange(n) if rows is None else np.asarray(rows)
    ref = FR.recommend(s.uf, s.uh, s.itf, s.ih, users[rows], topk, mask, weight, *_sub(flt, rows))
    G._same((got[0][rows], got[1][rows], got[2][rows]), ref, what)
    return got


def check_sim(native, s, queries, topk, flt, mask=None, weight=None, keep=False, rows=None, names=(), qf=None):
    n = len(queries)
    qf = native.QueryFilter(n, *flt) if qf is None else qf
    got = s.m.similar_batch(queries, topk, mask, weight, keep, query_filter=qf)
    p = s.path()
    want = F.expect_sim_path(s.kp, queries, s.ih, topk, True, _listed(flt[1], n))
    what = ("similar", s.kp, n, [len(q) for q in queries][:4], topk, mask is not None, weight is not None, keep)
    assert p == want and set(names) <= p, (what, p, want, names)
    rows = np.arange(n) if rows is None else np.asarray(rows)
    ref = FR.similar_batch(s.itf, s.ih, [queries[j] for j in rows], topk, mask, weight, keep, *_sub(flt, rows))
    G._same((got[0][rows], got[1][rows], got[2][rows]), ref, what)
    return got


def mixed_filter(rng, n, n_items, white_share=0.3):
    return F.random_filter(rng, n, n_items, None, white_share=white_share)


# ---- a. ties ----------------------------------------------------------------------------------------------------------
def _block_filters(order, n_items):
    """per tie block: exclude its two smallest ids / white-list the block and its neighbours / a set row taking every
    other member (by id); plus one query without a filter"""
    ex, wl, six = [], [], []
    sets = []
    for b, (start, length) in enumerate(G.TIE_BLOCKS):
        members = np.sort(order[start:start + length])
        sets.append(np.zeros(n_items, np.uint8))
        sets[-1][members[::2]] = 1
        ex += [[int(v) for v in members[:2]], [], []]
        wl += [None, [int(v) for v in order[max(0, start - 1):start + length + 1]], None]
        six += [-1, -1, b]
    ex.append([])
    wl.append(None)
    six.append(-1)
    return ex, wl, np.array(six, np.int32), np.array(sets)


@pytest.mark.parametrize("rank", [24, 100])
def test_ties_cut_at_the_topk_boundary(native, rank):
    s, anchor, order, off_ids = G.controlled(native, rank)
    assert_permuted(s.m)
    ni = s.ih.shape[0]
    flt = _block_filters(order, ni)
    n = len(flt[0])
    mask, weight = G._mask_weight(ni, np.random.default_rng(rank))
    for topk in TIE_TOPKS:
        check_rec(native, s, [0] * n, topk, flt, names={"filtered", "listed"})
        check_sim(native, s, [[anchor]] * n, topk, flt, names={"filtered", "listed"})
        check_sim(native, s, [[anchor]] * n, topk, flt, keep=True)
    check_rec(native, s, [0] * n, 33, flt, mask=mask, weight=weight)
    check_sim(native, s, [[anchor]] * n, 33, flt, mask=mask, weight=weight)
    # the zero user: weights 0 / -1 give +0 / -0 scores that tie in id order; filters cut through the first ids
    w01 = np.where(np.arange(ni) % 2 == 0, 0.0, -1.0)
    act = np.flatnonzero(s.ih)
    for topk in ZERO_TOPKS:
        cut = act[min(topk, act.size - 1)]
        zsets = np.zeros((1, ni), np.uint8)
        zsets[0, act[:2 * topk:2]] = 1
        zf = ([[int(act[0]), int(act[1])], [int(cut)], [], [], []],
              [None, None, [int(v) for v in act[max(0, topk - 3):topk + 3]], None, None],
              np.array([-1, -1, -1, 0, -1], np.int32), zsets)
        check_rec(native, s, [1] * 5, topk, zf, weight=w01, names={"filtered", "listed"})
        for keep in (False, True):
            check_sim(native, s, [[anchor], [anchor, int(act[1])], [anchor], [anchor], [int(act[3])]], topk, zf,
                      weight=w01, keep=keep)


# ---- b. rank ladder -----------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("rank", G.RANKS)
def test_rank_ladder_every_route(native, monkeypatch, rank):
    s = G._trained(native, monkeypatch, rank, {})
    assert_permuted(s.m)
    ni = s.ih.shape[0]
    rng = np.random.default_rng(rank)
    act = np.flatnonzero(s.ih)
    users = list(range(40))
    blocked = {"dot_blocked"} if s.kp <= 64 else {"dot_batched"}
    check_rec(native, s, users, 10, mixed_filter(rng, 40, ni), names=blocked | {"filtered", "listed"})
    check_rec(native, s, users, 40, mixed_filter(rng, 40, ni), names={"dot_batched", "filtered", "listed"})
    short = [[int(v) for v in rng.choice(act, rng.integers(1, 4))] for _ in range(24)]
    check_sim(native, s, short, 10, mixed_filter(rng, 24, ni),
              names=({"cos_blocked"} if s.kp <= 64 else {"cos_multi"}) | {"filtered", "listed"})
    check_sim(native, s, short, 40, mixed_filter(rng, 24, ni), keep=True, names={"cos_multi", "filtered", "listed"})
    s5 = short[:5] + [[int(v) for v in rng.choice(act, 50, replace=False)]]
    check_sim(native, s, s5, 20, mixed_filter(rng, 6, ni, white_share=0.0))


# ---- c. item-count ladder -----------------------------------------------------------------------------------------------
def _last_word_sets(ni):
    """set rows whose only bits are in the last (partial) 32-bit word, and one naming item 0"""
    last = SET_WORD * ((ni - 1) // SET_WORD)
    sets = np.zeros((4, ni), np.uint8)
    sets[0, ni - 1] = 1
    sets[1, last:] = 1
    sets[2, last + 1::2] = 1
    sets[3, 0] = 1
    return sets


def test_item_count_ladder(native):
    for ni in G._item_ladder() + SET_ITEMS:
        s, rng = random_model(native, ni, 40, ni)
        sets = _last_word_sets(ni)
        last = SET_WORD * ((ni - 1) // SET_WORD)
        n = 20
        ex = [[0, ni - 1] if j % 3 == 0 else [ni - 1] if j % 3 == 1 else [] for j in range(n)]
        wl = [[0, ni - 1, ni - 1, -1, ni] if j % 4 == 3 else list(range(last, ni)) if j % 5 == 4 else None
              for j in range(n)]
        six = np.array([j % 5 - 1 for j in range(n)], np.int32)
        for flt in ((ex, wl, six, sets), (None, None, six, sets)):
            for topk in (10, ni + 5):
                check_rec(native, s, list(range(n)), topk, flt)
                queries = [[int(v) for v in rng.integers(-1, ni + 2, 3)] for _ in range(n)]
                check_sim(native, s, queries, topk, flt, keep=topk == 10)
        s.m.close()


# ---- d. dispatch edges --------------------------------------------------------------------------------------------------
def _valid_query(rng, act, off, n_valid, n_ids):
    ids = list(rng.choice(act, n_valid, replace=False)) + list(rng.choice(off, n_ids - n_valid))
    rng.shuffle(ids)
    return [int(v) for v in ids]


def test_dispatch_edges(native):
    s, rng = random_model(native, 777, 64, 5)
    ni = 777
    act = np.flatnonzero(s.ih)
    off = np.concatenate([np.flatnonzero(s.ih == 0), [ni, ni + 9, -1]])
    for n in REC_USERS:
        for topk in REC_TOPKS:
            users = rng.integers(-1, 42, n).astype(np.int32)
            check_rec(native, s, users, topk, mixed_filter(rng, n, ni))
    # S3 / S4 at DB_QW valid vectors per query
    for nv in QUERY_VALID:
        qs = [_valid_query(rng, act, off, nv, nv + 2)] + [[int(v)] for v in rng.choice(act, 3)]
        check_sim(native, s, qs, 20, mixed_filter(rng, 4, ni, 0.0),
                  names={"cos_blocked" if nv <= G.DB_QW else "cos_multi", "filtered"})
    # S4 / S5 at SM_NV valid vectors per group of eight
    for gv in GROUP_VECTORS:
        qs = [_valid_query(rng, act, off, gv // 8 + (j < gv % 8), gv // 8 + 2) for j in range(8)]
        check_sim(native, s, qs, 33, mixed_filter(rng, 8, ni, 0.0),
                  names={"cos_multi", "filtered"} if gv <= G.SM_NV else {"cos_batched"})
    # the query ids of an S4 query in shared memory up to SM_QIDS, read from global memory above; the best items of
    # the query sit at both ends of its id list
    top = np.argsort(-scoring_ref.cosine_scores(s.itf, s.ih, [int(act[0])]), kind="stable")
    for n_ids in QUERY_IDS:
        q = [int(act[0])] + [int(v) for v in rng.choice(off, n_ids - 3)] + [int(top[1]), int(top[2])]
        qs = [q] + [[int(v)] for v in rng.choice(act, 7)]
        for keep in (False, True):
            check_sim(native, s, qs, 33, mixed_filter(rng, 8, ni, 0.0), keep=keep, names={"cos_multi", "filtered"})
    # S5 queries take the host-built dense mask; the kernel split lies between 56 and 57 valid vectors
    for nv in S5_VALID:
        qs = [_valid_query(rng, act, off, nv, nv + 3), [int(act[1])], [int(act[2]), int(act[3])]]
        flt = mixed_filter(rng, 3, ni, 0.0)
        want = "cos_batched" if G.s5_smem(s.kp, nv, nv + 3, 20) <= G.S5_SMEM_LIMIT else "cos_fallback"
        check_sim(native, s, qs, 20, flt, names={want})
        check_sim(native, s, qs, 20, flt, mask=(np.arange(ni) % 9 == 0).astype(np.uint8), keep=True)
    # an all-empty batch: nothing to gather (the scanned part goes per query and launches nothing)
    empty = [[] for _ in range(20)]
    check_sim(native, s, empty, 10, mixed_filter(rng, 20, ni, 0.0))
    check_sim(native, s, empty, 10, mixed_filter(rng, 20, ni, 0.5))
    s.m.close()


def test_identity_order_control(native):
    """the dispatch edges of the recommend side and a listed / S3 / S4 similar batch on an imported handle"""
    m, uf, itf, uh, ih = F.make_model(native, 64, seed=9)     # from_factors: internal row == external id
    s = G.Scorer(m, uf, itf, uh, ih)
    rng = np.random.default_rng(9)
    ni = itf.shape[0]
    for n in REC_USERS:
        for topk in REC_TOPKS:
            check_rec(native, s, rng.integers(0, F.N_USERS, n).astype(np.int32), topk, mixed_filter(rng, n, ni))
    qs = [[int(v) for v in rng.integers(0, ni, rng.integers(1, 4))] for _ in range(24)]
    for topk in (10, 40):
        check_sim(native, s, qs, topk, mixed_filter(rng, 24, ni))
    m.close()


# ---- e. the listed route ------------------------------------------------------------------------------------------------
def _white_list(rng, ids, length):
    """`length` entries from ids whose SORTED order repeats an id at entries (d, d + 1) for every d of WL_DUPS that fits,
    given in shuffled order"""
    n_dup = sum(1 for d in WL_DUPS if length > d + 1)
    wl = sorted(int(v) for v in rng.choice(ids, length - n_dup, replace=False))
    for d in WL_DUPS:
        if length > d + 1:
            wl.insert(d, wl[d])
    assert len(wl) == length
    for d in WL_DUPS:
        if length > d + 1:
            assert wl[d] == wl[d + 1]
    out = list(wl)
    rng.shuffle(out)
    return out


def test_listed_route(native):
    ni = 1500
    s, rng = random_model(native, ni, 48, 21, ties=False)
    all_ids = np.arange(ni)
    act = np.flatnonzero(s.ih)
    n = len(WL_LENGTHS)
    wl = [_white_list(rng, all_ids, L) for L in WL_LENGTHS]
    flt = (None, wl, None, None)
    mixed = ([[int(v) for v in rng.choice(ni, 40)] for _ in range(n)], wl, np.arange(n, dtype=np.int32) % 2,
             (rng.random((2, ni)) < 0.3).astype(np.uint8))
    users = rng.integers(0, 40, n).astype(np.int32)
    queries = [[int(v) for v in rng.choice(act, 2)] for _ in range(n)]
    own = [w + q for w, q in zip(wl, queries)]          # cosine queries whose own ids are white-listed
    for topk in (10, 300, 600):
        check_rec(native, s, users, topk, flt, names={"listed"})
        check_rec(native, s, users, topk, mixed, names={"listed"})
        for keep in (False, True):
            check_sim(native, s, queries, topk, mixed, keep=keep, names={"listed"})
            check_sim(native, s, queries, topk, (mixed[0], own, mixed[2], mixed[3]), keep=keep, names={"listed"})
    # every item white-listed; a white list meeting an exclusion list and a set row
    every = [list(range(ni))] * 3
    check_rec(native, s, [0, 1, 2], 129, (None, every, None, None))
    check_sim(native, s, [[int(act[0])], [int(act[1])], [int(act[2])]], 10, (None, every, None, None))
    w = [int(v) for v in rng.choice(act, 200, replace=False)]
    sets = np.zeros((1, ni), np.uint8)
    sets[0, w[50:150]] = 1
    inter = ([w[:100]] * 4, [w] * 4, np.array([0, 0, -1, 0], np.int32), sets)
    check_rec(native, s, [0, 1, 2, 5], 64, inter)
    check_sim(native, s, [[w[0]], [w[120], w[199]], [w[160]], [int(act[0])]], 64, inter, keep=True)
    check_sim(native, s, [[w[0]], [w[120], w[199]], [w[160]], [int(act[0])]], 64, inter)
    # exactly 128 / 256 allowed items: the pass bound runs out at the second or third pass
    q = [int(act[5])]
    cos = scoring_ref.cosine_scores(s.itf, s.ih, q)
    pos = np.setdiff1d(np.flatnonzero((cos > 0) & (s.ih == 1)), q)
    for n_allowed in EXHAUST:
        rw = [[int(v) for v in rng.choice(act, n_allowed, replace=False)] for _ in range(3)]
        sw = [[int(v) for v in rng.choice(pos, n_allowed, replace=False)] + q for _ in range(3)]
        for topk in EXHAUST_TOPKS:
            got = check_rec(native, s, [1, 2, 5], topk, (None, rw, None, None))
            assert (got[2] == min(topk, n_allowed)).all()
            for keep in (False, True):
                got = check_sim(native, s, [q] * 3, topk, (None, sw, None, None), keep=keep)
                assert (got[2] == min(topk, n_allowed + keep)).all()
    s.m.close()


# ---- f. exhaustion on the scan route ------------------------------------------------------------------------------------
def test_scan_exhaustion(native):
    ni = 1500
    s, rng = random_model(native, ni, 40, 31, ties=False)
    act = np.flatnonzero(s.ih)
    q = [int(act[7])]
    cos = scoring_ref.cosine_scores(s.itf, s.ih, q)
    pos = np.setdiff1d(np.flatnonzero((cos > 0) & (s.ih == 1)), q)
    n = 20
    for n_left in EXHAUST:
        keep_r = rng.choice(act, n_left, replace=False)
        keep_s = rng.choice(pos, n_left, replace=False)
        sets = np.ones((2, ni), np.uint8)
        sets[0, keep_r] = 0
        sets[1, keep_s] = 0
        ex_r = [int(v) for v in np.setdiff1d(act, keep_r)]
        ex_s = [int(v) for v in np.setdiff1d(pos, keep_s)]
        rec_f = ([ex_r if j % 2 else [] for j in range(n)], None, np.array([-1 if j % 2 else 0 for j in range(n)], np.int32),
                 sets)
        sim_f = ([ex_s if j % 2 else [] for j in range(9)], None, np.array([-1 if j % 2 else 1 for j in range(9)], np.int32),
                 sets)
        for topk in EXHAUST_TOPKS:
            got = check_rec(native, s, rng.integers(8, 40, n), topk, rec_f, names={"dot_batched", "filtered"})
            assert (got[2] == min(topk, n_left)).all()
            got = check_sim(native, s, [q] * 9, topk, sim_f, names={"cos_multi", "filtered"})
            assert (got[2] == min(topk, n_left)).all()
    s.m.close()


# ---- g. grid split, similar side ----------------------------------------------------------------------------------------
def _csr_filter(native, n, ex=None, wl=None, set_ix=None, sets=None):
    """a QueryFilter from [n, w] arrays of per-query lists (fixed width)"""
    qf = native.QueryFilter(n, None, None, set_ix, sets)
    if ex is not None:
        qf.ex_ptr, qf.ex_items = np.arange(n + 1, dtype=np.int64) * ex.shape[1], np.ascontiguousarray(ex.reshape(-1), np.int32)
    if wl is not None:
        qf.has_wl = np.ones(n, np.uint8)
        qf.wl_ptr, qf.wl_items = np.arange(n + 1, dtype=np.int64) * wl.shape[1], np.ascontiguousarray(wl.reshape(-1), np.int32)
    return qf


def _split_check(native, s, queries, topk, flt, arrays, chunk, part, keep=False, names=()):
    """the whole call against the reference on rows around every chunk boundary, and against sub-calls of `part`
    queries (below the split), each with its slice of the filter"""
    n = len(queries)
    rng = np.random.default_rng(chunk)
    rows = G._split_rows(n, chunk, rng)
    got = check_sim(native, s, queries, topk, flt, keep=keep, rows=rows, names=names, qf=_csr_filter(native, n, *arrays))
    ex, wl, six, sets = arrays
    for c0 in range(0, n, part):
        c1 = min(n, c0 + part)
        sl = lambda a: None if a is None else a[c0:c1]   # noqa: E731
        qf = _csr_filter(native, c1 - c0, sl(ex), sl(wl), sl(six), sets)
        want = s.m.similar_batch(queries[c0:c1], topk, None, None, keep, query_filter=qf)
        G._same((got[0][c0:c1], got[1][c0:c1], got[2][c0:c1]), want, ("split vs parts", topk, c0))


def test_grid_split_similar(native):
    ni, rank = 600, 8
    rng = np.random.default_rng(41)
    itf = rng.standard_normal((ni, rank)).astype(np.float32)
    ih = (rng.random(ni) > 0.1).astype(np.uint8)
    s = permuted(native, rng.standard_normal((30, rank)).astype(np.float32), itf, None, ih, 41)
    n_q = G.SPLIT_QUERIES
    lens = rng.integers(0, 4, n_q)
    flat = rng.integers(-1, ni + 2, int(lens.sum())).astype(np.int32)
    ptr = np.concatenate([[0], np.cumsum(lens)])
    queries = [flat[ptr[j]:ptr[j + 1]] for j in range(n_q)]
    ex = rng.integers(-1, ni + 1, (n_q, 3))
    six = rng.integers(-1, 3, n_q).astype(np.int32)
    sets = (rng.random((3, ni)) < 0.3).astype(np.uint8)
    flt = (list(ex), None, six, sets)
    # bins of the blocked kernel, as plan_similar_batch packs them
    bins, bq, bv = [0], 0, 0
    for j, q in enumerate(queries):
        nv = G._n_valid(q, ih)
        if bq == G.CB_QPW or bv + nv > G.DB_QW:
            bins.append(j)
            bq = bv = 0
        bq, bv = bq + 1, bv + nv
    assert len(bins) > G.GROUP_CHUNK * G.DB_WPR and n_q > G.GROUP_CHUNK * G.SM_QG
    _split_check(native, s, queries, 20, flt, (ex, None, six, sets), bins[G.GROUP_CHUNK * G.DB_WPR], 100_000,
                 names={"cos_blocked", "filtered"})
    _split_check(native, s, queries, 33, flt, (ex, None, six, sets), G.GROUP_CHUNK * G.SM_QG, 100_000,
                 names={"cos_multi", "filtered"})
    # white-listed cosine queries: one group each, so the listed route splits at GROUP_CHUNK queries
    n = LISTED_SPLIT
    lq = queries[:n]
    wl = rng.integers(-1, ni + 1, (n, 6))
    wl[:, 0] = [q[0] if len(q) else 0 for q in lq]        # a query id of its own in the white list
    for keep in (False, True):
        _split_check(native, s, lq, 5, (list(ex[:n]), list(wl), six[:n], sets), (ex[:n], wl, six[:n], sets),
                     G.GROUP_CHUNK, 20_000, keep=keep, names={"listed"})
    s.m.close()


# ---- h. a tie over 300 007 items under a filter -------------------------------------------------------------------------
@pytest.mark.parametrize("rank", OVERFLOW_RANKS)
def test_large_tie_survives_a_filter(native, rank):
    """the all-ties user: exclusions and a set row remove part of the tie, the survivors still number far more than
    any pool holds"""
    ni = OVERFLOW_ITEMS
    s, rng = random_model(native, ni, rank, rank)
    sets = np.zeros((1, ni), np.uint8)
    sets[0, :20_000:2] = 1
    ex = [list(range(0, 3000, 3)), [], list(range(100)) + [ni - 1], []]
    flt = (ex, None, np.array([0, -1, 0, -1], np.int32), sets)
    for topk in OVERFLOW_TOPKS:
        check_rec(native, s, [0, 0, 0, 1], topk, flt, names={"dot_batched", "filtered"})
    check_rec(native, s, [0, 0, 0, 1], 77, flt, weight=np.where(np.arange(ni) % 3 == 0, -1.0, 0.0))
    check_sim(native, s, [[0, 5], [0, 5]], 128, (ex[:2], None, np.array([0, -1], np.int32), sets))
    s.m.close()
