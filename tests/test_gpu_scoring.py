"""GPU: every top-k scoring path against the fp64 restatement in tests/scoring_ref.py, bit for bit.

pio_als.h promises that recommend / similar / similar_batch return results identical to the fp64 reference on every path,
ties going to the smaller item id.  Each case below compares ids, scores (as bits) and counts with scoring_ref and asserts
pio_als_stats.last_score_path, so it provably ran the kernels it names.  The dispatch (csrc/score_plan.h, DESIGN.md 4.6):

  R1 recommend, n == 1, KP <= 64, topk <= 128            score_one           S1 one query of 1..8 ids, KP <= 64, topk <= 128
  R2 n <= 16, topk <= 128                                dot_batched         S2 one query of 1..40 ids, topk <= 128
  R3 n > 16, KP <= 64, topk <= 32                        dot_blocked         S3 batch, KP <= 64, topk <= 32, <= 8 valid / query
  R4 otherwise, several passes above topk 128            dot_batched         S4 batch, <= 40 valid vectors per 8-query group
                                                                             S5 the rest, one query at a time: cos_batched if
                                                                                its shared memory fits 100 KB, else cos_fallback
"""
import os
import subprocess
import sys
import textwrap
from pathlib import Path

import numpy as np
import pytest

import scoring_ref

pytestmark = pytest.mark.gpu

# dispatch constants of topk_geometry.h / score_plan.h; tests/test_scoring_plan.py checks them, and the planner's rules,
# against the sources, and that the ladders below straddle each one
TK_MAXK, DB_MAXK, SB_QB, S1_MAXNV, SM_NV, SM_QG, SM_QIDS, DB_QW = 128, 32, 16, 8, 40, 8, 64, 8
CB_QPW, DB_WPR = 4, 2
SB_THREADS, SC_G, S5_SMEM_LIMIT, GROUP_CHUNK = 256, 8, 100 * 1024, 32768

RANKS = [1, 7, 16, 17, 33, 48, 63, 64, 65, 100, 127, 128]
ITEM_LADDER = [1, 2, 31, 33, 255, 257, 511, 513, 1023, 1025]
MULTI_TOPK = [129, 256, 257, 1000]
S2_QUERY_IDS = [40, 41]                     # ids of one similar query: S2 up to SM_NV ids (valid or not), S5 above
GROUP_VECTORS = [40, 41]                    # valid vectors of one 8-query batch group: S4 up to SM_NV, S5 above
S5_QUERY_VALID = [40, 41, 56, 57, 70]       # valid items (plus three invalid ids) of one S5 query at KP 64, topk 20:
                                            # the shared-memory / fallback kernel boundary lies between 56 and 57
LONG_QUERY_IDS = 70                         # > SM_QIDS: query ids read from global memory
TIE_BLOCKS = [(0, 3), (8, 5), (30, 5), (126, 5), (254, 5), (500, 300)]   # (first rank, length) of equal-score blocks
SPLIT_USERS, SPLIT_QUERIES = 600_000, 300_000   # above GROUP_CHUNK groups of SB_QB users / SM_QG queries


def kp_of(rank):
    return 16 if rank <= 16 else 32 if rank <= 32 else 64 if rank <= 64 else 128


def s5_smem(kp, nqv, nq, topk):
    nqp = (nqv + SC_G - 1) // SC_G * SC_G
    return 8 * (kp * nqp + nqp) + 4 * SB_THREADS * (kp + 4) + 12 * (SB_THREADS // 32) * min(topk, TK_MAXK) + 4 * nq + 16


def rec_path(kp, n, topk):
    if n == 1 and kp <= 64 and topk <= TK_MAXK:
        return {"score_one"}
    if n <= SB_QB and topk <= TK_MAXK:
        return {"dot_batched"}
    if kp <= 64 and topk <= DB_MAXK:
        return {"dot_blocked"}
    return {"dot_batched"} | ({"multi_pass"} if topk > TK_MAXK else set())


def _n_valid(q, ih):
    q = np.asarray(q, np.int64)
    q = q[(q >= 0) & (q < ih.shape[0])]
    return int(ih[q].astype(bool).sum())


def _s5_path(kp, q, ih, topk):
    nqv = _n_valid(q, ih)
    if nqv == 0:
        return set()
    p = {"cos_batched" if s5_smem(kp, nqv, len(q), topk) <= S5_SMEM_LIMIT else "cos_fallback"}
    return p | ({"multi_pass"} if topk > TK_MAXK else set())


def sim_path(kp, queries, ih, topk):
    if len(queries) == 1:
        nq = len(queries[0])
        if kp <= 64 and topk <= TK_MAXK and 1 <= nq <= S1_MAXNV:
            return {"score_one"}
        if 1 <= nq <= SM_NV and topk <= TK_MAXK:
            return {"cos_multi"}
    elif sum(len(q) for q in queries) > 0:
        nv = [_n_valid(q, ih) for q in queries]
        if kp <= 64 and topk <= DB_MAXK and max(nv) <= DB_QW:
            return {"cos_blocked"}
        if max(sum(nv[g:g + SM_QG]) for g in range(0, len(nv), SM_QG)) <= SM_NV:
            return {"cos_multi"} | ({"multi_pass"} if topk > TK_MAXK else set())
    return set().union(*[_s5_path(kp, q, ih, topk) for q in queries])


def _same(got, want, what):
    gi, gs, gc = got
    wi, ws, wc = want
    assert np.array_equal(np.asarray(gc), np.asarray(wc)), (what, "count", gc, wc)
    bad = np.flatnonzero(~(np.asarray(gi) == np.asarray(wi)).reshape(-1))
    assert bad.size == 0, (what, "items", bad[:8], np.asarray(gi).reshape(-1)[bad[:8]], np.asarray(wi).reshape(-1)[bad[:8]])
    assert np.array_equal(np.asarray(gs, np.float32).view(np.uint32), np.asarray(ws, np.float32).view(np.uint32)), (what, "scores")


class Scorer:
    """A handle plus the factors it scores (get_factors / the imported arrays) and the checks against scoring_ref."""

    def __init__(self, m, uf, itf, uh, ih):
        self.m, self.uf, self.itf, self.uh, self.ih = m, uf, itf, uh, ih
        self.kp = kp_of(itf.shape[1])

    def path(self):
        return self.m.stats()["last_score_path"]

    def rec(self, users, topk, path=None, mask=None, weight=None):
        users = np.asarray(users, np.int32)
        got = self.m.recommend(users, topk, mask, weight)
        p = self.path()
        want = scoring_ref.recommend(self.uf, self.uh, self.itf, self.ih, users, topk, mask, weight)
        what = ("recommend", self.kp, len(users), topk, mask is not None, weight is not None)
        _same(got, want, what)
        assert p == (rec_path(self.kp, len(users), topk) if path is None else path), (what, p)
        return got

    def sim(self, queries, topk, mask=None, weight=None, keep=False, batch=None):
        """queries: a list of id lists; one query goes through similar() unless batch is set."""
        if len(queries) == 1 and not batch:
            gi, gs, gc = self.m.similar(np.asarray(queries[0], np.int32), topk, mask, weight, keep)
            got = (gi[None], gs[None], np.array([gc]))
        else:
            got = self.m.similar_batch(queries, topk, mask, weight, keep)
        p = self.path()
        want = scoring_ref.similar_batch(self.itf, self.ih, queries, topk, mask, weight, keep)
        what = ("similar", self.kp, [len(q) for q in queries][:4], topk, mask is not None, weight is not None, keep)
        _same(got, want, what)
        assert p == sim_path(self.kp, queries, self.ih, topk), (what, p)
        return got


# ---- a. controlled values in a degree-permuted layout -----------------------------------------------------------------
def _designed_rows(k, rng):
    """Item rows whose score order (for the user e_0, and as cosines to the item e_0) is fixed by their slot; each slot
    is a block of bit-identical rows, placed so that the blocks straddle topk 1, 10, 32/33, 128/129, 256/257."""
    sizes, pos = [], 0
    for start, length in TIE_BLOCKS:
        sizes += [1] * (start - pos)
        sizes.append(length)
        pos = start + length
    sizes += [1] * 24
    pattern = rng.standard_normal(k).astype(np.float32)
    rows = []
    for p, size in enumerate(sizes):
        c = np.float32(2.0 - p / 1000.0)
        row = np.zeros(k, np.float32)
        row[0] = c
        if k > 1:
            row[1] = c * np.float32(0.01 * p)
        if k > 2:
            row[2:] = c * np.float32(1e-3) * pattern[2:]
        rows += [row] * size
    return np.array(rows, np.float32)


def controlled(native, rank, seed=0, n_users=40):
    """NativeALS with set_ratings whose item degrees rise with the item id (the degree-descending internal order scans
    the external order backwards, and the smallest id of a tie block last), hand-made set_init factors, no training.
    Returns (Scorer, anchor item id, designed item ids in rank order)."""
    rng = np.random.default_rng(seed)
    k = rank
    designed = _designed_rows(k, rng)
    n_rand, n_off, nd = 300, 60, designed.shape[0]
    ni = nd + 3 + n_rand + n_off
    ids = rng.permutation(ni)
    d_ids, anchor, r_ids, off_ids = ids[:nd], int(ids[nd]), ids[nd + 3:nd + 3 + n_rand], ids[ni - n_off:]
    lone = [int(ids[nd + 1]), int(ids[nd + 2])]    # e_(k-1), e_(k-2): cosine 1 with themselves, ~0 with the rest
    itf0 = np.zeros((ni, k), np.float32)
    itf0[d_ids] = designed
    itf0[anchor, 0] = 1.0
    itf0[lone[0], k - 1] = itf0[lone[1], k - 2] = 1.0
    rnd = rng.standard_normal((n_rand, k)).astype(np.float32)
    rnd[:, 0] = -np.abs(rnd[:, 0]) - 0.5           # below every designed item for the user e_0, cosine < 0 to the anchor
    itf0[r_ids] = rnd
    itf0[off_ids] = rng.standard_normal((n_off, k)).astype(np.float32)
    itf0[off_ids, 0] = 5.0                         # would win everything if a factor-less row were ever scored
    off_users = np.array([3, 17, 29])
    uf0 = rng.standard_normal((n_users, k)).astype(np.float32)
    uf0[0] = 0.0
    uf0[0, 0] = 1.0                                # the tie user e_0
    uf0[1] = 0.0                                   # the zero user: every score is 0, the ranking is pure id order
    # ratings: degree 1 + (position among active items) * D / n_active -- rising with the id
    active_items = np.setdiff1d(np.arange(ni), off_ids)
    active_users = np.setdiff1d(np.arange(n_users), off_users)
    na = active_items.shape[0]
    D = max(1, min(na, 400_000 // na))
    deg = 1 + (np.arange(na) * D) // na
    item = np.repeat(active_items, deg)
    user = rng.choice(active_users, item.shape[0])
    user[:active_users.shape[0]] = active_users    # every active user owns a rating
    rating = rng.random(item.shape[0]).astype(np.float32) + 0.5
    m = native.NativeALS(rank, n_users, ni, lam=0.01)
    m.set_ratings(user, item, rating)
    m.set_init(uf0, itf0)
    uf, itf, uh, ih = m.get_factors()
    assert ih.sum() == na and not ih[off_ids].any() and not itf[off_ids].any()
    assert uh.sum() == n_users - off_users.shape[0] and not uh[off_users].any() and not uf[off_users].any()
    assert np.array_equal(itf[ih == 1], itf0[ih == 1]) and np.array_equal(uf[uh == 1], uf0[uh == 1])
    order = d_ids   # designed items in slot order = rank order for e_0
    s = Scorer(m, uf, itf, uh, ih)
    s.lone = lone
    return s, anchor, order, off_ids


def _mask_weight(ni, rng):
    mask = (rng.random(ni) < 0.08).astype(np.uint8)
    weight = rng.choice(np.array([0.0, -1.0, 0.5, 1.0, 2.0]), ni)
    return mask, weight


def _long_query(rng, s, anchor, order, off_ids, n_valid, n_ids):
    """n_ids query ids, n_valid of them valid: high-ranked designed items first and last (the exclusion must see both
    ends of the list), the rest factor-less, out-of-range or negative."""
    ni = s.ih.shape[0]
    valid = [int(order[0])] + list(rng.choice(order[1:], n_valid - 2, replace=False)) + [anchor] if n_valid >= 2 else [anchor]
    valid = valid[:n_valid]
    filler = list(rng.choice(np.concatenate([off_ids, [ni, ni + 7, -1]]), n_ids - n_valid))
    q = [valid[0]] + filler + valid[1:]
    return [int(v) for v in q]


@pytest.mark.parametrize("rank", [16, 24, 40, 100])
def test_controlled_recommend(native, rank):
    s, anchor, order, off_ids = controlled(native, rank)
    kp = s.kp
    rng = np.random.default_rng(rank)
    mask, weight = _mask_weight(s.ih.shape[0], rng)
    few = [0, 1, 2, 3, 4, 5]
    many = list(range(40))
    cases = []
    if kp <= 64:
        cases += [([u], t) for u in (0, 1, 2, 3) for t in (1, 10, 33, 128)]          # R1
    cases += [(few, t) for t in (1, 10, 32, 33, 128)] + [([0, 1], 100)]             # R2
    cases += [(many, t) for t in (1, 10, 32)]                                      # R3 (R4 at KP 128)
    cases += [(many, t) for t in (33, 128, 129, 256, 257, 1000)] + [(few, 129)]    # R4
    for users, topk in cases:
        s.rec(users, topk)
        s.rec(users, topk, mask=mask, weight=weight)
    # signed zeros: weights 0 and -1 on the zero user give +0 and -0 scores that tie in id order across every list and pass
    w01 = np.where(np.arange(s.ih.shape[0]) % 2 == 0, 0.0, -1.0)
    for users, topk in (([1], 128), ([1, 0], 128), (many, 32), (many, 257)):
        s.rec(users, topk, weight=w01)
    # exactly 128 and 256 candidates: the last pass finds nothing left
    act = np.flatnonzero(s.ih)
    for n_cand in (128, 256):
        mk = np.ones(s.ih.shape[0], np.uint8)
        mk[act[rng.permutation(act.shape[0])[:n_cand]]] = 0
        for topk in (128, 129, 256, 257):
            s.rec(many, topk, mask=mk)
            s.rec(few, topk, mask=mk)


@pytest.mark.parametrize("rank", [16, 24, 40, 100])
def test_controlled_similar(native, rank):
    s, anchor, order, off_ids = controlled(native, rank)
    kp = s.kp
    rng = np.random.default_rng(rank + 1)
    ni = s.ih.shape[0]
    mask, weight = _mask_weight(ni, rng)
    top = [int(v) for v in order[:3]]
    q8 = [anchor, top[0], int(off_ids[0]), ni + 2, anchor, -1, top[2], int(order[40])]
    q20 = _long_query(rng, s, anchor, order, off_ids, 14, 20)
    for keep in (False, True):
        for topk in (1, 10, 33, 128):
            for q in ([anchor], [anchor, top[1]], q8, q20, [int(off_ids[0]), int(off_ids[1])]):
                s.sim([q], topk, keep=keep)                          # S1 (S2 at KP 128) / S2
                s.sim([q], topk, mask=mask, weight=weight, keep=keep)
    batch = [[anchor], [top[0], top[1]], q8, [], [int(off_ids[2])], [anchor, anchor], [int(order[200])], [ni + 1]] * 3
    for topk in (1, 10, 32):
        s.sim(batch, topk)                                           # S3 (S4 at KP 128)
        s.sim(batch, topk, mask=mask, weight=weight, keep=True)
    for topk in (33, 128) + tuple(MULTI_TOPK):
        s.sim(batch, topk)                                           # S4
        s.sim(batch, topk, mask=mask, weight=weight)
    # a batch query of more than SM_QIDS ids (global-memory exclusion), <= 40 valid vectors in its group
    long_ids = _long_query(rng, s, anchor, order, off_ids, 12, LONG_QUERY_IDS)
    for topk in (10, 33, 129):
        s.sim([long_ids, [anchor], [top[0]]], topk)
        s.sim([[anchor], long_ids], topk, keep=True)
    # the first and the last of the ids are the two best candidates unless they are excluded, in a batch (S4, ids in
    # global memory) and as one query (S5)
    ends = [s.lone[0]] + [int(v) for v in rng.choice(np.concatenate([off_ids, [ni, ni + 7, -1]]), LONG_QUERY_IDS - 2)]
    ends.append(s.lone[1])
    for topk in (10, 33, 129):
        s.sim([ends, [anchor]], topk)
        s.sim([ends], topk)
    # S5: one query with more than 40 items, or topk above 128; a batch group with more than 40 vectors
    for nv in S5_QUERY_VALID:
        q = _long_query(rng, s, anchor, order, off_ids, nv, nv + 3)
        s.sim([q], 20)
        s.sim([q], 129, mask=mask, weight=weight)
    for topk in MULTI_TOPK:
        s.sim([[anchor]], topk)
        s.sim([q8], topk, keep=True)
    # the S2 / S5 split counts query ids: SM_NV ids, some of them invalid, take S2; one more takes S5
    for n_ids in S2_QUERY_IDS:
        q = _long_query(rng, s, anchor, order, off_ids, n_ids - 6, n_ids)
        assert len(q) == n_ids
        for topk in (20, 128):
            s.sim([q], topk)
            s.sim([q], topk, mask=mask, weight=weight, keep=True)
    # the S4 / S5 split counts the valid vectors of an 8-query group: exactly SM_NV take S4, one more takes S5; 8 x 5
    # vectors at topk > 32 and 4 x 10 at topk 20 (a query of more than DB_QW vectors keeps it off the blocked kernel)
    for n_vec in GROUP_VECTORS:
        for n_q, topks in ((8, (33, 129)), (4, (20,))):
            group = [_long_query(rng, s, anchor, order, off_ids, n_vec // n_q, n_vec // n_q + 2) for _ in range(n_q)]
            group[-1].append(int(order[-1]) if n_vec % n_q else ni + 5)
            assert sum(_n_valid(q, s.ih) for q in group) == n_vec
            for topk in topks:
                s.sim(group + [[ni + 1]] * (SM_QG - n_q) + [[anchor], [top[0]]], topk)
                s.sim(group, topk, mask=mask, weight=weight)
    big = [_long_query(rng, s, anchor, order, off_ids, 9, 10) for _ in range(5)]
    s.sim(big, 20)
    s.sim(big, 257)
    # all-factor-less and empty queries
    s.sim([[int(off_ids[3])]], 10)
    s.sim([[int(v) for v in off_ids[:50]]], 10)
    s.sim([[], []], 10)
    s.sim([[]], 10)
    # exactly 128 and 256 candidates for the anchor query
    for n_cand in (128, 256):
        mk = np.ones(ni, np.uint8)
        mk[order[rng.permutation(order.shape[0])[:n_cand]]] = 0
        for topk in (128, 129, 256, 257):
            s.sim([[anchor]], topk, mask=mk)
            s.sim([[anchor]] * 9, topk, mask=mk)


# ---- b. rank ladder on trained handles (guards the zero padding of the factor columns) -------------------------------
def _trained(native, monkeypatch, rank, env):
    """Two iterations on the solve kernel `env` selects; the phase_ms() labels prove which one ran on both sides."""
    from pio_b200 import synth
    from test_gpu_halfstep import path_of, set_env
    set_env(monkeypatch, env)
    nu, ni, nnz = 600, 900, 30000
    u, i, r = synth.synth_ratings(nu, ni, nnz, seed=rank, implicit=False)
    keep = (i % 37 != 5) & (u % 41 != 7)           # items and users without a rating
    m = native.NativeALS(rank, nu, ni, lam=0.05)
    m.set_ratings(u[keep], i[keep], r[keep])
    m.set_init(synth.synth_init_factors(nu, rank, 1, 0), synth.synth_init_factors(ni, rank, 1, 1))
    m.run(2)
    ph, label = m.phase_ms(), path_of(rank, env)[0]
    assert (ph["item_kernel"], ph["user_kernel"]) == (label, label), (rank, env, ph)
    uf, itf, uh, ih = m.get_factors()
    return Scorer(m, uf, itf, uh, ih)


def _all_paths(s, rng):
    ni = s.ih.shape[0]
    mask, weight = _mask_weight(ni, rng)
    act = np.flatnonzero(s.ih)
    users = list(range(40))
    for users_, topk in (([5], 10), ([41 * 3 + 7], 10), ([0, 5, 9], 50), (users, 10), (users, 33), (users, 200)):
        s.rec(users_, topk)
        s.rec(users_, topk, mask=mask, weight=weight)
    q3 = [int(v) for v in act[:3]]
    q12 = [int(v) for v in rng.choice(act, 12)]
    q60 = [int(v) for v in rng.choice(act, 60, replace=False)]
    for queries, topk in (([q3], 10), ([q12], 40), ([q3, q12[:5], [int(act[7])]], 10), ([q3, q12], 40), ([q60], 20),
                          ([q3], 150), ([q12] * 5, 20)):
        s.sim(queries, topk)
        s.sim(queries, topk, mask=mask, weight=weight)


@pytest.mark.parametrize("rank", RANKS)
def test_rank_ladder_trained(native, monkeypatch, rank):
    _all_paths(_trained(native, monkeypatch, rank, {}), np.random.default_rng(rank))


# at KP 128 every setting runs the one FP32 kernel, so rank 100 has no variant beyond test_rank_ladder_trained[100]
@pytest.mark.parametrize("rank,env", [(33, {"PIO_ALS_MMA": "0"}), (33, {"PIO_ALS_MMA": "1"}), (33, {"PIO_ALS_TC": "1"}),
                                      (48, {"PIO_ALS_MMA": "0"}), (48, {"PIO_ALS_MMA": "1"}), (48, {"PIO_ALS_TC": "1"})])
def test_rank_ladder_solve_variants(native, monkeypatch, rank, env):
    _all_paths(_trained(native, monkeypatch, rank, env), np.random.default_rng(rank))


# ---- c. item-count ladder --------------------------------------------------------------------------------------------
def _imported(native, n_items, rank, seed, n_users=40):
    rng = np.random.default_rng(seed)
    itf = rng.standard_normal((n_items, rank)).astype(np.float32)
    itf[1::7] = itf[0]                              # tie blocks
    ih = (rng.random(n_items) > 0.1).astype(np.uint8)
    ih[0] = 1
    itf[ih == 0] = 0.0
    uf = rng.standard_normal((n_users, rank)).astype(np.float32)
    uf[0] = 0.0                                     # the all-ties user
    uh = np.ones(n_users, np.uint8)
    m = native.NativeALS.from_factors(uf, itf, uh, ih)
    return Scorer(m, uf, itf, uh, ih), rng


def _item_ladder():
    from pio_b200 import native as n
    sm = n.NativeALS.from_factors(np.ones((1, 4), np.float32), np.ones((1, 4), np.float32)).stats()["sm_count"]
    return ITEM_LADDER + [256 * sm - 1, 256 * sm + 1]


@pytest.mark.parametrize("rank", [40, 100])
def test_item_count_ladder(native, rank):
    for ni in _item_ladder():
        s, rng = _imported(native, ni, rank, ni)
        ids = lambda c: [int(v) for v in rng.integers(-1, ni + 3, c)]   # noqa: E731  (some unknown / out of range)
        for users, topk in (([0], ni + 5), ([2], 10), ([0, 3], 128), (list(range(20)), 10), (list(range(20)), ni + 5),
                            (list(range(20)), 129)):
            s.rec(users, topk)
        for queries, topk in (([[0, 1]], ni + 5), ([ids(12)], 20), ([ids(3) for _ in range(10)], 10),
                              ([ids(5) for _ in range(10)], ni + 5), ([ids(50)], 20), ([ids(5)], 129)):
            s.sim(queries, topk)


def test_large_matrix_fused_merge_overflow(native):
    """~300k items: the all-ties user at topk 128 leaves more survivors than the fused final merge holds, at each KP."""
    for rank in (8, 24, 40):
        s, rng = _imported(native, 300_007, rank, rank)
        s.rec([0], 128)
        s.rec([0], 77, weight=np.where(np.arange(300_007) % 3 == 0, -1.0, 0.0))
        s.rec([1], 128)
        s.sim([[0, 5]], 128)
    s.rec([0, 1, 2], 129)
    s.sim([[0, 5]], 300)


# ---- f. the grid.y split of the batch paths (more than 32768 query groups per launch) --------------------------------
def _split_rows(n, chunk, rng):
    rows = set(rng.choice(n, 2000, replace=False).tolist())
    for b in range(chunk, n, chunk):
        rows.update(range(max(0, b - 2000), min(n, b + 2000)))
    return np.array(sorted(rows))


def test_grid_split_recommend(native):
    n_users, ni, rank = SPLIT_USERS, 700, 8
    rng = np.random.default_rng(11)
    uf = rng.standard_normal((n_users, rank)).astype(np.float32)
    uf[::1000] = 0.0
    uh = (rng.random(n_users) > 0.1).astype(np.uint8)
    uf[uh == 0] = 0.0
    itf = rng.standard_normal((ni, rank)).astype(np.float32)
    itf[3::50] = itf[1]
    m = native.NativeALS.from_factors(uf, itf, uh, None)
    s = Scorer(m, uf, itf, uh, np.ones(ni, np.uint8))
    users = np.arange(n_users, dtype=np.int32)
    rows = _split_rows(n_users, GROUP_CHUNK * SB_QB, rng)
    for topk in (10, 33):
        gi, gs, gc = m.recommend(users, topk)
        assert s.path() == rec_path(s.kp, n_users, topk)
        want = scoring_ref.recommend(uf, uh, itf, None, users[rows], topk)
        _same((gi[rows], gs[rows], gc[rows]), want, ("split recommend", topk))
        # the whole output against the same users scored in calls below the split
        for c0 in range(0, n_users, 200_000):
            part = m.recommend(users[c0:c0 + 200_000], topk)
            _same((gi[c0:c0 + 200_000], gs[c0:c0 + 200_000], gc[c0:c0 + 200_000]), part, ("split vs parts", topk, c0))


def test_grid_split_similar_batch(native):
    n_q, ni, rank = SPLIT_QUERIES, 600, 8
    rng = np.random.default_rng(12)
    itf = rng.standard_normal((ni, rank)).astype(np.float32)
    ih = (rng.random(ni) > 0.1).astype(np.uint8)
    itf[ih == 0] = 0.0
    m = native.NativeALS.from_factors(None, itf, None, ih)
    s = Scorer(m, None, itf, None, ih)
    lens = rng.integers(0, 4, n_q)
    flat = rng.integers(-1, ni + 2, int(lens.sum())).astype(np.int32)
    ptr = np.concatenate([[0], np.cumsum(lens)])
    queries = [flat[ptr[j]:ptr[j + 1]] for j in range(n_q)]
    # the blocked kernel packs consecutive queries into bins of <= CB_QPW queries and <= DB_QW vectors, DB_WPR bins per group
    bins, bq, bv = [0], 0, 0
    for j, q in enumerate(queries):
        nv = _n_valid(q, ih)
        if bq == CB_QPW or bv + nv > DB_QW:
            bins.append(j)
            bq = bv = 0
        bq, bv = bq + 1, bv + nv
    assert len(bins) > GROUP_CHUNK * DB_WPR
    for topk, chunk in ((20, bins[GROUP_CHUNK * DB_WPR]), (33, GROUP_CHUNK * SM_QG)):
        gi, gs, gc = m.similar_batch(queries, topk)
        assert s.path() == sim_path(s.kp, queries, ih, topk)
        rows = _split_rows(n_q, chunk, rng)
        want = scoring_ref.similar_batch(itf, ih, [queries[j] for j in rows], topk)
        _same((gi[rows], gs[rows], gc[rows]), want, ("split similar", topk))
        for c0 in range(0, n_q, 100_000):
            part = m.similar_batch(queries[c0:c0 + 100_000], topk)
            _same((gi[c0:c0 + 100_000], gs[c0:c0 + 100_000], gc[c0:c0 + 100_000]), part, ("split vs parts", topk, c0))


# ---- g. call sequences that lower another call site's shared-memory limit ------------------------------------------------
_SEQUENCE = textwrap.dedent("""
    import sys
    import numpy as np
    sys.path[:0] = [sys.argv[1], sys.argv[1] + "/tests"]
    import pio_b200
    from pio_b200 import native
    import scoring_ref
    rank = int(sys.argv[2])
    rng = np.random.default_rng(rank)
    uf = rng.standard_normal((200, rank)).astype(np.float32)
    itf = rng.standard_normal((5000, rank)).astype(np.float32)
    m = native.NativeALS.from_factors(uf, itf)
    def same(got, want):
        return (np.array_equal(got[0], want[0]) and np.array_equal(got[2], want[2]) and
                np.array_equal(np.asarray(got[1], np.float32).view(np.uint32), want[1].view(np.uint32)))
    def outcome(ok):
        return ("ok:" if ok else "stale:") + ",".join(sorted(m.stats()["last_score_path"]))
    def rec(users, topk):
        users = np.asarray(users, np.int32)
        try:
            got = m.recommend(users, topk)
        except native.NativeError as e:
            return "error%d" % e.code
        return outcome(same(got, scoring_ref.recommend(uf, None, itf, None, users, topk)))
    def sim(queries, topk):
        try:
            got = m.similar_batch(queries, topk) if len(queries) > 1 else m.similar(queries[0], topk)
        except native.NativeError as e:
            return "error%d" % e.code
        got = got if len(queries) > 1 else (got[0][None], got[1][None], np.array([got[2]]))
        return outcome(same(got, scoring_ref.similar_batch(itf, None, queries, topk)))
    out = [rec([0, 1], 100), rec(list(range(100)), 40), rec([2, 3], 100),
           sim([list(range(20))], 128), sim([[j] for j in range(100, 300)], 33), sim([list(range(20, 40))], 128)]
    print(" ".join(out))
""")


@pytest.mark.parametrize("rank", [64, 128])
def test_call_sequence_shared_memory_limit(native, rank):
    """recommend top-100 of 2 users (R2), then 100 users top-40 (R4, same kernel, smaller shared memory), then top-100
    of 2 other users again; the same on the similar side (S2 top-128, S4 top-33, S2).  A fresh interpreter: the limits
    are per process."""
    root = str(Path(__file__).resolve().parent.parent)
    r = subprocess.run([sys.executable, "-c", _SEQUENCE, root, str(rank)], capture_output=True, text=True, timeout=600,
                       env=dict(os.environ))
    assert r.returncode == 0, r.stderr[-3000:]
    # steps 1-3 on score_dot_topk_batched_kernel (R2, R4, R2), steps 4-6 on score_cos_topk_multi_kernel (S2, S4, S2)
    assert r.stdout.split() == ["ok:dot_batched"] * 3 + ["ok:cos_multi"] * 3, r.stdout
