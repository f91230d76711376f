"""CPU: tests/filtered_ref.py against the definition taken query by query (dense mask + scoring_ref), on hand-computed
cases, and the ladders of tests/test_gpu_filtered_bounds.py against the constants in the CUDA sources."""
import re
from pathlib import Path

import numpy as np
import pytest

import filtered_ref as FR
import scoring_ref
import test_gpu_filtered as F
import test_gpu_filtered_bounds as B
import test_gpu_scoring as G

CSRC = Path(__file__).resolve().parent.parent / "incubator-predictionio_b200" / "csrc"


def _model(rng, n_users, n_items, rank, ties=True):
    uf = rng.standard_normal((n_users, rank)).astype(np.float32)
    itf = rng.standard_normal((n_items, rank)).astype(np.float32)
    if ties:
        itf[1::5] = itf[0]
    uf[0] = 0.0
    uh = (rng.random(n_users) > 0.1).astype(np.uint8)
    ih = (rng.random(n_items) > 0.1).astype(np.uint8)
    uf[uh == 0] = 0
    itf[ih == 0] = 0
    return uf, uh, itf, ih


def _per_query_rec(uf, uh, itf, ih, users, topk, mask, weight, flt):
    ex, wl, six, sets = flt
    out = [scoring_ref.recommend(uf, uh, itf, ih, users[j:j + 1], topk,
                                 F.dense_mask(itf.shape[0], mask, ex, wl, six, sets, j), weight)
           for j in range(len(users))]
    return tuple(np.concatenate([o[t] for o in out]) for t in range(3))


def _per_query_sim(itf, ih, queries, topk, mask, weight, keep, flt):
    ex, wl, six, sets = flt
    out = [scoring_ref.similar(itf, ih, queries[j], topk, F.dense_mask(itf.shape[0], mask, ex, wl, six, sets, j), weight,
                               keep) for j in range(len(queries))]
    return np.array([o[0] for o in out]), np.array([o[1] for o in out]), np.array([o[2] for o in out], np.int32)


@pytest.mark.parametrize("seed", range(6))
def test_agrees_with_the_dense_mask_per_query(seed):
    rng = np.random.default_rng(seed)
    n_items = [1, 31, 33, 64, 150][seed % 5]
    uf, uh, itf, ih = _model(rng, 30, n_items, [1, 7, 16, 33][seed % 4])
    n = 23
    users = rng.integers(-2, 32, n).astype(np.int32)
    queries = [[int(v) for v in rng.integers(-2, n_items + 2, rng.integers(0, 5))] for _ in range(n)]
    mask = (rng.random(n_items) < 0.1).astype(np.uint8) if seed % 2 else None
    weight = rng.choice([0.0, -0.0, -1.0, 0.5, 2.0], n_items) if seed % 3 else None
    for topk in (1, 5, n_items + 3):
        flt = F.random_filter(rng, n, n_items, None, white_share=0.4)
        got = FR.recommend(uf, uh, itf, ih, users, topk, mask, weight, *flt)
        G._same(got, _per_query_rec(uf, uh, itf, ih, users, topk, mask, weight, flt), ("recommend", seed, topk))
        for keep in (False, True):
            got = FR.similar_batch(itf, ih, queries, topk, mask, weight, keep, *flt)
            G._same(got, _per_query_sim(itf, ih, queries, topk, mask, weight, keep, flt), ("similar", seed, topk, keep))


def test_chunks_do_not_change_the_result(monkeypatch):
    rng = np.random.default_rng(7)
    uf, uh, itf, ih = _model(rng, 50, 200, 8)
    users = rng.integers(0, 50, 40).astype(np.int32)
    queries = [[int(v) for v in rng.integers(0, 200, 3)] for _ in range(40)]
    flt = F.random_filter(rng, 40, 200, None, white_share=0.3)
    a = FR.recommend(uf, uh, itf, ih, users, 12, None, None, *flt)
    b = FR.similar_batch(itf, ih, queries, 12, None, None, False, *flt)
    monkeypatch.setattr(FR, "_chunk", lambda n_items: 3)
    G._same(FR.recommend(uf, uh, itf, ih, users, 12, None, None, *flt), a, "recommend chunks")
    G._same(FR.similar_batch(itf, ih, queries, 12, None, None, False, *flt), b, "similar chunks")


def _identity_items(n_items):
    """user x = e_0 and item i scoring n_items - i: the ranking is the id order, scores known exactly"""
    itf = np.zeros((n_items, 2), np.float32)
    itf[:, 0] = n_items - np.arange(n_items)
    uf = np.array([[1.0, 0.0]], np.float32)
    return uf, itf


def test_hand_computed_cases():
    uf, itf = _identity_items(10)
    u = np.zeros(1, np.int32)

    def rec(topk, ex=None, wl=None, six=None, sets=None, ih=None):
        return FR.recommend(uf, None, itf, ih, u, topk, None, None, ex, wl, six, sets)

    # an empty white list: no candidates, padded with -1 / 0
    i, s, c = rec(3, wl=[[]])
    assert c[0] == 0 and (i == -1).all() and (s == 0).all()
    # a white list meeting the exclusions
    i, s, c = rec(4, ex=[[2, 5]], wl=[[5, 2, 7, 1]])
    assert list(i[0]) == [1, 7, -1, -1] and c[0] == 2 and list(s[0]) == [9.0, 3.0, 0.0, 0.0]
    # a white list of invalid or factor-less ids only
    ih = np.ones(10, np.uint8)
    ih[[3, 4]] = 0
    i, s, c = rec(5, wl=[[-1, 10, 2 ** 31 - 1, 3, 4]], ih=ih)
    assert c[0] == 0 and (i == -1).all()
    # set_ix -1 names no row; a set row removes its items; duplicates and out-of-range ids in the exclusions
    sets = np.zeros((2, 10), np.uint8)
    sets[1, [0, 1]] = 1
    i, s, c = rec(3, six=np.array([-1], np.int32), sets=sets)
    assert list(i[0]) == [0, 1, 2]
    i, s, c = rec(3, six=np.array([1], np.int32), sets=sets)
    assert list(i[0]) == [2, 3, 4]
    i, s, c = rec(3, ex=[[0, 0, -4, 10, 99, 1, 1]])
    assert list(i[0]) == [2, 3, 4] and c[0] == 3
    # duplicates in a white list count once; topk above the candidates pads
    i, s, c = rec(6, wl=[[8, 8, 9, 9, 9]])
    assert list(i[0]) == [8, 9, -1, -1, -1, -1] and c[0] == 2 and list(s[0][:2]) == [2.0, 1.0]
    # an unknown user has no candidates whatever its filter
    i, s, c = FR.recommend(uf, None, itf, None, np.array([1, -1], np.int32), 2, None, None, [[], []], [None, [0]])
    assert (c == 0).all() and (i == -1).all()
    # similar: the query's own ids go unless kept, also when white-listed; score > 0 only
    itf2 = np.array([[1, 0], [1, 0], [0, 1], [-1, 0], [1, 1]], np.float32)
    i, s, c = FR.similar_batch(itf2, None, [[0], [0]], 5, None, None, False, None, [[0, 1, 2, 3, 4], None])
    assert list(i[0]) == [1, 4, -1, -1, -1] and list(i[1]) == [1, 4, -1, -1, -1]
    i, s, c = FR.similar_batch(itf2, None, [[0], [0]], 5, None, None, True, None, [[0, 1, 2, 3, 4], [1]])
    assert list(i[0]) == [0, 1, 4, -1, -1] and list(i[1]) == [1, -1, -1, -1, -1] and list(c) == [3, 1]


def test_signed_zero_scores_tie_in_id_order():
    uf = np.zeros((1, 3), np.float32)
    itf = np.ones((8, 3), np.float32)
    w = np.where(np.arange(8) % 2 == 0, 0.0, -1.0)          # +0 and -0 scores
    i, s, c = FR.recommend(uf, None, itf, None, np.zeros(1, np.int32), 8, None, w, [[0, 3]], None)
    assert list(i[0]) == [1, 2, 4, 5, 6, 7, -1, -1] and c[0] == 6
    assert list(np.signbit(s[0][:6])) == [True, False, False, True, False, True]


# ---- the ladders of the GPU file straddle the constants of the sources ------------------------------------------------
def _constants():
    env = {}
    for f in ("topk_geometry.h", "score_plan.h"):
        for name, expr in re.findall(r"^constexpr int (\w+) = ([^;]+);", (CSRC / f).read_text(), re.M):
            env[name] = int(eval(expr, {}, dict(env)))   # integer literals and earlier constants only
    return env


def _straddles(ladder, c):
    return c in ladder and c + 1 in ladder


def test_ladders_straddle_the_constants():
    c = _constants()
    assert (B.LS_THREADS, G.DB_QW, G.SM_NV, G.SM_QIDS, G.DB_MAXK, G.TK_MAXK, G.GROUP_CHUNK) == (
        c["LS_THREADS"], c["DB_QW"], c["SM_NV"], c["SM_QIDS"], c["DB_MAXK"], c["TK_MAXK"], c["GROUP_CHUNK"])
    assert (G.SM_QG, G.DB_WPR, G.CB_QPW, G.SB_QB) == (c["SM_QG"], c["DB_WPR"], c["CB_QPW"], c["SB_QB"])
    # the warp width and the 32-bit set word: the listed kernel takes 32 entries per warp, LS_THREADS per step
    src = (CSRC / "topk.cuh").read_text()
    assert "base += LS_THREADS" in src and "warp * 32" in src and "ext >> 5" in src and "ext & 31" in src
    assert B.WARP == 32 and B.SET_WORD == 32 and c["LS_WARPS"] * B.WARP == c["LS_THREADS"]
    # white-list lengths around a warp and a CTA step, and duplicates placed across both
    for b in (B.WARP, c["LS_THREADS"]):
        assert {b - 1, b, b + 1} <= set(B.WL_LENGTHS) and b - 1 in B.WL_DUPS
    assert 0 in B.WL_LENGTHS and 1 in B.WL_LENGTHS and max(B.WL_LENGTHS) > 2 * c["LS_THREADS"]
    # item counts around one and two set words
    for b in (B.SET_WORD, 2 * B.SET_WORD):
        assert {b - 1, b, b + 1} <= set(B.SET_ITEMS)
    # the similar dispatch: valid vectors per query (DB_QW), per group (SM_NV), ids per query (SM_QIDS)
    assert _straddles(B.QUERY_VALID, c["DB_QW"]) and _straddles(B.GROUP_VECTORS, c["SM_NV"])
    assert _straddles(B.QUERY_IDS, c["SM_QIDS"])
    # the S5 kernel split lies between the two valid-vector counts (KP 64, topk 20, three invalid ids)
    lo, hi = B.S5_VALID
    assert hi == lo + 1
    assert G.s5_smem(64, lo, lo + 3, 20) <= G.S5_SMEM_LIMIT < G.s5_smem(64, hi, hi + 3, 20)
    # topk around the blocked limit and the pass size, on the recommend side, the ties and the exhaustion cases
    for ladder in (B.REC_TOPKS, B.TIE_TOPKS):
        assert _straddles(ladder, c["DB_MAXK"]) and _straddles(ladder, c["TK_MAXK"])
    assert _straddles(B.TIE_TOPKS, 2 * c["TK_MAXK"]) and 1 in B.TIE_TOPKS
    assert set(B.EXHAUST) == {c["TK_MAXK"], 2 * c["TK_MAXK"]}
    for n in B.EXHAUST:
        assert _straddles(B.EXHAUST_TOPKS, n)
    # recommend user counts: one, the arena limit SB_QB and one more (a filtered call takes neither route)
    assert B.REC_USERS == [1, c["SB_QB"], c["SB_QB"] + 1]
    # the grid split: listed queries (one group each), cos_blocked bins and cos_multi groups past GROUP_CHUNK
    assert c["GROUP_CHUNK"] < B.LISTED_SPLIT < 2 * c["GROUP_CHUNK"]
    assert G.SPLIT_QUERIES > c["GROUP_CHUNK"] * c["SM_QG"]
    # the large tie: more survivors than any pool holds, at topk below, at and above one pass
    assert B.OVERFLOW_ITEMS > 256 * 1024 and min(B.OVERFLOW_TOPKS) < c["TK_MAXK"] < max(B.OVERFLOW_TOPKS)
