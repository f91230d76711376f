"""CPU: the NumPy scoring restatement (tests/scoring_ref.py) equals the C oracle bit for bit.

Random cases with masks, weights of 0, -1 and 0.5 (signed-zero and negative scores), exact ties from duplicated rows and a
zero user, keep-query, duplicate / out-of-range / factor-less query ids, and topk above the number of candidates.
"""
import numpy as np
import pytest

import scoring_ref


def _model(seed, n_users, n_items, rank):
    rng = np.random.default_rng(seed)
    uf = rng.standard_normal((n_users, rank)).astype(np.float32)
    itf = rng.standard_normal((n_items, rank)).astype(np.float32)
    itf[5:9] = itf[20]                       # a block of bit-identical item rows: exact ties
    itf[30:33] = 2 * itf[40]                 # parallel rows: equal cosines
    uf[0] = 0.0                              # every score 0: pure id order
    uh = (rng.random(n_users) > 0.1).astype(np.uint8)
    ih = (rng.random(n_items) > 0.15).astype(np.uint8)
    uh[0] = 1
    uf[uh == 0] = 0.0
    itf[ih == 0] = 0.0
    mask = (rng.random(n_items) < 0.1).astype(np.uint8)
    weight = rng.choice(np.array([0.0, -1.0, 0.5, 1.0, 2.0]), n_items)
    return rng, uf, itf, uh, ih, mask, weight


def _eq(a, b):
    for x, y in zip(a, b):
        x, y = np.asarray(x), np.asarray(y)
        assert x.shape == y.shape and np.array_equal(x.view(np.uint8) if x.dtype == np.float32 else x,
                                                     y.view(np.uint8) if y.dtype == np.float32 else y), (x, y)


@pytest.mark.parametrize("seed,rank,n_items", [(0, 1, 50), (1, 7, 97), (2, 16, 300), (3, 33, 128), (4, 128, 64)])
def test_recommend_matches_oracle(oracle, seed, rank, n_items):
    rng, uf, itf, uh, ih, mask, weight = _model(seed, 20, n_items, rank)
    users = np.array([0, 1, 2, 3, 19, 5, 5], np.int32)
    for topk in (1, 5, n_items, n_items + 7):
        for mk, wt in ((None, None), (mask, None), (None, weight), (mask, weight)):
            got = scoring_ref.recommend(uf, uh, itf, ih, users, topk, mk, wt)
            want = oracle.recommend(uf, uh, itf, ih, users, topk, mk, wt)
            _eq(got, want)


def test_recommend_signed_zero_ties(oracle):
    # weight 0 and -1 on a zero user: +0.0 and -0.0 scores tie and rank by id
    _, uf, itf, uh, ih, _, _ = _model(7, 4, 48, 8)
    weight = np.where(np.arange(48) % 2 == 0, 0.0, -1.0)
    got = scoring_ref.recommend(uf, uh, itf, ih, np.array([0], np.int32), 48, None, weight)
    want = oracle.recommend(uf, uh, itf, ih, np.array([0], np.int32), 48, None, weight)
    _eq(got, want)
    assert np.array_equal(got[0][0, :got[2][0]], np.flatnonzero(ih))


@pytest.mark.parametrize("seed,rank,n_items", [(10, 1, 60), (11, 8, 200), (12, 17, 150), (13, 64, 90), (14, 128, 48)])
def test_similar_matches_oracle(oracle, seed, rank, n_items):
    rng, _, itf, _, ih, mask, weight = _model(seed, 2, n_items, rank)
    off = int(np.flatnonzero(ih == 0)[0])
    queries = [[20], [20, 20], [5, 40, n_items + 3, -1], [off], [off, 30, off], [],
               list(rng.integers(0, n_items, 12)), [n_items, -5]]
    for q in queries:
        for topk in (1, 4, n_items + 3):
            for keep in (False, True):
                for mk, wt in ((None, None), (mask, weight)):
                    got = scoring_ref.similar(itf, ih, np.asarray(q, np.int32), topk, mk, wt, keep)
                    want = oracle.similar(itf, ih, np.asarray(q, np.int32), topk, mk, wt, keep)
                    _eq(got[:2], want[:2])
                    assert got[2] == want[2]
