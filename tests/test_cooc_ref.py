"""CPU checks of cooc_ref.py, the vectorised co-occurrence restatement the GPU tests compare against: equal to the
set-based oracle.cooc_train on small workloads with repeated views, one-item users, ties and items nobody co-viewed."""
import numpy as np
import pytest

import cooc_ref


def workload(rng, nu, ni, n):
    u = rng.integers(0, nu, n).astype(np.int32)
    i = np.minimum((rng.random(n) ** 2 * ni).astype(np.int32), max(ni - 2, 0))
    u[:20] = nu - 1
    i[:20] = 0                             # one user viewing one item 20 times
    return u, i


@pytest.mark.parametrize("nu,ni,n", [(1, 1, 5), (3, 2, 10), (40, 7, 300), (200, 60, 3000), (800, 300, 20000)])
@pytest.mark.parametrize("topn", [1, 7, 400])
def test_restatement_matches_oracle(oracle, nu, ni, n, topn):
    rng = np.random.default_rng(nu + ni + topn)
    u, i = workload(rng, nu, ni, n)
    got = cooc_ref.cooc_train(u, i, ni, topn)
    want = oracle.cooc_train(u, i, ni, topn)
    for g, w in zip(got, want):
        assert g.dtype == w.dtype and np.array_equal(g, w)


def test_pair_total():
    u = np.array([0, 0, 0, 0, 1, 1, 2, 3, 3, 3], np.int32)
    i = np.array([5, 1, 5, 2, 1, 1, 4, 0, 1, 2], np.int32)
    assert cooc_ref.pair_total(u, i, 6) == 3 + 0 + 0 + 3
    k = 92_700
    assert cooc_ref.pair_total(np.zeros(k, np.int32), np.arange(k, dtype=np.int32), k) == k * (k - 1) // 2 > 2 ** 32
