"""GPU tests (-m gpu) of item co-occurrence (pio_cooc_train, csrc/cooc.cuh) against cooc_ref.py, the vectorised
restatement of CooccurrenceAlgorithm.trainCooccurrence.  All work is integer: every output is compared exactly.

The kernels pack keys by bit width: (user, item) in bits_u + bits_i bits, pairs in 2 bits_i, ranking keys in
2 bits_i + bits_c with bits_c = min(32, 64 - 2 bits_i) (32 up to 65 536 items, 30 at 65 537, 24 at 2^20, the largest
item count accepted).  The cases step over those widths, the power-of-two user counts, one user whose list spans many
sort tiles, many users with one list (large counts), users with one item and repeated views, and topn below and above
every item's partner count.  A user list long enough for more than 2^31 - 1 pairs is rejected; at about 92 700 items the
pair total no longer fits in 32 bits, which the rejection must not depend on.
"""
import numpy as np
import pytest

import cooc_ref

pytestmark = pytest.mark.gpu

MAX_ITEMS = 1 << 20


def workload(rng, nu, ni, n):
    """Events over every user and item index range: a popular head of items, the largest user and item indices
    viewed together, one user viewing one item many times, and users with a single item."""
    u = rng.integers(0, nu, n).astype(np.int32)
    i = np.minimum((rng.random(n) ** 3 * ni).astype(np.int32), ni - 1)
    u[:30], i[:30] = nu - 1, ni - 1
    u[30:60], i[30:60] = 0, 0
    u[60:62], i[60:62] = nu - 1, (0, ni // 2)
    return u, i


def check(native, u, i, nu, ni, topn):
    got = native.cooc_train(u, i, nu, ni, topn)
    want = cooc_ref.cooc_train(u, i, ni, topn)
    for name, g, w in zip(("items", "counts", "n"), got, want):
        assert np.array_equal(g, w), (name, int((g != w).sum()))
    return got


@pytest.mark.parametrize("n_items", [1, 2, 3, 512, 513, 65536, 65537, MAX_ITEMS])
@pytest.mark.parametrize("topn", [1, 7])
def test_item_counts_across_key_widths(native, n_items, topn):
    rng = np.random.default_rng(n_items + topn)
    u, i = workload(rng, 3000, n_items, 60000)
    _, _, gn = check(native, u, i, 3000, n_items, topn)
    if n_items == 1:
        assert (gn == 0).all()
    else:
        assert gn[n_items - 1] >= 1


def test_item_count_over_the_key_limit_is_rejected(native):
    u = np.zeros(4, np.int32)
    i = np.arange(4, dtype=np.int32)
    with pytest.raises(native.NativeError) as ei:
        native.cooc_train(u, i, 1, MAX_ITEMS + 1, 5)
    assert ei.value.code == native.ERR_ARG


@pytest.mark.parametrize("n_users", [1, 2, 255, 256, 257, 65536, 65537])
def test_user_counts_at_power_of_two_edges(native, n_users):
    rng = np.random.default_rng(n_users)
    u, i = workload(rng, n_users, 300, 40000)
    check(native, u, i, n_users, 300, 7)


@pytest.mark.parametrize("topn", [1, 7, 6000])
def test_one_user_with_thousands_of_items(native, topn):
    """One user's 5 000 distinct items span many sort and scan tiles (12.5 M pairs); short lists around it."""
    rng = np.random.default_rng(5)
    ni, nu = 8000, 2000
    big = rng.choice(ni, 5000, replace=False).astype(np.int32)
    u, i = workload(rng, nu, ni, 20000)
    u = np.r_[u, np.full(big.shape[0], 777, np.int32)]
    i = np.r_[i, big]
    perm = rng.permutation(u.shape[0])
    check(native, u[perm], i[perm], nu, ni, topn)


@pytest.mark.parametrize("topn", [1, 7, 250])
def test_many_users_with_one_list(native, topn):
    """500 users view the same 200 items (counts of 500 for every pair of them), some users add a few more."""
    rng = np.random.default_rng(6)
    ni, nu = 1000, 600
    lst = rng.choice(ni, 200, replace=False).astype(np.int32)
    u = np.repeat(np.arange(500, dtype=np.int32), lst.shape[0])
    i = np.tile(lst, 500)
    extra_u = rng.integers(400, nu, 3000).astype(np.int32)
    extra_i = rng.integers(0, ni, 3000).astype(np.int32)
    _, gc, _ = check(native, np.r_[u, extra_u], np.r_[i, extra_i], nu, ni, topn)
    assert gc.max() >= 500


def test_single_item_users_and_repeated_views(native):
    """Most users view one item, many times; the few pairs come from a handful of users."""
    rng = np.random.default_rng(7)
    nu, ni = 5000, 400
    u = np.repeat(np.arange(nu, dtype=np.int32), 4)
    i = np.repeat(rng.integers(0, ni, nu).astype(np.int32), 4)
    u = np.r_[u, [3, 3, 3, 9, 9]].astype(np.int32)
    i = np.r_[i, [1, 2, 2, 1, 2]].astype(np.int32)
    for topn in (1, 7, 500):
        check(native, u, i, nu, ni, topn)
    gi, gc, gn = native.cooc_train(u[:4 * nu], i[:4 * nu], nu, ni, 3)     # no pairs at all
    assert (gn == 0).all() and (gi == -1).all() and (gc == 0).all()


@pytest.mark.parametrize("k", [65537, 92700])
def test_pair_total_over_int32_is_rejected(native, k):
    """One user with k distinct items has k (k - 1) / 2 pairs: 2.15e9 (below 2^32) and 4.297e9 (above 2^32, where a
    32-bit total wraps to a small number).  Both are over 2^31 - 1 and must be rejected, not indexed."""
    total = cooc_ref.pair_total(np.zeros(k, np.int32), np.arange(k, dtype=np.int32), k)
    assert total == k * (k - 1) // 2 >= 2 ** 31
    with pytest.raises(native.NativeError) as ei:
        native.cooc_train(np.zeros(k, np.int32), np.arange(k, dtype=np.int32), 1, k, 5)
    assert ei.value.code == native.ERR_ARG and "co-occurrence pairs" in str(ei.value)
    rng = np.random.default_rng(k)
    u, i = workload(rng, 50, 40, 500)
    check(native, u, i, 50, 40, 5)                                        # the library still trains afterwards
