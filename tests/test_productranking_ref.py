"""CPU: the vectorised product ranking restatement (tests/productranking_ref.rank_lists, what the GPU tests compare
pio_als_rank_lists with) equals the line-by-line transcription of the Scala predict, and the template's host logic turns
queries into index arrays and results into PredictedResult objects as predict would."""
import numpy as np
import pytest

from tests import productranking_ref as ref

ORDER = [float("nan"), float("inf"), 1.0, 0.0, -0.0, -1.0, float("-inf")]


def _bits(a):
    return np.asarray(a, np.float64).view(np.uint64)


def test_order_key_is_double_compare_descending():
    rng = np.random.default_rng(0)
    for _ in range(20):
        perm = rng.permutation(len(ORDER))
        vals = np.array(ORDER)[perm]
        got = vals[np.argsort(ref.order_key(vals), kind="stable")]
        assert np.array_equal(_bits(got[1:]), _bits(ORDER[1:])) and np.isnan(got[0])
    # every NaN is the same key, and Double.compare agrees with the key on every pair
    nans = np.array([0x7FF8000000000000, 0xFFF8000000000000, 0x7FF0000000000001], np.uint64).view(np.float64)
    assert len(set(ref.order_key(nans).tolist())) == 1
    for a in ORDER:
        for b in ORDER:
            ka, kb = ref.order_key([a])[0], ref.order_key([b])[0]
            assert ref.double_compare(a, b) == int(kb > ka) - int(kb < ka), (a, b)


def _literal_batch(uf, uh, itf, ih, users, ptr, items):
    pos, sc, ranked = [], [], []
    for q, u in enumerate(users):
        p, s, orig = ref.predict_literal(uf, uh, itf, ih, int(u), items[ptr[q]:ptr[q + 1]])
        pos += p
        sc += s
        ranked.append(not orig)
    return np.array(pos, np.int32), np.array(sc, np.float64), np.array(ranked, bool)


def _check(uf, uh, itf, ih, lists):
    users = np.array([u for u, _ in lists], np.int64)
    ptr = np.zeros(len(lists) + 1, np.int64)
    ptr[1:] = np.cumsum([len(x) for _, x in lists])
    items = np.array([i for _, x in lists for i in x], np.int64)
    want = _literal_batch(uf, uh, itf, ih, users, ptr, items)
    got = ref.rank_lists(uf, uh, itf, ih, users, ptr, items)
    assert np.array_equal(got[0], want[0])
    assert np.array_equal(_bits(got[1]), _bits(want[1]))
    assert np.array_equal(got[2], want[2])
    return got


def test_hand_made_cases():
    # rank 2; item 3 has no factor, item 4 is a zero row (ties with unknown entries), user 2 has no factor
    uf = np.array([[1, 0], [0, 1], [5, 5]], np.float32)
    uh = np.array([1, 1, 0], np.uint8)
    itf = np.array([[2, 1], [-1, 3], [2, 1], [9, 9], [0, 0]], np.float32)
    ih = np.array([1, 1, 1, 0, 1], np.uint8)
    pos, sc, ranked = _check(uf, uh, itf, ih, [
        (0, [0, 1, 2, 0, 7, -1, 3, 4]),   # duplicates, unknown ids, no factor, zero row
        (1, [1, 0]),
        (2, [0, 1]),                       # user without a factor
        (9, [0]),                          # unknown user
        (0, [3, 7, -5]),                   # no entry has a score
        (0, []),                           # empty list
        (-1, []),
    ])
    assert pos[:8].tolist() == [0, 2, 3, 4, 5, 6, 7, 1]   # 2, 2, 2 in query order; then the four 0.0; then -1
    assert sc[:8].tolist() == [2, 2, 2, 0, 0, 0, 0, -1]
    assert ranked.tolist() == [True, True, False, False, False, False, False]
    assert pos[8:10].tolist() == [0, 1] and pos[10:].tolist() == [0, 1, 0, 0, 1, 2]


def test_nan_and_infinities():
    inf = np.float32(np.inf)
    uf = np.array([[1, 1], [inf, 0], [-inf, 1]], np.float32)
    itf = np.array([[1, 0], [0, 1], [-1, 0], [inf, 0], [inf, -inf], [0, 0], [-2, 1]], np.float32)
    uh, ih = np.ones(3, np.uint8), np.ones(7, np.uint8)
    _, sc, _ = _check(uf, uh, itf, ih, [(u, list(range(7)) + [9, 4, 0]) for u in range(3)])
    assert np.isnan(sc).any() and np.isinf(sc).any()
    assert _bits(sc[np.isnan(sc)]).tolist() == [0x7FF8000000000000] * int(np.isnan(sc).sum())


@pytest.mark.parametrize("seed", range(6))
def test_seeded_batches(seed):
    rng = np.random.default_rng(seed)
    k = int(rng.integers(1, 9))
    nu, ni = 12, 30
    # few distinct values so that ties are common
    uf = rng.integers(-2, 3, (nu, k)).astype(np.float32) * np.float32(0.5)
    itf = rng.integers(-2, 3, (ni, k)).astype(np.float32)
    uh = (rng.random(nu) < 0.8).astype(np.uint8)
    ih = (rng.random(ni) < 0.8).astype(np.uint8)
    lists = [(int(rng.integers(-2, nu + 2)), rng.integers(-3, ni + 3, int(rng.integers(0, 40))).tolist())
             for _ in range(50)]
    _check(uf, uh, itf, ih, lists)


# ---- the template's host logic ----------------------------------------------------------------------------------------
class _Factors:
    """A MatrixFactorizationModel stand-in whose rankLists is the restatement."""

    def __init__(self, uf, uh, itf, ih):
        self.rank, self.args = uf.shape[1], (uf, uh, itf, ih)

    def rankLists(self, users, list_ptr, items):
        assert users.dtype == np.int32 and list_ptr.dtype == np.int64 and items.dtype == np.int32
        return ref.rank_lists(*self.args, users, list_ptr, items)


def test_template_predict_many_builds_results_as_predict():
    from pio_b200.storage import BiMap
    from pio_b200.templates import productranking as pr
    rng = np.random.default_rng(7)
    uf = rng.standard_normal((4, 3)).astype(np.float32)
    itf = rng.standard_normal((6, 3)).astype(np.float32)
    uh = np.array([1, 1, 0, 1], np.uint8)
    ih = np.array([1, 0, 1, 1, 1, 1], np.uint8)
    model = pr.ALSModel(_Factors(uf, uh, itf, ih), BiMap.stringInt([f"u{k}" for k in range(4)]),
                        BiMap.stringInt([f"i{k}" for k in range(6)]))
    algo = pr.ALSAlgorithm(pr.ALSAlgorithmParams(rank=3, numIterations=1))
    qs = [pr.Query("u0", ["i1", "i3", "i10", "i2", "i5", "i31", "i3"]), pr.Query("u2", ["i0", "i2"]),
          pr.Query("nobody", ["i0"]), pr.Query("u1", []), pr.Query("u3", ["i1", "x"]), pr.Query("u3", ["i4", "i0"])]
    got = algo.predictMany(model, qs)
    assert got == [algo.predict(model, q) for q in qs]
    for q, r in zip(qs, got):
        u = model.userStringIntMap.getOrElse(q.user, -1)
        items = [model.itemStringIntMap.getOrElse(x, -1) for x in q.items]
        pos, sc, orig = ref.predict_literal(uf, uh, itf, ih, u, items)
        assert r.isOriginal == orig
        assert [(s.item, s.score) for s in r.itemScores] == [(q.items[p], v) for p, v in zip(pos, sc)]
    assert [r.isOriginal for r in got] == [False, True, True, True, True, False]
    assert [s.item for s in got[0].itemScores].count("i3") == 2


def test_template_requires_ratings():
    from pio_b200.templates import productranking as pr
    td = pr.TrainingData(users={"u": pr.User()}, items={"i": pr.Item()}, viewEvents=[pr.ViewEvent("v", "i", 0)])
    with pytest.raises(ValueError, match="mllibRatings cannot be empty"):
        pr.ALSAlgorithm(pr.ALSAlgorithmParams(rank=2, numIterations=1)).train(None, td)
