"""CPU: the restatement of pio_serve_zscore_merge (serve_merge_ref.py) -- its pairwise sum is np.add.reduce bit for bit,
and its merge is the similarproduct template's Serving.serve query by query (item strings, float bits and order) on
random lists and at the rule's edges: num == 1, empty and one-entry lists, all-equal scores, items shared by two or three
algorithms, and exact ties in the combined score."""
import numpy as np
import pytest

import serve_merge_ref as ref


def bits(x):
    return np.float64(x).tobytes()


@pytest.mark.parametrize("kind", ["normal", "scaled", "zeros", "mixed_zeros", "ints"])
def test_pairwise_sum_is_numpy_add_reduce(kind):
    rng = np.random.default_rng(["normal", "scaled", "zeros", "mixed_zeros", "ints"].index(kind))
    for n in list(range(0, 300)) + list(range(1000, 1101)) + [511, 512, 513, 2047, 2048, 2049, 4099]:
        if kind == "normal":
            a = rng.standard_normal(n)
        elif kind == "scaled":
            a = rng.standard_normal(n) * 10.0 ** rng.integers(-200, 200, n)
        elif kind == "zeros":
            a = np.full(n, -0.0)
        elif kind == "mixed_zeros":
            a = np.where(rng.random(n) < 0.5, -0.0, 0.0)
            a[rng.random(n) < 0.1] = rng.standard_normal() * 1e-300
        else:
            a = rng.integers(-2 ** 53, 2 ** 53, n).astype(np.float64)
        assert bits(ref.add_reduce(a)) == bits(np.add.reduce(a)), n


def test_pairwise_is_not_first_plus_rest():
    """The documented trap: np.add.reduce is 0.0 + pairwise(a), not a[0] + pairwise(a[1:])."""
    rng = np.random.default_rng(5)
    differ = 0
    for n in range(9, 400):
        a = rng.standard_normal(n) * 10.0 ** rng.integers(-8, 8, n)
        v = a.tolist()
        assert bits(ref.add_reduce(a)) == bits(np.add.reduce(a))
        differ += bits(v[0] + ref.pairwise(v, 1, n - 1)) != bits(np.add.reduce(a))
    assert differ > 0


def serve(num, lists):
    from pio_b200.templates import similarproduct as sp
    prs = [sp.PredictedResult([sp.ItemScore(it, float(s)) for it, s in lst]) for lst in lists]
    return [(x.item, x.score) for x in sp.Serving().serve(sp.Query(items=["x"], num=num), prs).itemScores]


def same(got, want):
    assert [it for it, _ in got] == [it for it, _ in want]
    assert [bits(v) for _, v in got] == [bits(v) for _, v in want]


def random_lists(rng, n_algos, pool, widths):
    out = []
    for a in range(n_algos):
        n = int(rng.integers(0, widths + 1))
        items = rng.choice(pool, min(n, len(pool)), replace=False).tolist()
        scale = float(10.0 ** rng.integers(-3, 6))
        out.append([(it, float(rng.standard_normal() * scale) if a < 2 else float(rng.integers(1, 50)))
                    for it in items])
    return out


def test_merge_equals_serve_on_random_lists():
    rng = np.random.default_rng(1)
    pool = [f"i{k}" for k in range(40)]
    for t in range(1500):
        lists = random_lists(rng, int(rng.integers(1, 4)), pool, int(rng.choice([1, 3, 10, 25, 40])))
        num = int(rng.choice([1, 2, 3, 10, 100]))
        same(ref.merge_one(lists, num), serve(num, lists))


@pytest.mark.parametrize("case", ["num1", "empty", "one_entry", "all_equal", "shared", "ties", "long", "neg_zero"])
def test_merge_equals_serve_at_the_edges(case):
    rng = np.random.default_rng(7)
    L = {
        "num1": ([[("a", 3.0), ("b", 1.0)], [("b", 2.5), ("c", 0.5)], [("a", 0.25)]], 1),
        "empty": ([[], [("a", 1.0)], []], 5),
        "one_entry": ([[("a", 7.0)], [("b", -3.0)], [("a", 1.0)]], 4),
        "all_equal": ([[("a", 2.0), ("b", 2.0), ("c", 2.0)], [("c", 5.0), ("d", 1.0)]], 10),
        "shared": ([[("a", 1.0), ("b", 2.0), ("c", 3.0)], [("c", 0.5), ("a", 4.0)], [("b", 9.0), ("a", 9.0), ("c", 1.0)]], 3),
        # a and b tie on each list: equal z-scores, ordered by first appearance (b before a)
        "ties": ([[("b", 1.0), ("a", 1.0), ("c", 0.0)], [("d", 2.0), ("e", 2.0)], [("e", 3.0), ("d", 3.0)]], 10),
        "long": ([[(f"i{k}", float(rng.standard_normal())) for k in range(300)],
                  [(f"i{k}", float(rng.integers(1, 9))) for k in range(0, 600, 3)]], 50),
        "neg_zero": ([[("a", -0.0), ("b", 0.0)], [("b", -0.0)]], 1),
    }[case]
    lists, num = L
    got, want = ref.merge_one(lists, num), serve(num, lists)
    same(got, want)
    if case == "ties":
        assert [it for it, _ in got][:2] == ["b", "a"] and got[0][1] == got[1][1]


def test_array_merge_and_parts():
    """merge over id arrays equals merge_one on the same lists; parts close before the query that would overflow."""
    rng = np.random.default_rng(3)
    Q, widths = 50, [6, 9, 4]
    items = [np.full((Q, w), -1, np.int32) for w in widths]
    scores = [np.zeros((Q, w)) for w in widths]
    counts = [rng.integers(0, w + 1, Q).astype(np.int32) for w in widths]
    for a, w in enumerate(widths):
        for j in range(Q):
            c = counts[a][j]
            items[a][j, :c] = rng.choice(15, c, replace=False)
            scores[a][j, :c] = rng.standard_normal(c).round(1)   # rounded: ties
    num = rng.choice([1, 2, 5, 40], Q)
    oi, os_, oc = ref.merge(items, scores, counts, num, 7)
    for j in range(Q):
        want = ref.merge_one([list(zip(items[a][j, :counts[a][j]].tolist(), scores[a][j, :counts[a][j]].tolist()))
                              for a in range(3)], int(num[j]))[:7]
        assert oc[j] == len(want) and oi[j, :oc[j]].tolist() == [i for i, _ in want]
        assert [bits(v) for v in os_[j, :oc[j]]] == [bits(v) for _, v in want]
        assert (oi[j, oc[j]:] == -1).all() and (os_[j, oc[j]:] == 0).all()
    ent = sum(c.astype(np.int64) for c in counts)
    first = ref.parts(counts, 20)
    for p, j0 in enumerate(first):
        j1 = first[p + 1] if p + 1 < len(first) else Q
        assert j1 - j0 == 1 or ent[j0:j1].sum() <= 20
        assert j1 == Q or ent[j0:j1 + 1].sum() > 20
    assert ref.parts(counts, 10 ** 12) == [0]
