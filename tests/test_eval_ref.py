"""tests/eval_ref.py (the k-fold evaluation on global indices that pio_eval_folds computes) against the recommendation
template's own definitions, on seeded random cases: DataSource.readEval's split and query order, BiMap.stringInt of each
fold's training strings, PrecisionAtK / PositiveCount.calculate_one, and the means the columnar metrics take from the
per-query counts."""
import numpy as np
import pytest

import eval_ref
from pio_b200 import native
from pio_b200 import storage as s
from pio_b200.evaluation import EvalColumns
from pio_b200.templates import recommendation as rec

# (seed, ratings, users, items, kFold): small id ranges give repeated (user, item) pairs in a test fold, users and items
# seen in one fold only (unknown to its training set) and ids whose first two occurrences share a fold
CASES = [(1, 200, 30, 20, 2), (2, 300, 60, 40, 5), (3, 120, 90, 15, 5), (4, 400, 25, 80, 2), (5, 60, 40, 40, 5)]
VALUES = (1.0, 2.0, 3.0, 4.0, 4.5, 5.0)
THRESHOLDS = (1.0, 2.0, 4.0, 4.5, 6.0)


def _case(seed, n, n_users, n_items):
    rng = np.random.default_rng(seed)
    users = [f"u{x}" for x in rng.integers(0, n_users, n)]
    items = [f"i{x}" for x in rng.integers(0, n_items, n)]
    return users, items, rng.choice(VALUES, n)


def _global(strings):
    """Global indices in first-occurrence order (what ids_encode returns) and the string of each index."""
    m = s.BiMap.stringInt(strings)
    return np.array([m(x) for x in strings], np.int64), list(m.toMap())


def _read_eval(monkeypatch, users, items, ratings, k_fold, num):
    cols = rec.RatingColumns(native._str_column([x.encode() for x in users]), native._str_column([x.encode() for x in items]),
                             np.asarray(ratings, np.float64), np.ones(len(users), bool))
    ds = rec.DataSource(rec.DataSourceParams("App", rec.DataSourceEvalParams(kFold=k_fold, queryNum=num)))
    monkeypatch.setattr(ds, "getRatingColumns", lambda sc: cols)
    return ds.readEval(None)


@pytest.mark.parametrize("seed,n,n_users,n_items,k_fold", CASES)
def test_fold_maps_coo_and_queries_match_the_template(monkeypatch, seed, n, n_users, n_items, k_fold):
    users, items, ratings = _case(seed, n, n_users, n_items)
    gu, ustr = _global(users)
    gi, istr = _global(items)
    ref = eval_ref.split(gu, gi, ratings, k_fold)
    for f, (td, _, qas) in enumerate(_read_eval(monkeypatch, users, items, ratings, k_fold, 10)):
        um = s.BiMap.stringInt(r.user for r in td.ratings)
        im = s.BiMap.stringInt(r.item for r in td.ratings)
        assert list(um.toMap()) == [ustr[g] for g in ref[f]["user"]]
        assert list(im.toMap()) == [istr[g] for g in ref[f]["item"]]
        assert np.array_equal(ref[f]["train_user"], [um(r.user) for r in td.ratings])
        assert np.array_equal(ref[f]["train_item"], [im(r.item) for r in td.ratings])
        assert np.array_equal(ref[f]["train_rating"], np.array([r.rating for r in td.ratings], np.float32))
        assert [q.user for q, _ in qas] == [ustr[g] for g in ref[f]["query_user"]]
        assert np.array_equal(ref[f]["query_train_user"], [um.getOrElse(q.user, -1) for q, _ in qas])


def test_cases_cover_the_edge_cases():
    seen = set()
    for seed, n, n_users, n_items, k_fold in CASES:
        users, items, ratings = _case(seed, n, n_users, n_items)
        gu, _ = _global(users)
        gi, _ = _global(items)
        for f, fold in enumerate(eval_ref.split(gu, gi, ratings, k_fold)):
            if (fold["query_train_user"] < 0).any():
                seen.add("test user unknown to training")
            if not np.isin(fold["test_item"], fold["item"]).all():
                seen.add("test item unknown to training")
            pairs = fold["test_q"] * (int(gi.max()) + 1) + fold["test_item"]
            if np.unique(pairs).shape[0] < pairs.shape[0]:
                seen.add("repeated (user, item) pair in a test fold")
            for thr in (2.0, 4.0):
                if (fold["test_rating"] == thr).any():
                    seen.add(f"rating at threshold {thr}")
                pos = np.zeros(fold["query_user"].shape[0], bool)
                pos[fold["test_q"][fold["test_rating"] >= thr]] = True
                if not pos.all():
                    seen.add(f"query without positives at {thr}")
        for g in range(int(gu.max()) + 1):
            occ = np.flatnonzero(gu == g)
            if occ.shape[0] > 1 and occ[0] % k_fold == occ[1] % k_fold:
                seen.add(f"id whose first two occurrences share a fold, kFold {k_fold}")
    assert seen == {"test user unknown to training", "test item unknown to training",
                    "repeated (user, item) pair in a test fold", "rating at threshold 2.0", "rating at threshold 4.0",
                    "query without positives at 2.0", "query without positives at 4.0",
                    "id whose first two occurrences share a fold, kFold 2",
                    "id whose first two occurrences share a fold, kFold 5"}


def _predictions(rng, fold, num):
    """A top-N result of the fold: per query a random run of distinct training items, count 0 for unknown users."""
    nq, ni = fold["query_user"].shape[0], fold["item"].shape[0]
    items = np.full((nq, num), -1, np.int32)
    count = np.zeros(nq, np.int32)
    for q in range(nq):
        if fold["query_train_user"][q] >= 0:
            c = int(rng.integers(0, min(num, ni) + 1))
            items[q, :c] = rng.permutation(ni)[:c]
            count[q] = c
    return items, count


class _RefResult:
    """A fold result whose rank counts come from eval_ref (what native.EvalResult returns from the device)."""

    def __init__(self, fold, items, count):
        self.fold, self.items, self.count = fold, items, count

    def rank_counts(self, k, threshold):
        return eval_ref.rank_counts(self.fold, self.items, self.count, k, threshold)


@pytest.mark.parametrize("seed,n,n_users,n_items,k_fold", CASES)
@pytest.mark.parametrize("num", [1, 4, 10])
def test_rank_counts_match_the_metrics(monkeypatch, seed, n, n_users, n_items, k_fold, num):
    users, items, ratings = _case(seed, n, n_users, n_items)
    gu, _ = _global(users)
    gi, istr = _global(items)
    ref = eval_ref.split(gu, gi, ratings, k_fold)
    rng = np.random.default_rng(seed + 100)
    obj, cols = [], []
    for f, (_, _, qas) in enumerate(_read_eval(monkeypatch, users, items, ratings, k_fold, num)):
        it, cnt = _predictions(rng, ref[f], num)
        qpa = [(q, rec.PredictedResult([rec.ItemScore(istr[ref[f]["item"][it[j, t]]], 0.0) for t in range(cnt[j])]), a)
               for j, (q, a) in enumerate(qas)]
        obj.append((None, qpa))
        cols.append((None, None, _RefResult(ref[f], it, cnt)))
        for k in sorted({1, max(num - 1, 1), num, num + 3}):
            for thr in THRESHOLDS:
                hits, npos, nraw = eval_ref.rank_counts(ref[f], it, cnt, k, thr)
                pk, pc = rec.PrecisionAtK(k, thr), rec.PositiveCount(thr)
                for j, (q, p, a) in enumerate(qpa):
                    want = pk.calculate_one(q, p, a)
                    assert (want is None) == (npos[j] == 0)
                    if want is not None:
                        assert hits[j] / min(k, npos[j]) == want
                    assert float(nraw[j]) == pc.calculate_one(q, p, a)
    for k in (1, num, num + 3):
        for thr in THRESHOLDS:
            for m in (rec.PrecisionAtK(k, thr), rec.PositiveCount(thr)):
                want = m.calculate(None, obj)
                got = m.calculate_columns(None, EvalColumns(cols))
                assert got == want or (np.isnan(got) and np.isnan(want))
