"""CPU tests of the text classification template's device evaluation rules (tests/text_eval_ref.py): the split, the
test renumbering, the fold lists cut from one featurization against the host-cut subsets, the vectorised categoryMap,
serveColumns against Serving.serve, and which evaluations take the columnar path."""
import math
from types import SimpleNamespace

import numpy as np
import pytest

from pio_b200 import evaluation as ev
from pio_b200 import native
from pio_b200.controller import EngineParams
from pio_b200.templates import textclassification as tc
from tests import text_eval_ref as er
from tests import textclassification_ref as ref

WORDS = [b"a", b"bb", b"ccc", b"dddd", b"spam", b"free", b"the", b"\xc3\xa9", b"x y"]


def _texts(n, seed):
    rng = np.random.default_rng(seed)
    return [b" ".join(WORDS[int(j)] for j in rng.integers(0, len(WORDS), int(rng.integers(0, 9)))) for _ in range(n)]


class _Folds:
    """A stand-in for native.TextFolds on the CPU: the split's sizes only."""

    def __init__(self, n, k):
        self.n, self.k_fold = n, k

    def sizes(self, f):
        m = (self.n + self.k_fold - 1 - f) // self.k_fold
        return self.n - m, m


def _data(n, seed, n_labels=2):
    rng = np.random.default_rng(seed)
    cats = [["spam", "ham", "eggs"][int(c)] for c in rng.integers(0, n_labels, n)]
    cats = [c if rng.random() < 0.7 else c.upper() for c in cats]      # several categories per label
    labels = np.array([1.0 if c == "spam" else 0.0 for c in cats])
    tb, to = native.text_tokens([t.decode() for t in _texts(n, seed)])
    return tc.TrainingData((tb, to), labels, cats, ["the"])


@pytest.mark.parametrize("n", [1, 2, 3, 7, 20])
@pytest.mark.parametrize("k", [1, 2, 3, 5, 8])
def test_split_and_sizes(n, k):
    seen = np.zeros(n, np.int64)
    for f in range(k):
        train, test = er.fold_docs(n, k, f)
        assert np.array_equal(np.sort(np.r_[train, test]), np.arange(n))
        assert (test % k == f).all() and (train % k != f).all()
        assert _Folds(n, k).sizes(f) == (train.shape[0], test.shape[0])
        fold = tc.TextFold(_Folds(n, k), f, _data(n, n + k))
        assert np.array_equal(fold.rows(False), train) and np.array_equal(fold.rows(True), test)
        t = er.held_out_position(test, k, f)
        assert np.array_equal(t, np.arange(test.shape[0]))     # t = (d - f) / k numbers the test documents in order
        seen[test] += 1
    assert (seen == 1).all()


@pytest.mark.parametrize("k", [1, 2, 3, 5])
@pytest.mark.parametrize("n_gram,D", [(1, 97), (2, 1 << 18), (3, 1)])
def test_fold_lists_equal_the_subsets(k, n_gram, D):
    texts = _texts(40, k * 10 + n_gram)
    labels = np.where(np.arange(40) % 3 == 0, 1.0, 0.0)
    stop = [b"the"]
    ptr, idx, tf = ref.features(texts, n_gram, D, stop)
    for f in range(k):
        train, test = er.fold_docs(40, k, f)
        if not train.shape[0]:
            continue
        j, c, cls, classes = er.training_list(ptr, idx, tf, labels, k, f)
        sp, sj, sv = ref.features([texts[i] for i in train], n_gram, D, stop)
        assert np.array_equal(np.bincount(j, minlength=D), np.bincount(sj, minlength=D))   # the fold's df
        scls = np.repeat(np.searchsorted(classes, labels[train]), np.diff(sp))
        assert sorted(zip(cls.tolist(), j.tolist(), c.tolist())) == sorted(zip(scls.tolist(), sj.tolist(), sv.tolist()))
        _, _, idf, pi, theta, _ = er.fold_model(texts, labels, ["c"] * 40, k, f, n_gram, D, 1.0, stop)
        tp, tj, tv, t = er.held_out_list(ptr, idx, tf * idf[idx], k, f)
        assert (np.diff(t) >= 0).all()
        want = ref.features([texts[i] for i in test], n_gram, D, stop, idf)
        assert np.array_equal(tp, want[0]) and np.array_equal(tj, want[1]) and np.array_equal(tv, want[2])
        raw = ref.scores(tp, tj, tv, pi, theta)
        assert np.array_equal(raw, er.fold_predictions(texts, k, f, n_gram, D, stop, idf, pi, theta)[0], equal_nan=True)


@pytest.mark.parametrize("n,k,n_labels", [(30, 5, 2), (9, 4, 3), (5, 5, 2), (1, 2, 2), (12, 1, 3)])
def test_vectorised_category_map_equals_the_subsets(n, k, n_labels):
    td = _data(n, n * 31 + k, n_labels)
    for f in range(k):
        fold = tc.TextFold(_Folds(n, k), f, td)
        classes, cls_doc, cm = fold.train_classes()
        sub = td.subset(er.fold_docs(n, k, f)[0])
        want = tc.category_map(sub.labels, sub.categories)
        assert list(cm.items()) == list(want.items())
        assert np.array_equal(classes, np.unique(sub.labels))
        train = fold.rows(False)
        assert np.array_equal(classes[cls_doc[train]], td.labels[train])


def test_fold_training_data_cuts_lazily_and_empty_raises():
    td = _data(6, 2)
    fold = tc.TextFold(_Folds(6, 3), 1, td)
    ftd = tc.TrainingData(stopWords=td.stopWords, fold=fold)
    assert ftd.on_device and len(ftd) == 4
    sub = td.subset([0, 2, 3, 5])
    assert np.array_equal(ftd.labels, sub.labels) and ftd.categories == sub.categories and not ftd.on_device
    assert np.array_equal(ftd.tokens[0], sub.tokens[0]) and np.array_equal(ftd.tokens[1], sub.tokens[1])
    assert [(o.label, o.text, o.category) for o in ftd.data] == [(o.label, o.text, o.category) for o in sub.data]
    empty = tc.TrainingData(stopWords=td.stopWords, fold=tc.TextFold(_Folds(1, 1), 0, _data(1, 3)))
    pd = tc.Preparator(tc.PreparatorParams(nGram=1)).prepare(None, empty)
    with pytest.raises(ValueError) as e:
        tc.NBAlgorithm(tc.NBAlgorithmParams(1.0)).train(None, pd)
    host = tc.Preparator(tc.PreparatorParams(nGram=1)).prepare(None, _data(1, 3).subset([]))
    with pytest.raises(ValueError) as e_host:
        tc.NBAlgorithm(tc.NBAlgorithmParams(1.0)).train(None, host)
    assert str(e.value) == str(e_host.value)


def test_serve_columns_equals_serve():
    rng = np.random.default_rng(5)
    n = 400
    for n_algo in (1, 2, 3):
        preds = []
        for a in range(n_algo):
            conf = rng.choice([0.25, 0.5, 0.75, 1.0, math.nan], n)
            cat = np.array([f"c{a}{int(x)}" for x in rng.integers(0, 3, n)], dtype=object)
            preds.append(tc.PredictedColumns(cat, conf))
        got = tc.Serving().serveColumns(None, preds)
        for i in range(n):
            want = tc.Serving().serve(None, [tc.PredictedResult(p.category[i], float(p.confidence[i])) for p in preds])
            assert got.category[i] == want.category
            assert got.confidence[i] == want.confidence or (math.isnan(want.confidence) and math.isnan(got.confidence[i]))


def test_accuracy_columns_is_the_mean_of_the_values():
    folds = []
    values = []
    for m, correct in ((7, 3), (0, 0), (5, 5)):
        actual = np.array(["spam"] * m, dtype=object)
        served = np.array(["spam"] * correct + ["ham"] * (m - correct), dtype=object)
        folds.append((None, SimpleNamespace(n_test=m, actual=lambda a=actual: a),
                      tc.PredictedColumns(served, np.ones(m))))
        values += [1.0] * correct + [0.0] * (m - correct)
    assert tc.Accuracy().calculate_columns(None, folds) == sum(values) / len(values)
    assert math.isnan(tc.Accuracy().calculate_columns(None, folds[1:2]))


def test_columnar_opt_in():
    E, G = tc.AccuracyEvaluation, tc.EngineParamsList()
    sc = SimpleNamespace(world_size=1)
    assert all(ev._columnar(E.engine, ep, E.evaluator, sc) for ep in G.engineParamsList)
    two = EngineParams(dataSourceParams=G.engineParamsList[0].dataSourceParams,
                       preparatorParams=G.engineParamsList[0].preparatorParams,
                       algorithmParamsList=[("nb", tc.NBAlgorithmParams(1.0)), ("nb", tc.NBAlgorithmParams(2.0))])
    assert ev._columnar(E.engine, two, E.evaluator, sc)
    assert not ev._columnar(E.engine, G.engineParamsList[0], E.evaluator, SimpleNamespace(world_size=2))
    plain = ev.MetricEvaluator(tc.Accuracy(), otherMetrics=[type("Plain", (ev.AverageMetric,), {
        "calculate_one": lambda self, q, p, a: 1.0})()])
    assert not ev._columnar(E.engine, G.engineParamsList[0], plain, sc)
