"""CPU checks of the classification evaluation's restatement (tests/cls_eval_ref.py) against the template's own
definitions -- readEval's cut, np.unique, Accuracy / Precision through calculate_one -- and of MetricEvaluator's
outputPath variant."""
import json
import math

import numpy as np
import pytest

import pio_b200  # noqa: F401
from pio_b200 import evaluation as ev
from pio_b200.controller import EngineParams
from pio_b200.templates import classification as cl

from tests import cls_eval_ref as ref


def _object_scores(labels, preds, k):
    """Accuracy and Precision(0/1/2/never-predicted) through calculate / calculate_one over readEval-shaped folds."""
    data = []
    for f in range(k):
        _, test = ref.fold_rows(labels.shape[0], k, f)
        data.append((None, [(cl.Query(0.0, 0.0, 0.0), cl.PredictedResult(float(preds[i])), cl.ActualResult(float(labels[i])))
                            for i in test]))
    metrics = [cl.Accuracy()] + [cl.Precision(v) for v in (0.0, 1.0, 2.0, 1.5, 99.0)]
    return [m.calculate(None, data) for m in metrics]


def _ref_scores(labels, preds, k):
    out = []
    for j, lab in enumerate((0.0, 0.0, 1.0, 2.0, 1.5, 99.0)):
        fc = []
        for f in range(k):
            _, test = ref.fold_rows(labels.shape[0], k, f)
            fc.append(ref.counts(preds[test], labels[test], lab))
        out.append(ref.accuracy(fc) if j == 0 else ref.precision(fc))
    return out


def _same(a, b):
    return all((math.isnan(x) and math.isnan(y)) or x == y for x, y in zip(a, b))


@pytest.mark.parametrize("n,k,seed", [(1, 1, 0), (1, 3, 1), (4, 5, 2), (7, 7, 3), (8, 7, 4), (997, 5, 5), (1000, 3, 6),
                                      (50, 2, 7), (13, 20, 8)])
@pytest.mark.parametrize("kind", ["int", "frac"])
def test_counts_give_the_object_scores(n, k, seed, kind):
    rng = np.random.default_rng(seed)
    vals = np.array([0.0, 1.0, 2.0, 3.0]) if kind == "int" else np.array([0.0, 1.5, 2.0, 0.25])
    labels = rng.choice(vals, n)
    preds = np.where(rng.uniform(size=n) < 0.6, labels, rng.choice(vals, n))
    assert _same(_object_scores(labels, preds, k), _ref_scores(labels, preds, k))


def test_precision_of_a_label_never_predicted_is_nan():
    labels = np.array([0.0, 1.0, 1.0, 0.0])
    s = _object_scores(labels, labels.copy(), 2)
    assert math.isnan(s[-1]) and math.isnan(_ref_scores(labels, labels.copy(), 2)[-1])


@pytest.mark.parametrize("n,k", [(1, 1), (1, 2), (4, 3), (5, 5), (6, 5), (30, 7), (3, 9)])
def test_fold_cut_and_training_classes(n, k):
    rng = np.random.default_rng(n * 31 + k)
    labels = rng.choice([0.0, 1.0, 2.5, 7.0], n)
    labels[n - 1] = 42.0                       # a label whose only row tests in one fold
    for f in range(k):
        train, test = ref.fold_rows(n, k, f)
        assert np.array_equal(np.sort(np.concatenate([train, test])), np.arange(n))
        assert np.array_equal(ref.train_position(train, k, f), np.arange(train.shape[0]))
        assert np.array_equal(test, f + np.arange(test.shape[0]) * k)
        assert np.array_equal(ref.train_classes(labels, k, f), np.unique(labels[train]))


def test_read_eval_cut_matches_the_restatement(monkeypatch):
    rng = np.random.default_rng(3)
    n = 23
    labels = rng.choice([0.0, 1.0, 1.5], n)
    x64 = rng.uniform(0, 9, (n, 3))
    ds = cl.DataSource(cl.DataSourceParams(appName="A", evalK=4))
    monkeypatch.setattr(ds, "_read", lambda sc: cl.TrainingData(labels, x64.astype(np.float32), x64))
    folds = ds.readEval(None)
    assert len(folds) == 4
    for f, (td, ei, qas) in enumerate(folds):
        train, test = ref.fold_rows(n, 4, f)
        assert ei is None
        assert np.array_equal(td.labels, labels[train]) and np.array_equal(td.features64, x64[train])
        assert td.features.dtype == np.float32 and np.array_equal(td.features, x64[train].astype(np.float32))
        assert [(q.attr0, q.attr1, q.attr2) for q, _ in qas] == [tuple(r) for r in x64[test].tolist()]
        assert [a.label for _, a in qas] == labels[test].tolist()


def test_read_eval_needs_evalK():
    ds = cl.DataSource(cl.DataSourceParams(appName="A"))
    for read in (ds.readEval, ds.readEvalColumns):
        with pytest.raises(AssertionError, match="requirement failed: DataSourceParams.evalK must not be None"):
            read(None)


def test_engine_json_without_evalK_parses_as_before():
    eng = cl.ClassificationEngine().apply()
    ep = eng.jValueToEngineParams({"datasource": {"params": {"appName": "X"}},
                                   "algorithms": [{"name": "naive", "params": {"lambda": 2.0}}]})
    assert ep.dataSourceParams[1] == cl.DataSourceParams(appName="X", evalK=None)


def test_generators_and_headers():
    g = cl.EngineParamsList(evalK=5)
    assert [ep.algorithmParamsList[0][1].lambda_ for ep in g.engineParamsList] == [10.0, 100.0, 1000.0]
    assert all(ep.dataSourceParams[1].evalK == 5 for ep in g.engineParamsList)
    rf = cl.RandomForestParamsList()
    assert [ep.algorithmParamsList[0][1].maxDepth for ep in rf.engineParamsList] == [4, 6, 8]
    ev_ = cl.CompleteEvaluation.evaluator
    assert ev_.outputPath == "best.json"
    assert [m.header for m in ev_.otherMetrics] == ["Precision(label = 0.0)", "Precision(label = 1.0)",
                                                   "Precision(label = 2.0)"]
    assert cl.PrecisionEvaluation.evaluator.metric.header == "Precision(label = 1.0)"


class _Metric(ev.AverageMetric):
    def calculate_one(self, q, p, a):
        return p


def test_metric_evaluator_writes_the_best_variant(tmp_path):
    """outputPath: the best engine params as an engine variant that jValueToEngineParams reads back."""
    eng = cl.ClassificationEngine().apply()
    eps = [EngineParams(dataSourceParams=("", cl.DataSourceParams(appName="A", evalK=3)),
                        algorithmParamsList=[("naive", cl.AlgorithmParams(lam))]) for lam in (1.0, 2.0)]
    eps.append(EngineParams(dataSourceParams=("", cl.DataSourceParams(appName="B", evalK=None)),
                            algorithmParamsList=[("randomforest", cl.RandomForestAlgorithmParams(4, 5, "auto", "gini", 6,
                                                                                                  100)),
                                                 ("naive", cl.AlgorithmParams(3.5))]))
    out = tmp_path / "best.json"
    me = ev.MetricEvaluator(_Metric(), outputPath=str(out))
    for best in range(3):
        data = [(ep, [(None, [(None, 1.0 if j == best else 0.0, None)])]) for j, ep in enumerate(eps)]
        r = me.evaluateBase(None, data, cl.CompleteEvaluation)
        assert r.bestIdx == best
        variant = json.loads(out.read_text())
        assert variant["engineFactory"] == "pio_b200.templates.classification.CompleteEvaluation"
        assert variant["description"] == "" and variant["id"].startswith(variant["engineFactory"] + " ")
        assert eng.jValueToEngineParams(variant) == eps[best]
    alg = json.loads(out.read_text())["algorithms"]
    assert alg[1] == {"name": "naive", "params": {"lambda": 3.5}}
    from pio_b200 import workflow as w
    assert isinstance(w.get_engine(variant["engineFactory"]), type(eng))


def test_metric_evaluator_without_output_path_writes_nothing(tmp_path, monkeypatch):
    monkeypatch.chdir(tmp_path)
    me = ev.MetricEvaluator(_Metric())
    me.evaluateBase(None, [("a", [(None, [(None, 1.0, None)])])], cl.CompleteEvaluation)
    assert list(tmp_path.iterdir()) == []
