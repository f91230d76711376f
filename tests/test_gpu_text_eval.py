"""GPU tests (-m gpu) of the text classification template's device evaluation (native.TextFolds, DESIGN.md 4.18.1).

Every fold's NBModel trained from the resident entries equals, byte for byte, NBAlgorithm.train on readEval's host-cut
subset; every fold's raw test scores equal model.raw_scores of the test texts (the object path's route through
json.dumps), NaN patterns included, and its categories and confidences equal predict per query; run_evaluation's
columnar scores and bestIdx equal the object path's with one read and one featurization per (nGram, numFeatures)."""
import json
import math

import numpy as np
import pytest

from pio_b200 import evaluation as ev
from pio_b200 import native
from pio_b200 import storage as s
from pio_b200 import workflow as w
from pio_b200.controller import EngineParams
from pio_b200.templates import textclassification as tc
from tests.test_gpu_textclassification import CORNERS, _events, corpus, same

pytestmark = pytest.mark.gpu


def _sc():
    return w.WorkflowContext(mode="Evaluation")


def _td(texts, cats, stop=("the", "now", "\ud800")):
    labels = np.array([1.0 if c == "spam" else 0.0 for c in cats])
    return tc.TrainingData(native.text_tokens(texts), labels, cats, stop)


def _cats(n, seed, only_in=None, k=1):
    rng = np.random.default_rng(seed)
    cats = [("spam", "ham", "Ham", "eggs")[int(c)] for c in rng.integers(0, 4, n)]
    if only_in is not None:   # "spam" only in documents that test in fold `only_in`
        cats = [("spam" if (d % k == only_in and c == "spam") else ("ham" if c == "spam" else c))
                for d, c in enumerate(cats)]
    return cats


def _model_bytes_equal(a, b):
    assert np.array_equal(a.labels, b.labels) and a.labels.dtype == b.labels.dtype
    for key in ("pi", "theta", "idf"):
        x, y = getattr(a, key), getattr(b, key)
        assert x.shape == y.shape and x.dtype == y.dtype and x.tobytes() == y.tobytes(), key
    assert a.df.tobytes() == b.df.tobytes() and a.df.dtype == b.df.dtype
    assert list(a.categoryMap.items()) == list(b.categoryMap.items())
    assert (a.nGram, a.numFeatures, a.stopWords) == (b.nGram, b.numFeatures, b.stopWords)


def _check_folds(td, k, n_gram, D, lams):
    """Every fold of td: the device model and predictions against the object path's."""
    folds = native.TextFolds(*td.tokens, sorted(td.stopWords), k)
    texts = [o.text for o in td.data]
    pp = tc.PreparatorParams(nGram=n_gram, numFeatures=D)
    for f in range(k):
        fold = tc.TextFold(folds, f, td)
        train, test = fold.rows(False), fold.rows(True)
        assert (fold.n_train, fold.n_test) == (train.shape[0], test.shape[0])
        ftd = tc.TrainingData(stopWords=td.stopWords, fold=fold)
        for lam in lams:
            algo = tc.NBAlgorithm(tc.NBAlgorithmParams(lam))
            if not train.shape[0]:
                with pytest.raises(ValueError, match="training data is empty"):
                    algo.train(_sc(), tc.Preparator(pp).prepare(_sc(), ftd))
                continue
            got = algo.train(_sc(), tc.Preparator(pp).prepare(_sc(), ftd))
            assert ftd.on_device
            want = algo.train(_sc(), tc.Preparator(pp).prepare(_sc(), td.subset(train)))
            _model_bytes_equal(got, want)
            raw = folds.scores(f, got.idf, got.pi, got.theta)
            assert same(raw, want.raw_scores([texts[i] for i in test.tolist()]))
            cols = algo.batchPredictColumns(_sc(), got, fold)
            per_query = [algo.predict(want, tc.Query(texts[i])) for i in test.tolist()]
            assert cols.category.tolist() == [p.category for p in per_query]
            assert same(cols.confidence, [p.confidence for p in per_query])
    return folds


def _cases():
    n = 40
    return [(k, g, D, lam) for k, g, D, lam in [
        (1, 1, 97, 0.5), (2, 2, 1 << 18, 0.0), (3, 3, 1, 5.0), (5, 1, 1 << 18, 0.5), (n - 1, 2, 97, 5.0),
        (n, 3, 1 << 18, 0.5), (n + 1, 1, 1, 0.0), (5, 3, 97, 0.0), (3, 1, 97, 0.5)]]


@pytest.mark.parametrize("k,n_gram,D,lam", _cases())
def test_fold_models_and_scores_equal_the_object_path(native, k, n_gram, D, lam):
    texts = corpus(100 + k + n_gram, 40)
    _check_folds(_td(texts, _cats(40, k + D)), k, n_gram, D, (lam,))


def test_corner_texts_and_a_label_that_tests_in_one_fold(native):
    texts = list(CORNERS) + corpus(9, 30)[len(CORNERS):]
    for k in (2, 3, 5):
        _check_folds(_td(texts, _cats(len(texts), k, only_in=1, k=k)), k, 2, 97, (0.0, 0.5, 5.0))


@pytest.mark.parametrize("parts", [1, 2, 3])
def test_parts_give_the_same_bytes(native, monkeypatch, parts):
    texts = corpus(17, 90)
    tb, to = native.text_tokens(texts)
    monkeypatch.setenv("PIO_TEXT_BUDGET", str((int(to[-1]) + parts - 1) // parts))
    folds = _check_folds(_td(texts, _cats(90, 3)), 4, 2, 1000, (0.5,))
    assert folds.stats()["parts"] >= parts and folds.stats()["featurizations"] == 1


def test_featurization_is_kept_per_pair(native):
    td = _td(corpus(4, 50), _cats(50, 4))
    folds = native.TextFolds(*td.tokens, sorted(td.stopWords), 3)
    for g, D, want in ((1, 50, 1), (1, 50, 1), (2, 50, 2), (2, 60, 3), (2, 60, 3)):
        folds.featurize(g, D)
        assert folds.stats()["featurizations"] == want
    assert folds.stats()["entries"] == native.TextModel(sorted(td.stopWords), 2, 60).features(
        *td.tokens, use_idf=False)[1].shape[0]


def test_bad_arguments_are_rejected(native):
    import ctypes as C
    L = native.lib()
    tb, to = native.text_tokens(["a", "b c"])
    h = C.c_void_p()
    for n, k in ((0, 1), (2, 0)):
        assert L.pio_text_folds_create(0, None, np.zeros(1, np.int64).ctypes.data, 0, tb.ctypes.data, to.ctypes.data,
                                       n, k, C.addressof(h)) == native.ERR_ARG
    folds = native.TextFolds(tb, to, [], 2)
    with pytest.raises(native.NativeError) as e:
        folds.train_nb(0, [0, 0], 1, 1.0)
    assert e.value.code == native.ERR_STATE
    folds.featurize(1, 10)
    for fold in (-1, 2):
        with pytest.raises(native.NativeError) as e:
            folds.sizes(fold)
        assert e.value.code == native.ERR_ARG
    for cls, lam in (([0, 1], 1.0), ([0, 0], -1.0), ([0, 0], float("nan"))):
        with pytest.raises(native.NativeError) as e:
            folds.train_nb(0, cls, 1, lam)     # document 1 trains in fold 0: its class must be < n_class
        assert e.value.code == native.ERR_ARG
    for args in ((0, 10), (1, 0)):
        with pytest.raises(native.NativeError) as e:
            folds.featurize(*args)
        assert e.value.code == native.ERR_ARG


# ---- the template end to end -------------------------------------------------------------------------------------------
RAW_TEXTS = ['"caf\xc3\xa9 na\xc3\xafve \xe6\x97\xa5\xe6\x9c\xac"', '"a\\/b \\/ c/"', '"\\ud83d\\ude00 x \\ud83d\\ude00"',
             '"\xf0\x9f\x98\x80 raw \xf0\x9f\x98\x80\xf0\x9f\x98\x80"', '"lone \\ud800 and \\udc00 z\\udc00z"',
             '"mix \\u00e9 \xc3\xa9 \\\\ \\" the"']


def _import(app, n, seed, raw=True):
    evs = _events(n, seed)
    s.import_events(app, evs)
    if raw:   # lines written by hand: raw UTF-8, \/, escaped and raw surrogate pairs, lone surrogates
        line = json.loads(s.app_file(app).read_text().splitlines()[0])
        line.pop("eventId", None)
        with open(s.app_file(app), "ab") as fh:
            for i, t in enumerate(RAW_TEXTS * 3):
                line["entityId"] = f"r{i}"
                line["properties"] = {"text": "@TEXT@", "label": "spam" if i % 2 else "ham"}
                fh.write(json.dumps(line).encode().replace(b'"@TEXT@"', t.encode("latin-1")) + b"\n")
    return evs


class _Spy:
    def __init__(self, monkeypatch):
        self.columns = self.reads = 0
        self.folds = []
        real_cols, real_read, real_folds = tc.Engine.evalColumns, tc.DataSource._read, native.TextFolds
        spy = self

        def cols(eng, *a, **kw):
            spy.columns += 1
            return real_cols(eng, *a, **kw)

        def read(ds, sc):
            spy.reads += 1
            return real_read(ds, sc)

        class Folds(real_folds):
            def __init__(self, *a, **kw):
                super().__init__(*a, **kw)
                spy.folds.append(self)
        monkeypatch.setattr(tc.Engine, "evalColumns", cols)
        monkeypatch.setattr(tc.DataSource, "_read", read)
        monkeypatch.setattr(native, "TextFolds", Folds)


def _object(evaluation, gen, sc):
    return evaluation.evaluator.evaluateBase(sc, [(ep, evaluation.engine.eval(sc, ep)) for ep in gen.engineParamsList])


def _same_scores(a, b):
    def eq(u, v):
        return (u != u and v != v) or u == v
    assert a.bestIdx == b.bestIdx
    assert a.bestEngineParams == b.bestEngineParams
    for (_, x), (_, y) in zip(a.engineParamsScores, b.engineParamsScores):
        assert eq(x.score, y.score) and all(eq(u, v) for u, v in zip(x.otherScores, y.otherScores))


def _generator(ep_list):
    g = tc.EngineParamsList()
    g.engineParamsList = ep_list
    return g


def test_event_file_raw_tokens_equal_the_object_path(native, tmp_path, monkeypatch):
    monkeypatch.setenv("PIO_EVENTDATA_DIR", str(tmp_path / "events"))
    _import("MyTextApp", 60, 11)
    td = tc.DataSource(tc.DataSourceParams(appName="MyTextApp"))._read(_sc())
    assert len(td) == 60 + 3 * len(RAW_TEXTS)
    for k, g in ((3, 1), (5, 2)):
        _check_folds(td, k, g, 500, (0.5, 5.0))


@pytest.mark.parametrize("variant", ["doc", "two_ngrams", "two_nb"])
def test_run_evaluation_columnar_equals_object(native, tmp_path, monkeypatch, variant):
    monkeypatch.setenv("PIO_EVENTDATA_DIR", str(tmp_path / "events"))
    monkeypatch.chdir(tmp_path)
    _import("MyTextApp", 300, 12)
    G = tc.EngineParamsList(evalK=5)
    if variant == "two_ngrams":
        G = _generator(G.engineParamsList + tc.EngineParamsList(evalK=5, nGram=2).engineParamsList)
    elif variant == "two_nb":
        base = G.engineParamsList[0]
        G = _generator([EngineParams(dataSourceParams=base.dataSourceParams, preparatorParams=base.preparatorParams,
                                     algorithmParamsList=[("nb", tc.NBAlgorithmParams(a)), ("nb", tc.NBAlgorithmParams(b))])
                        for a, b in ((0.5, 5.0), (5.0, 0.5), (0.0, 1.0), (1.0, 1.0))])
    spy = _Spy(monkeypatch)
    got = ev.run_evaluation(tc.AccuracyEvaluation, G, _sc())
    assert spy.columns == len(G.engineParamsList) and spy.reads == 1 and len(spy.folds) == 1
    assert spy.folds[0].stats()["featurizations"] == (2 if variant == "two_ngrams" else 1)
    _same_scores(got, _object(tc.AccuracyEvaluation, G, _sc()))


def test_best_json_trains_the_best_variant(native, tmp_path, monkeypatch):
    monkeypatch.setenv("PIO_EVENTDATA_DIR", str(tmp_path / "events"))
    monkeypatch.setenv("PIO_MODELDATA_DIR", str(tmp_path / "models"))
    monkeypatch.chdir(tmp_path)
    _import("MyTextApp", 200, 13)
    variant = tmp_path / "engine.json"
    variant.write_text(json.dumps({
        "engineFactory": "pio_b200.templates.textclassification.TextClassificationEngine",
        "datasource": {"params": {"appName": "MyTextApp"}}, "preparator": {"params": {"nGram": 1}},
        "algorithms": [{"name": "nb", "params": {"lambda": 1.0}}]}))
    res = w.CreateWorkflow.main([
        "--engine-id", "tc", "--engine-version", "1", "--engine-variant", str(variant),
        "--evaluation-class", "pio_b200.templates.textclassification.AccuracyEvaluation",
        "--engine-params-generator-class", "pio_b200.templates.textclassification.EngineParamsList"])
    assert isinstance(res, ev.MetricEvaluatorResult)
    _same_scores(res, _object(tc.AccuracyEvaluation, tc.EngineParamsList(), _sc()))
    best = json.loads((tmp_path / "best.json").read_text())
    assert best["algorithms"][0]["params"]["lambda"] == res.bestEngineParams.algorithmParamsList[0][1].lambda_
    inst = w.CreateWorkflow.main(["--engine-id", "tc", "--engine-version", "1", "--engine-variant", "best.json"])
    assert inst.status == "COMPLETED"
    model = w.deploy(inst.id).models[0]
    want = tc.TextClassificationEngine().apply().train(w.WorkflowContext(), res.bestEngineParams)[0]
    _model_bytes_equal(model, want)


def _raises(fn):
    try:
        fn()
    except Exception as e:   # noqa: BLE001
        return type(e), str(e)
    return None


def test_empty_training_fold_raises_as_the_object_path(native, tmp_path, monkeypatch):
    monkeypatch.setenv("PIO_EVENTDATA_DIR", str(tmp_path / "events"))
    _import("MyTextApp", 1, 14, raw=False)
    for k in (1, 2):
        G = tc.EngineParamsList(evalK=k)
        assert tc.DataSource(tc.DataSourceParams(appName="MyTextApp", evalK=k)).readEvalColumns(_sc()) is not None
        got = _raises(lambda: ev.run_evaluation(tc.AccuracyEvaluation, G, _sc()))
        assert got is not None and got[0] is ValueError
        assert got == _raises(lambda: _object(tc.AccuracyEvaluation, G, _sc()))


def test_evalK_0_and_an_empty_app_take_the_object_path(native, tmp_path, monkeypatch):
    monkeypatch.setenv("PIO_EVENTDATA_DIR", str(tmp_path / "events"))
    _import("MyTextApp", 30, 15, raw=False)
    s.import_events("Empty", [dict(event="stopwords", entityType="resource", entityId="s", properties={"word": "a"})])
    for app, k in (("MyTextApp", 0), ("Empty", 3)):
        assert tc.DataSource(tc.DataSourceParams(appName=app, evalK=k)).readEvalColumns(_sc()) is None
        G = tc.EngineParamsList(appName=app, evalK=k)
        got = _raises(lambda: ev.run_evaluation(tc.AccuracyEvaluation, G, _sc()))
        assert got == _raises(lambda: _object(tc.AccuracyEvaluation, G, _sc()))
        if got is None:
            assert all(math.isnan(x.score) for _, x in ev.run_evaluation(tc.AccuracyEvaluation, G, _sc()).engineParamsScores)
    G = tc.EngineParamsList(evalK=None)
    got = _raises(lambda: ev.run_evaluation(tc.AccuracyEvaluation, G, _sc()))
    assert got is not None and got == _raises(lambda: _object(tc.AccuracyEvaluation, G, _sc()))
