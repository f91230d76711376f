"""GPU tests (-m gpu) of the classification template's device evaluation (native.ClsFolds, DESIGN.md 4.12): fold sizes
and training classes equal the host cut (tests/cls_eval_ref.py), models trained from a fold equal -- bit for bit, node
for node -- those trained on the host-cut rows, predicted labels equal predict per query, run_evaluation's columnar
scores and bestIdx equal the object path's, best.json trains the best variant, and bad input raises as on the host."""
import json

import numpy as np
import pytest

from pio_b200 import evaluation as ev
from pio_b200 import mllib
from pio_b200 import native
from pio_b200 import storage as s
from pio_b200 import workflow as w
from pio_b200.templates import classification as cl
from tests import cls_eval_ref as ref

pytestmark = pytest.mark.gpu

NODE_KEYS = ("tree_off", "feature", "left", "right", "prediction", "count", "threshold", "impurity", "gain")


def _rows(n, seed, labels=(0.0, 1.0, 2.0, 3.0)):
    rng = np.random.default_rng(seed)
    x = rng.integers(0, 10, (n, 3)).astype(np.float64) + np.round(rng.uniform(0, 1, (n, 3)), 1)
    y = np.asarray(labels, np.float64)[np.clip(((x[:, 0] + x[:, 1]) // 5).astype(int), 0, len(labels) - 1)]
    noise = rng.uniform(size=n) < 0.2
    y[noise] = rng.choice(np.asarray(labels, np.float64), int(noise.sum()))
    return y, x


def _cases():
    out = []
    for k in (1, 2, 3, 5, 7):
        for n in sorted({1, k - 1, k, k + 1, 997}):
            if n >= 1:
                out.append((n, k))
    out.append((12_600, 5))      # 10 080 training rows per fold: above the forest's split-sample cut of 10 000
    return out


@pytest.mark.parametrize("n,k", _cases())
def test_fold_sizes_classes_and_nb(native, n, k):
    y, x = _rows(n, n + k)
    if n > k:
        y[k] = 9.5                # a label whose only row tests in fold 0
    folds = native.ClsFolds(y, x, k)
    for f in range(k):
        train, test = ref.fold_rows(n, k, f)
        assert folds.sizes(f) == (train.shape[0], test.shape[0])
        assert np.array_equal(folds.classes(f), np.unique(y[train]))
        if not train.shape[0]:
            continue
        for lam in (10.0, 100.0, 1000.0):
            got = mllib.NaiveBayes.trainFold(folds, f, lam)
            want = mllib.NaiveBayes.train(y[train], x[train].astype(np.float32), lam)
            assert np.array_equal(got.labels, want.labels)
            assert np.array_equal(got.pi, want.pi) and np.array_equal(got.theta, want.theta)
        if test.shape[0]:
            r = folds.nb_predict(f, got.pi, got.theta, got.labels)
            want_p = [got.predict(list(row)) for row in x[test]]
            assert r.labels().tolist() == want_p
            for lab in (0.0, 1.0, 9.5):
                assert r.counts(lab) == ref.counts(np.array(want_p), y[test], lab)


@pytest.mark.parametrize("n,k", [(1, 2), (4, 3), (8, 7), (997, 5), (12_600, 5)])
@pytest.mark.parametrize("impurity,trees,strategy,bins", [("gini", 5, "auto", 100), ("entropy", 1, "sqrt", 32),
                                                          ("gini", 1, "auto", 32), ("entropy", 5, "sqrt", 100)])
def test_forest_from_fold_equals_host(native, n, k, impurity, trees, strategy, bins):
    y, x = _rows(n, n * 7 + k, labels=(0.0, 1.5, 2.0, 3.25))
    folds = native.ClsFolds(y, x, k)
    for f in range(k):
        train, test = ref.fold_rows(n, k, f)
        if not train.shape[0]:
            continue
        args = (4, {}, trees, strategy, impurity, 6, bins)
        got = mllib.RandomForest.trainClassifierFold(folds, f, *args)
        want = mllib.RandomForest.trainClassifier(y[train], x[train], *args)
        for key in NODE_KEYS:
            assert np.array_equal(got.nodes[key], want.nodes[key]), key
        if test.shape[0]:
            r = folds.rf_predict(f, got.nodes, got.numClasses)
            algo = cl.RandomForestAlgorithm(cl.RandomForestAlgorithmParams(4, trees, strategy, impurity, 6, bins))
            assert r.labels().tolist() == [algo.predict(got, cl.Query(*row)).label for row in x[test].tolist()]


def test_forest_fold_timing_counts_the_gather_as_h2d(native):
    y, x = _rows(2000, 1)
    folds = native.ClsFolds(y, x, 5)
    mllib.RandomForest.trainClassifierFold(folds, 2, 4, {}, 5, "auto", "gini", 4, 100)
    t = native.rf_train_timing()
    assert t["h2d_ms"] > 0 and t["levels"] >= 1


# ---- errors ---------------------------------------------------------------------------------------------------------
def _raises(fn):
    try:
        fn()
    except Exception as e:   # noqa: BLE001
        return type(e), str(e)
    return None


def test_training_errors_equal_the_host_ones(native):
    y, x = _rows(40, 2)
    x[13, 1] = -0.5                                    # a negative feature in a training row of fold 0 (row 13 % 3 = 1)
    folds = native.ClsFolds(y, x, 3)
    train, _ = ref.fold_rows(40, 3, 0)
    got = _raises(lambda: mllib.NaiveBayes.trainFold(folds, 0, 1.0))
    assert got is not None and got == _raises(lambda: mllib.NaiveBayes.train(y[train], x[train].astype(np.float32)))
    train1, _ = ref.fold_rows(40, 3, 1)                # row 13 tests in fold 1: its training rows are clean
    assert np.array_equal(mllib.NaiveBayes.trainFold(folds, 1, 1.0).pi, mllib.NaiveBayes.train(y[train1], x[train1]).pi)
    y2 = y.copy()
    y2[20] = 4.0                                       # a label >= numClasses in a training row
    y2[31] = -1.0
    x2 = x.copy()
    x2[25, 2] = np.inf
    errors = 0
    for yy, xx in ((y2, x), (y, x2), (y2, x2)):
        folds = native.ClsFolds(yy, xx, 3)
        for f in range(3):                             # a fold whose bad rows all test in it trains cleanly
            tr, _ = ref.fold_rows(40, 3, f)
            for imp in ("gini", "entropy"):
                args = (4, {}, 5, "auto", imp, 4, 32)
                got = _raises(lambda: mllib.RandomForest.trainClassifierFold(folds, f, *args))
                assert got == _raises(lambda: mllib.RandomForest.trainClassifier(yy[tr], xx[tr], *args))
                errors += got is not None
    assert errors == 16


def test_bad_abi_arguments_are_rejected(native):
    import ctypes as C
    L = native.lib()
    h = C.c_void_p()
    lab = np.zeros(4)
    x = np.zeros((4, 3))
    vp = lambda a: a.ctypes.data_as(C.c_void_p)  # noqa: E731
    for n, F, k in ((0, 3, 2), (4, 0, 2), (4, 3, 0)):
        assert L.pio_cls_folds_create(0, vp(lab), vp(x), C.c_int64(n), C.c_int32(F), C.c_int32(k), C.byref(h)) == native.ERR_ARG
    assert L.pio_cls_folds_create(0, None, vp(x), C.c_int64(4), C.c_int32(3), C.c_int32(2), C.byref(h)) == native.ERR_ARG
    bad = np.array([0.0, np.nan, 1.0, 2.0])
    assert L.pio_cls_folds_create(0, vp(bad), vp(x), C.c_int64(4), C.c_int32(3), C.c_int32(2), C.byref(h)) == native.ERR_ARG
    folds = native.ClsFolds(np.array([0.0, 1.0, 1.0, 2.0]), x, 2)
    out = np.zeros(2, np.int64)
    for fold in (-1, 2):
        assert L.pio_cls_folds_sizes(folds._h, C.c_int32(fold), vp(out)) == native.ERR_ARG
    pi, theta = np.zeros(3), np.zeros((3, 3))
    nc = len(folds.classes(0))
    assert L.pio_cls_folds_nb_train(folds._h, C.c_int32(0), C.c_double(1.0), C.c_int32(nc + 1), vp(pi), vp(theta)) == native.ERR_ARG
    assert L.pio_cls_folds_nb_train(folds._h, C.c_int32(0), C.c_double(1.0), C.c_int32(nc), None, vp(theta)) == native.ERR_ARG
    rid = C.c_int32(-1)
    assert L.pio_cls_folds_nb_predict(folds._h, C.c_int32(0), C.c_int32(0), vp(pi), vp(theta), vp(pi), C.byref(rid)) == native.ERR_ARG
    cnt = np.zeros(4, np.int64)
    assert L.pio_cls_folds_result_counts(folds._h, C.c_int32(123), C.c_double(0.0), vp(cnt)) == native.ERR_ARG
    assert L.pio_cls_folds_result_free(folds._h, C.c_int32(123)) == native.ERR_ARG
    with pytest.raises(native.NativeError):
        folds.rf_predict(0, {"tree_off": np.array([0, 1]), "feature": np.array([5]), "left": np.array([-1]),
                             "right": np.array([-1]), "prediction": np.array([0]), "threshold": np.array([0.0])}, 4)


# ---- the template end to end -----------------------------------------------------------------------------------------
def _import(app, n, seed, labels=None):
    import datetime as dt
    y, x = _rows(n, seed)
    if labels is not None:
        y = labels(y)
    t0 = dt.datetime(2021, 1, 1, tzinfo=dt.timezone.utc).isoformat()
    s.import_events(app, [dict(event="$set", entityType="user", entityId=f"u{i}", eventTime=t0,
                               properties={"plan": float(y[i]), "attr0": float(x[i, 0]), "attr1": float(x[i, 1]),
                                           "attr2": float(x[i, 2])}) for i in range(n)])


class _Spy:
    def __init__(self, monkeypatch):
        self.columns = self.reads = 0
        real_cols, real_read = cl.Engine.evalColumns, cl.DataSource._read

        def cols(eng, *a, **kw):
            self.columns += 1
            return real_cols(eng, *a, **kw)

        def read(ds, sc):
            self.reads += 1
            return real_read(ds, sc)
        monkeypatch.setattr(cl.Engine, "evalColumns", cols)
        monkeypatch.setattr(cl.DataSource, "_read", read)


def _object(evaluation, gen, sc):
    return evaluation.evaluator.evaluateBase(sc, [(ep, evaluation.engine.eval(sc, ep)) for ep in gen.engineParamsList])


def _same_scores(a, b):
    def eq(u, v):
        return (u != u and v != v) or u == v
    assert a.bestIdx == b.bestIdx
    for (_, x), (_, y) in zip(a.engineParamsScores, b.engineParamsScores):
        assert eq(x.score, y.score) and all(eq(u, v) for u, v in zip(x.otherScores, y.otherScores))


@pytest.mark.parametrize("evaluation,gen", [("AccuracyEvaluation", "EngineParamsList"),
                                            ("PrecisionEvaluation", "EngineParamsList"),
                                            ("CompleteEvaluation", "EngineParamsList"),
                                            ("CompleteEvaluation", "RandomForestParamsList")])
def test_run_evaluation_columnar_equals_object(native, tmp_path, monkeypatch, evaluation, gen):
    monkeypatch.setenv("PIO_EVENTDATA_DIR", str(tmp_path / "events"))
    monkeypatch.chdir(tmp_path)
    _import("MyApp1", 1500, 4)
    E, G = getattr(cl, evaluation), getattr(cl, gen)()
    sc = w.WorkflowContext(mode="Evaluation")
    spy = _Spy(monkeypatch)
    got = ev.run_evaluation(E, G, sc)
    assert spy.columns == len(G.engineParamsList) and spy.reads == 1
    _same_scores(got, _object(E, G, sc))


def test_best_json_trains_the_best_variant(native, tmp_path, monkeypatch):
    monkeypatch.setenv("PIO_EVENTDATA_DIR", str(tmp_path / "events"))
    monkeypatch.setenv("PIO_MODELDATA_DIR", str(tmp_path / "models"))
    monkeypatch.chdir(tmp_path)
    _import("MyApp1", 800, 5)
    variant = tmp_path / "engine.json"
    variant.write_text(json.dumps({"engineFactory": "pio_b200.templates.classification.ClassificationEngine",
                                   "datasource": {"params": {"appName": "MyApp1"}}}))
    res = w.CreateWorkflow.main(["--engine-id", "cls", "--engine-version", "1", "--engine-variant", str(variant),
                                 "--evaluation-class", "pio_b200.templates.classification.CompleteEvaluation",
                                 "--engine-params-generator-class", "pio_b200.templates.classification.EngineParamsList"])
    assert isinstance(res, ev.MetricEvaluatorResult)
    best = json.loads((tmp_path / "best.json").read_text())
    assert best["algorithms"][0]["params"]["lambda"] == res.bestEngineParams.algorithmParamsList[0][1].lambda_
    inst = w.CreateWorkflow.main(["--engine-id", "cls", "--engine-version", "1", "--engine-variant", "best.json"])
    assert inst.status == "COMPLETED"
    model = w.deploy(inst.id).models[0]
    want = cl.ClassificationEngine().apply().train(w.WorkflowContext(), res.bestEngineParams)[0]
    assert np.array_equal(model.pi, want.pi) and np.array_equal(model.theta, want.theta)
    assert np.array_equal(model.labels, want.labels)


@pytest.mark.parametrize("labels,declines", [(lambda y: np.where(np.arange(y.shape[0]) == 7, np.nan, y), True),
                                             (lambda y: np.where(y == 0, -0.0, y), True),
                                             (lambda y: y + 0.5, False)])
def test_readEvalColumns_declines_nan_and_negative_zero(native, tmp_path, monkeypatch, labels, declines):
    monkeypatch.setenv("PIO_EVENTDATA_DIR", str(tmp_path / "events"))
    _import("MyApp1", 300, 6, labels)
    sc = w.WorkflowContext(mode="Evaluation")
    ds = cl.DataSource(cl.DataSourceParams(appName="MyApp1", evalK=3))
    assert (ds.readEvalColumns(sc) is None) == declines
    G = cl.EngineParamsList(evalK=3)
    _same_scores(ev.run_evaluation(cl.CompleteEvaluation, G, sc), _object(cl.CompleteEvaluation, G, sc))


def test_evalK_1_and_unset_raise_as_the_object_path(native, tmp_path, monkeypatch):
    monkeypatch.setenv("PIO_EVENTDATA_DIR", str(tmp_path / "events"))
    _import("MyApp1", 50, 7)
    sc = w.WorkflowContext(mode="Evaluation")
    for G in (cl.EngineParamsList(evalK=1), cl.RandomForestParamsList(evalK=1), cl.EngineParamsList(evalK=None)):
        got = _raises(lambda: ev.run_evaluation(cl.AccuracyEvaluation, G, sc))
        assert got is not None and got == _raises(lambda: _object(cl.AccuracyEvaluation, G, sc))
