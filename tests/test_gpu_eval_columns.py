"""GPU tests (-m gpu) of the recommendation template's evaluation on device folds (native.EvalFolds,
DataSource.readEvalColumns, Engine.evalColumns): every fold map, factor, top-N and metric score equals what the object
path (DataSource.readEval -> Engine.eval -> calculate_one) gives on the same event file."""
import dataclasses
import datetime as dt

import numpy as np
import pytest

import eval_ref
from test_eval_ref import CASES, _case, _global, _predictions
from pio_b200 import controller as c
from pio_b200 import evaluation as ev
from pio_b200 import native
from pio_b200 import storage as s
from pio_b200 import synth
from pio_b200 import workflow as w
from pio_b200.templates import recommendation as rec

pytestmark = pytest.mark.gpu


def _import(tmp_path, monkeypatch, nu=300, ni=60, nnz=6000, seed=5, implicit=False, no_target=False):
    """A seeded event file of rate events (every third one a buy event when explicit; implicit: view counts as ratings,
    the train-with-view-event data); no_target: one more rate event without a targetEntityId."""
    monkeypatch.setenv("PIO_EVENTDATA_DIR", str(tmp_path / "events"))
    monkeypatch.setenv("PIO_MODELDATA_DIR", str(tmp_path / "models"))
    u, i, r = synth.synth_ratings(nu, ni, nnz, seed=seed, implicit=implicit)
    t0 = dt.datetime(2021, 1, 1, tzinfo=dt.timezone.utc)
    evs = []
    for e in range(nnz):
        d = dict(event="rate", entityType="user", entityId=f"u{u[e]}", targetEntityType="item", targetEntityId=f"i{i[e]}",
                 properties={"rating": float(r[e])}, eventTime=(t0 + dt.timedelta(seconds=e)).isoformat())
        if not implicit and e % 3 == 0:
            d["event"] = "buy"
            del d["properties"]
        evs.append(d)
    if no_target:
        evs.append(dict(event="rate", entityType="user", entityId="u1", targetEntityType="item", properties={"rating": 3.0},
                        eventTime=(t0 + dt.timedelta(seconds=nnz)).isoformat()))
    s.import_events("MyApp1", evs)


def _ds(k_fold=5, num=10):
    return rec.DataSource(rec.DataSourceParams("MyApp1", rec.DataSourceEvalParams(kFold=k_fold, queryNum=num)))


@pytest.mark.parametrize("k_fold", [2, 5])
def test_fold_maps_and_queries_equal_the_object_path(tmp_path, monkeypatch, k_fold):
    _import(tmp_path, monkeypatch)
    ds = _ds(k_fold)
    for (td, _, qas), (ctd, ei, fold) in zip(ds.readEval(None), ds.readEvalColumns(None)):
        assert ei is None and ctd.fold is fold and len(ctd) == len(td)
        um = s.BiMap.stringInt(r.user for r in td.ratings)
        im = s.BiMap.stringInt(r.item for r in td.ratings)
        cum, cim = fold.bimaps()
        assert list(cum.toMap().items()) == list(um.toMap().items())
        assert list(cim.toMap().items()) == list(im.toMap().items())
        assert (fold.n_users, fold.n_items, fold.n_train, fold.n_queries) == (um.size, im.size, len(td), len(qas))
        assert np.array_equal(fold.maps["query_train_user"], [um.getOrElse(q.user, -1) for q, _ in qas])
        assert [cum.inverse(int(x)) for x in fold.maps["query_train_user"] if x >= 0] == \
            [q.user for q, _ in qas if q.user in um]
        assert ctd.ratings == td.ratings                 # the object view of a device fold is the fold itself


@pytest.mark.parametrize("rank,implicit", [(5, False), (10, False), (32, False), (64, False), (10, True)])
def test_factors_from_the_device_fold_equal_the_fold_training(tmp_path, monkeypatch, rank, implicit):
    _import(tmp_path, monkeypatch, nu=400, ni=80, nnz=12000, seed=7)
    ds = _ds()
    sc = w.WorkflowContext(mode="Evaluation")
    algo = rec.ALSAlgorithm(rec.ALSAlgorithmParams(rank=rank, numIterations=5, seed=3, implicitPrefs=implicit))
    for f, ((td, _, _), (ctd, _, fold)) in enumerate(zip(ds.readEval(None), ds.readEvalColumns(sc))):
        if f > 1:
            break
        m_obj = algo.train(sc, rec.Preparator().prepare(sc, td))
        m_dev = algo.train(sc, rec.Preparator().prepare(sc, ctd))
        assert m_dev._bimaps is None                    # string maps not built by training
        for a in ("userFeatures", "productFeatures", "userHas", "productHas"):
            assert np.array_equal(getattr(m_dev, a), getattr(m_obj, a)), (f, a)
        assert m_dev.userStringIntMap.toMap() == m_obj.userStringIntMap.toMap()
        assert m_dev.itemStringIntMap.toMap() == m_obj.itemStringIntMap.toMap()


def test_fold_top_n_equals_batch_predict(tmp_path, monkeypatch):
    _import(tmp_path, monkeypatch)
    ds = _ds(num=7)
    sc = w.WorkflowContext(mode="Evaluation")
    algo = rec.ALSAlgorithm(rec.ALSAlgorithmParams(rank=10, numIterations=5, seed=3))
    for (td, _, qas), (ctd, _, fold) in zip(ds.readEval(None), ds.readEvalColumns(sc)):
        m_obj = algo.train(sc, td)
        m_dev = algo.train(sc, ctd)
        res = algo.batchPredictColumns(sc, m_dev, fold)
        items, scores, cnt = m_dev.recommendProductsForUsers(fold.maps["query_train_user"], fold.num)
        inv = m_dev.itemStringIntMap.inverse
        for (ix, p), row in zip(algo.batchPredict(m_obj, list(enumerate(q for q, _ in qas))), range(fold.n_queries)):
            n = int(res.count[row])
            assert n == len(p.itemScores) == min(int(cnt[row]), fold.num)
            assert [inv(int(x)) for x in res.items[row, :n]] == [x.item for x in p.itemScores]
            assert [float(x) for x in scores[row, :n]] == [x.score for x in p.itemScores]


@pytest.mark.parametrize("seed,n,n_users,n_items,k_fold", CASES)
@pytest.mark.parametrize("num", [1, 4, 10])
def test_rank_counts_equal_the_reference(seed, n, n_users, n_items, k_fold, num):
    users, items, ratings = _case(seed, n, n_users, n_items)
    gu, _ = _global(users)
    gi, _ = _global(items)
    ref = eval_ref.split(gu, gi, ratings, k_fold)
    folds = native.EvalFolds(gu, gi, ratings, k_fold)
    rng = np.random.default_rng(seed + 100)
    for f in range(k_fold):
        r = ref[f]
        assert folds.sizes(f) == (r["user"].shape[0], r["item"].shape[0], r["train_user"].shape[0],
                                  r["query_user"].shape[0])
        m = folds.maps(f)
        for key in ("user", "item", "query_user", "query_train_user"):
            assert np.array_equal(m[key], r[key]), key
        it, cnt = _predictions(rng, r, num)
        res = folds.add_result(f, it, cnt)
        for k in sorted({1, max(num - 1, 1), num, num + 3}):
            for thr in (1.0, 2.0, 4.0, 4.5, 6.0):
                got = res.rank_counts(k, thr)
                want = eval_ref.rank_counts(r, it, cnt, k, thr)
                for g, x in zip(got, want):
                    assert np.array_equal(g, x), (f, k, thr)


def test_eval_folds_rejects_bad_arguments():
    folds = native.EvalFolds(np.array([0, 1, 0]), np.array([0, 0, 1]), np.array([1.0, 2.0, 3.0]), 2)
    with pytest.raises(native.NativeError) as e:
        folds.sizes(2)
    assert e.value.code == native.ERR_ARG
    with pytest.raises(native.NativeError):
        native.EvalFolds(np.array([0, -1]), np.array([0, 0]), np.array([1.0, 2.0]), 2)
    nq = folds.sizes(0)[3]
    with pytest.raises(native.NativeError):
        folds.add_result(0, np.full((nq, 2), 5, np.int32), np.full(nq, 1, np.int32))   # item outside the fold
    als = native.NativeALS(4, 5, 5, seed=1, init_mode=native.INIT_HASH)
    with pytest.raises(native.NativeError):
        folds.set_ratings(0, als)                                                       # sizes do not match


def _implicit(gen):
    return [dataclasses.replace(ep, algorithmParamsList=[(n, dataclasses.replace(p, implicitPrefs=True))
                                                         for n, p in ep.algorithmParamsList])
            for ep in gen.engineParamsList]


def _spy(monkeypatch, cls, name):
    calls = []
    orig = getattr(cls, name)

    def spy(*a, **kw):
        calls.append(a)
        return orig(*a, **kw)
    monkeypatch.setattr(cls, name, staticmethod(spy) if isinstance(cls.__dict__[name], staticmethod) else spy)
    return calls


@pytest.mark.parametrize("implicit", [False, True])
def test_run_evaluation_takes_the_columnar_path_with_equal_scores(tmp_path, monkeypatch, implicit):
    _import(tmp_path, monkeypatch, implicit=implicit)
    evaluation = rec.RecommendationEvaluation()
    gen = rec.EngineParamsList(appName="MyApp1")
    if implicit:
        gen.engineParamsList = _implicit(gen)
    sc = w.WorkflowContext(mode="Evaluation")
    want = evaluation.evaluator.evaluateBase(sc, [(ep, evaluation.engine.eval(sc, ep)) for ep in gen.engineParamsList])
    spy = _spy(monkeypatch, c.Engine, "evalColumns")
    finds = _spy(monkeypatch, s.PEventStore, "findColumns")
    got = ev.run_evaluation(evaluation, gen, sc)
    assert len(spy) == 9 and len(finds) == 1
    assert got.bestIdx == want.bestIdx and got.metricHeader == want.metricHeader
    assert _scores(got) == _scores(want)
    assert not np.isnan(_scores(got)).any()


def _scores(res):
    return [[x.score, *x.otherScores] for _, x in res.engineParamsScores]


class _ObjectOnly(ev.AverageMetric):
    """PositiveCount without calculate_columns."""

    def __init__(self, threshold):
        self.inner = rec.PositiveCount(threshold)

    def calculate_one(self, q, p, a):
        return self.inner.calculate_one(q, p, a)


def test_object_path_when_a_metric_or_the_data_does_not_opt_in(tmp_path, monkeypatch):
    gen = rec.EngineParamsList(appName="MyApp1", ranks=(5, 10), iterations=(2,))
    sc = w.WorkflowContext(mode="Evaluation")
    base = rec.RecommendationEvaluation()

    class Partial(ev.Evaluation):
        engine = base.engine
        evaluator = ev.MetricEvaluator(metric=rec.PrecisionAtK(10, 4.0), otherMetrics=[_ObjectOnly(4.0)])
    _import(tmp_path / "a", monkeypatch)
    spy = _spy(monkeypatch, c.Engine, "evalColumns")
    got = ev.run_evaluation(Partial(), gen, sc)
    assert not spy
    want = Partial.evaluator.evaluateBase(sc, [(ep, base.engine.eval(sc, ep)) for ep in gen.engineParamsList])
    assert _scores(got) == _scores(want)

    _import(tmp_path / "b", monkeypatch, no_target=True)          # a rating without targetEntityId: readEval's path
    got = ev.run_evaluation(base, gen, sc)
    assert len(spy) == 2                                           # tried, declined by readEvalColumns
    want = base.evaluator.evaluateBase(sc, [(ep, base.engine.eval(sc, ep)) for ep in gen.engineParamsList])
    assert _scores(got) == _scores(want)
