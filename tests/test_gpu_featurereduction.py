"""GPU tests (-m gpu) of the dimensionality-reduction template's device path (native.FeatureData / FeatureModel,
pio_fr_*) and of the template (templates/featurereduction.py) against tests/featurereduction_ref.py.

Exact (byte for byte): the parsed rows with their statuses, the mean and Gramian of integer data, the projections,
sigma and the prediction scores.  Within a bound: the Gramian of non-integer data (gamma_m sum |x_i||x_j|), the loss
and gradient (1e-12 relative: the device's exp and log1p against NumPy's) and the trained objectives."""
import json
import math
import pickle

import numpy as np
import pytest

from pio_b200 import evaluation as ev
from pio_b200 import native
from pio_b200 import storage as s
from pio_b200 import workflow as w
from pio_b200.templates import featurereduction as fr
from tests import digits
from tests import featurereduction_ref as ref

pytestmark = pytest.mark.gpu


def same(a, b):
    a, b = np.asarray(a, np.float64), np.asarray(b, np.float64)
    return a.shape == b.shape and bool(np.all((np.isnan(a) & np.isnan(b)) | (a.view(np.uint64) == b.view(np.uint64))))


def rows_of(strings):
    return native.text_tokens(strings)


def device_rows(fd, p):
    """The parsed rows read back through an identity projection (exact up to the sign of zero)."""
    return fd.project(np.zeros(p), np.eye(p), copy_out=True)


def plan_parts(off, budget):
    """text_plan.h's rule: a part closes before the row that would take it over the budget."""
    parts, acc = 0, 0
    for r in range(off.shape[0] - 1):
        wd = int(off[r + 1] - off[r])
        if parts == 0 or acc + wd > budget:
            parts, acc = parts + 1, 0
        acc += wd
    return parts


MIXED = ["1, 2, 3", "4.5, -0, 7e2", "1d, 0x1p3, 2", " 8 , 9, 10, ", "9007199254740991, 1e22, 1e-22",
         "9007199254740993, 1e23, 1e-23", "0.000000000000000000000000001, 3, 3", "+5, .5, 5.", "NaN, 1, 2",
         "1, 2", "1, , 3", ", 1, 2", "1, 2, 3, 4", "1,2, 3", "1, 1e400, 2", "-Infinity, 0, 0"]


@pytest.mark.parametrize("budget", [None, "120", "60"])
def test_parse_statuses_and_values(budget, monkeypatch):
    if budget:
        monkeypatch.setenv("PIO_FR_BUDGET", budget)
    fd = native.FeatureData()
    status, p = fd.parse(*rows_of(MIXED))
    want_status, X, wp = ref.parse_rows([t.encode() for t in MIXED])
    assert p == wp == 3 and status.tolist() == want_status.tolist()
    assert fd.stats()["parts"] == plan_parts(rows_of(MIXED)[1], int(budget) if budget else 1 << 28)
    assert plan_parts(rows_of(MIXED)[1], int(budget) if budget else 1 << 28) == {None: 1, "120": 3, "60": 6}[budget]
    assert fd.stats()["host_rows"] == int((want_status == ref.HOST).sum())
    good = [t for t, st in zip(MIXED, want_status) if st >= 0]
    fd2 = native.FeatureData()
    st2, _ = fd2.parse(*rows_of(good))
    assert (st2 >= 0).all()
    _, Xg, _ = ref.parse_rows([t.encode() for t in good])
    assert same(device_rows(fd2, 3), Xg + 0.0)


def test_bad_first_row_and_long_rows():
    fd = native.FeatureData()
    status, p = fd.parse(*rows_of(["1, x", "1, 2"]))
    assert p == 0 and status.tolist() == [ref.BAD, 0]
    with pytest.raises(native.NativeError):
        fd.gramian()
    with pytest.raises(native.NativeError, match="65535"):
        native.FeatureData().parse(*rows_of([", ".join(["1"] * 65536)]))


def _ints(n, p, seed, hi=255):
    rng = np.random.default_rng(seed)
    X = rng.integers(0, hi + 1, size=(n, p)).astype(np.float64)
    X[rng.random((n, p)) < 0.6] = 0.0
    return X


def _strings(X):
    return [digits.feature_string(r) for r in X]


@pytest.mark.parametrize("n,p", [(2, 1), (255, 7), (256, 7), (257, 7), (4097, 65), (3000, 784), (300, 130)])
def test_mean_gram_projection_exact(n, p):
    X = _ints(n, p, n + p)
    fd = native.FeatureData()
    status, _ = fd.parse(*rows_of(_strings(X)))
    assert (status == 0).all()
    mean, G = fd.gramian()
    assert same(mean, ref.mean(X)) and same(G, X.T @ X)
    P = fr.principal_components(fr.covariance(G, mean, n), p)
    for k in sorted({1, p, min(250, p)}):
        y = fd.project(mean, P[:, :k], copy_out=True)
        assert same(y, ref.transform(X, mean, P[:, :k]))


def test_gram_bound_on_non_integer_data_and_budget_independence(monkeypatch):
    rng = np.random.default_rng(9)
    X = rng.normal(size=(300, 7)) * np.array([1e-3, 1, 10, 1e3, 0.5, 3, 7])
    strs = [", ".join(repr(float(v)) for v in r) for r in X]
    fd = native.FeatureData()
    fd.parse(*rows_of(strs))
    mean, G = fd.gramian()
    exact = ref.gram_exact(X)
    u = 2.0 ** -53
    gamma = 300 * u / (1 - 300 * u)
    assert np.all(np.abs(G - exact) <= gamma * (np.abs(X).T @ np.abs(X)))
    monkeypatch.setenv("PIO_FR_BUDGET", "4000")
    fd2 = native.FeatureData()
    fd2.parse(*rows_of(strs))
    assert fd2.stats()["parts"] >= 3
    m2, G2 = fd2.gramian()
    assert same(m2, mean) and same(G2, G)
    # from the device's covariance on, the pipeline is exact
    P = fr.principal_components(fr.covariance(G, mean, 300), 4)
    assert same(fd.project(mean, P, copy_out=True), ref.transform(X, mean, P))


def _prepared(n, p, k, labels, seed):
    x, y = digits.digits(n, seed=seed, labels=labels)
    X = x[:, :p].astype(np.float64)
    fd = native.FeatureData()
    fd.parse(*rows_of(_strings(X)))
    mean, G = fd.gramian()
    P = fr.principal_components(fr.covariance(G, mean, n), k)
    Y = fd.project(mean, P, copy_out=True)
    return fd, X, y, mean, P, Y


@pytest.mark.parametrize("n", [2, 255, 256, 257, 600])
def test_sigma_exact_and_loss_gradient_bound(n):
    fd, X, y, mean, P, Y = _prepared(n, 784, 12, 3, n)
    classes = np.unique(y)
    cls = np.searchsorted(classes, y).astype(np.int32)
    sd = fd.lr_prepare(cls, classes.shape[0])
    assert same(sd, ref.sigma(Y))
    rng = np.random.default_rng(n)
    labs = np.arange(classes.shape[0], dtype=np.int32)
    wb = rng.normal(size=(labs.shape[0], 13))
    for reg in (0.0, 0.5):
        f, g = fd.lr_eval(labs, wb, reg)
        for a, c in enumerate(labs.tolist()):
            rf, rg = ref.loss_grad(Y, sd, (cls == c).astype(np.float64), wb[a], reg)
            assert abs(f[a] - rf) <= 1e-12 * abs(rf)
            assert np.all(np.abs(g[a] - rg) <= 1e-12 * (np.abs(rg) + np.abs(wb[a]) * reg + 1e-3))
        # a class's values do not depend on its neighbours in the call
        f1, g1 = fd.lr_eval(labs[-1:], wb[-1:], reg)
        assert same(f1, f[-1:]) and same(g1, g[-1:])


def _train(pd, reg):
    return fr.LRAlgorithm(fr.LRAlgorithmParams(reg)).train(None, pd)


class _TD:
    def __init__(self, X, y):
        self.tokens, self.labels = rows_of(_strings(X)), np.asarray(y, np.float64)
        self.lines = np.arange(len(y))

    def __len__(self):
        return self.labels.shape[0]


@pytest.mark.parametrize("labels,k,reg", [(1, 3, 0.5), (2, 5, 0.1), (10, 40, 1.0)])
def test_training_against_the_restatement(labels, k, reg):
    x, y = digits.digits(900, seed=labels, labels=labels)
    X = x.astype(np.float64)
    pd = fr.PreparedData(_TD(X, y), fr.PreparatorParams(k))
    m = _train(pd, reg)
    m2 = _train(fr.PreparedData(_TD(X, y), fr.PreparatorParams(k)), reg)
    assert same(m.coef, m2.coef) and same(m.intercept, m2.intercept)       # run to run
    classes = np.unique(y)
    if labels == 1:
        assert m.intercept.tolist() == [math.inf] and not m.coef.any()
    _, Y = pd.transformedData
    sd = ref.sigma(Y)
    cls = np.searchsorted(classes, y)
    for c in range(classes.shape[0]):
        yb = (cls == c).astype(np.float64)
        if 0 < yb.sum() < yb.shape[0]:
            x0 = np.zeros(k + 1)
            x0[k] = math.log(yb.sum() / (yb.shape[0] - yb.sum()))

            def evaluate(idx, pts, yb=yb):
                fs, gs = zip(*[ref.loss_grad(Y, sd, yb, q, reg) for q in pts])
                return np.array(fs), np.array(gs)

            rx, rf, _, _ = fr.minimize_many([x0], evaluate)[0]
            wd = np.append(m.coef[c] * np.where(sd != 0, sd, 0), m.intercept[c])
            fd_ = ref.loss_grad(Y, sd, yb, wd, reg)[0]
            assert abs(fd_ - rf) <= 1e-9 * abs(rf)
    raw = m.raw_scores(_strings(X[:300]))
    assert same(raw, ref.scores(Y[:300], m.coef, m.intercept))
    got = fr.LRAlgorithm(fr.LRAlgorithmParams(reg)).predictMany(m, [fr.Query(t) for t in _strings(X[:300])])
    assert [p.label for p in got] == classes[ref.predict(raw)].tolist()


def _events(n, seed, labels=10):
    x, y = digits.digits(n, seed=seed, labels=labels)
    return digits.events(x, y), x


def test_template_end_to_end(tmp_path, monkeypatch):
    monkeypatch.setenv("PIO_EVENTDATA_DIR", str(tmp_path / "events"))
    monkeypatch.setenv("PIO_MODELDATA_DIR", str(tmp_path / "models"))
    evs, x = _events(600, 5)
    s.import_events("FeatureReduction", evs)
    variant = tmp_path / "engine.json"
    variant.write_text(json.dumps({
        "id": "default", "description": "Default settings",
        "engineFactory": "pio_b200.templates.featurereduction.ClassificationEngine",
        "datasource": {"params": {"appName": "FeatureReduction"}},
        "preparator": {"params": {"numFeatures": 250}},
        "algorithms": [{"name": "lr", "params": {"regParam": 1.0}}]}))
    inst = w.CreateWorkflow.main(["--engine-id", "fr", "--engine-version", "1", "--engine-variant", f"file:{variant}"])
    assert inst.status == "COMPLETED"
    server = w.deploy(inst.id)
    model, algo = server.models[0], server.algorithms[0]
    queries = [digits.feature_string(r) for r in x[:40]] + ["0, " * 783 + "1d"]
    got = [server.query({"features": q}) for q in queries]
    qs = [fr.Query(q) for q in queries]
    many = algo.predictMany(model, qs)
    assert [g["label"] for g in got] == [p.label for p in many]
    assert sum(p.label == e["properties"]["label"] for p, e in zip(many, evs[:40])) >= 30
    again = pickle.loads(pickle.dumps(model))
    assert "_handle" not in again.__dict__
    assert [p.label for p in algo.predictMany(again, qs)] == [p.label for p in many]
    with pytest.raises(ValueError, match="query 2"):
        algo.predictMany(model, [qs[0], qs[1], fr.Query("1, 2")])
    (tmp_path / "in.json").write_text("\n".join(json.dumps({"features": q}) for q in queries) + "\n")
    out = tmp_path / "out.json"
    assert w.BatchPredict.main(["--input", str(tmp_path / "in.json"), "--output", str(out),
                                "--engine-instance-id", inst.id]) == len(queries)
    lines = out.read_text().splitlines()
    assert lines == [json.dumps({"query": {"features": q}, "prediction": w.to_json(p)}, separators=(",", ":"))
                     for q, p in zip(queries, many)]


def test_bad_row_names_its_line(tmp_path, monkeypatch):
    monkeypatch.setenv("PIO_EVENTDATA_DIR", str(tmp_path / "events"))
    evs, _ = _events(6, 6)
    evs[3]["properties"]["features"] = "1, 2, x"
    s.import_events("FeatureReduction", evs)
    td = fr.DataSource(fr.DataSourceParams(appName="FeatureReduction")).readTraining(w.WorkflowContext())
    with pytest.raises(ValueError, match="line 4"):
        fr.PreparedData(td, fr.PreparatorParams(2))
    with pytest.raises(ValueError, match="<= 1 row"):
        fr.PreparedData(td.subset([0]), fr.PreparatorParams(2))


def test_evaluation_writes_best_json(tmp_path, monkeypatch):
    monkeypatch.setenv("PIO_EVENTDATA_DIR", str(tmp_path / "events"))
    monkeypatch.setenv("PIO_MODELDATA_DIR", str(tmp_path / "models"))
    monkeypatch.chdir(tmp_path)
    evs, _ = _events(300, 8)
    s.import_events("FeatureReduction", evs)
    variant = tmp_path / "engine.json"
    variant.write_text(json.dumps({
        "engineFactory": "pio_b200.templates.featurereduction.ClassificationEngine",
        "datasource": {"params": {"appName": "FeatureReduction"}}, "preparator": {"params": {"numFeatures": 20}},
        "algorithms": [{"name": "lr", "params": {"regParam": 1.0}}]}))
    gen = tmp_path / "gen_params.py"
    gen.write_text("from pio_b200.templates import featurereduction as fr\n"
                   "class Small(fr.EngineParamsList):\n"
                   "    def __init__(self):\n"
                   "        super().__init__(numFeatures=20)\n")
    monkeypatch.syspath_prepend(str(tmp_path))
    res = w.CreateWorkflow.main([
        "--engine-id", "fr", "--engine-version", "1", "--engine-variant", str(variant),
        "--evaluation-class", "pio_b200.templates.featurereduction.AccuracyEvaluation",
        "--engine-params-generator-class", "gen_params.Small"])
    assert isinstance(res, ev.MetricEvaluatorResult)
    best = json.loads((tmp_path / "best.json").read_text())
    assert best["algorithms"][0]["params"]["regParam"] == res.bestEngineParams.algorithmParamsList[0][1].regParam
    assert 0.5 <= res.bestScore.score <= 1.0
    (tmp_path / "best_variant.json").write_text(json.dumps({**best, "engineFactory":
                                                            "pio_b200.templates.featurereduction.ClassificationEngine"}))
    inst = w.CreateWorkflow.main(["--engine-id", "fr", "--engine-version", "1", "--engine-variant",
                                  str(tmp_path / "best_variant.json")])
    assert inst.status == "COMPLETED"
