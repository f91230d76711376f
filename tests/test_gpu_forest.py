"""GPU tests (-m gpu) of the RandomForest classifier (pio_rf_train / pio_rf_predict, mllib.RandomForest): every node of
every forest equals the NumPy restatement tests/forest_ref.py (gini exactly; entropy with gains within 1e-12 on
fixtures whose splits win by a margin), forests are deterministic and independent of how trees are grouped, bad input
raises before any device work, and the classification template trains "randomforest" from its unmodified engine.json."""
import json
import pickle

import numpy as np
import pytest

from pio_b200 import mllib
from pio_b200 import native
from pio_b200 import storage as s
from pio_b200 import workflow as w
from tests import forest_ref as fr

pytestmark = pytest.mark.gpu

INT_KEYS = ("tree_off", "feature", "left", "right", "prediction", "count")
F64_KEYS = ("threshold", "impurity", "gain")


def _data(n, n_feat, n_class, seed, present=None, decimals=1):
    """Features with repeated values and labels that depend on them (plus noise); labels only from `present` classes."""
    rng = np.random.default_rng(seed)
    x = np.round(rng.normal(size=(n, n_feat)) * 3, decimals)
    score = x[:, 0] + 0.5 * x[:, 1 % n_feat] - 0.3 * x[:, -1] + rng.normal(size=n)
    k = present or n_class
    y = np.clip(np.floor((score - score.min()) / (np.ptp(score) + 1e-9) * k), 0, k - 1)
    return y + rng.uniform(0, 0.99, n) * (rng.uniform(size=n) < 0.1), x     # some fractional labels (trunc)


def _assert_same(got, want, exact=True):
    for k in INT_KEYS:
        np.testing.assert_array_equal(got[k], want[k], err_msg=k)
    np.testing.assert_array_equal(got["threshold"].view(np.uint64), want["threshold"].view(np.uint64))
    for k in ("impurity", "gain"):
        if exact:
            np.testing.assert_array_equal(got[k].view(np.uint64), want[k].view(np.uint64), err_msg=k)
        else:
            np.testing.assert_allclose(got[k], want[k], rtol=0, atol=1e-12, err_msg=k)


def _check(y, x, C, T, strategy, impurity, depth, bins, seed=0, held=None):
    m = mllib.RandomForest.trainClassifier(y, x, C, {}, T, strategy, impurity, depth, bins, seed=seed)
    want = fr.train(y, x, C, T, strategy, impurity, depth, bins, seed=seed)
    _assert_same(m.nodes, want, exact=impurity == "gini")
    assert m.numTrees == T and m.totalNumNodes == want["feature"].size
    np.testing.assert_array_equal(m.depth, want["depth"])
    np.testing.assert_array_equal(m.numNodes, np.diff(want["tree_off"]))
    np.testing.assert_array_equal(m.predictBatch(x), fr.predict(want, x))
    if held is not None:
        np.testing.assert_array_equal(m.predictBatch(held), fr.predict(want, held))
    return m, want


GINI_CASES = [
    # n, F, C, present, T, strategy, depth, bins
    (2000, 3, 2, None, 1, "auto", 4, 32),
    (3000, 3, 4, None, 5, "auto", 4, 100),           # the template's parameters
    (1500, 6, 4, None, 64, "auto", 4, 32),
    (3000, 4, 3, None, 3, "all", 0, 32),
    (3000, 4, 3, None, 3, "all", 1, 32),
    (3000, 4, 3, None, 3, "sqrt", 12, 32),
    (2000, 3, 2, None, 5, "auto", 5, 2),
    (50, 3, 2, None, 5, "all", 6, 100),              # maxBins > n
    (9000, 3, 4, None, 5, "auto", 6, 32),            # below the split-sample threshold ...
    (60000, 3, 4, None, 5, "auto", 6, 32),           # ... and above it
    (2000, 5, 6, 4, 5, "auto", 5, 32),               # numClasses larger than the labels present
    (2000, 5, 2, None, 2, "all", 8, 16),
]


@pytest.mark.parametrize("n,F,C,present,T,strategy,depth,bins", GINI_CASES)
def test_gini_forest_equals_restatement(n, F, C, present, T, strategy, depth, bins):
    y, x = _data(n, F, C, seed=n + F + T, present=present)
    _, held = _data(500, F, C, seed=99)
    _check(y, x, C, T, strategy, "gini", depth, bins, seed=T, held=held)


@pytest.mark.parametrize("strategy", ["all", "sqrt", "log2", "onethird", "1", "1.0", "2", "0.5", "0.34"])
def test_every_subset_strategy(strategy):
    y, x = _data(1200, 7, 3, seed=4)
    _check(y, x, 3, 5, strategy, "gini", 4, 16, seed=11)


def test_entropy_forest():
    y, x = _data(3000, 4, 3, seed=8, decimals=2)
    y = np.trunc(y)
    args = (y, x, 3, 5, "sqrt", "entropy", 5, 32)
    _, info = fr.train(*args, seed=3, return_nodes=True)
    # every split of this fixture wins by more than the device's log could move it, and no best gain sits at 0
    for g, r in info["runner_up"]:
        assert abs(g) > 1e-9 and (g - r) > 1e-9 * abs(g), (g, r)
    _check(*args, seed=3)


def test_deterministic_and_independent_of_tree_groups(monkeypatch):
    y, x = _data(5000, 4, 4, seed=21)
    a = native.rf_train(y, x, 4, 12, "sqrt", native.RF_GINI, 6, 32, seed=5)
    b = native.rf_train(y, x, 4, 12, "sqrt", native.RF_GINI, 6, 32, seed=5)
    _assert_same(a, b)
    for per_pass in ("1", "5", "12"):
        monkeypatch.setenv("PIO_RF_TREES_PER_PASS", per_pass)
        _assert_same(native.rf_train(y, x, 4, 12, "sqrt", native.RF_GINI, 6, 32, seed=5), a)
    monkeypatch.delenv("PIO_RF_TREES_PER_PASS")
    big = native.rf_train(y, x, 4, 64, "sqrt", native.RF_GINI, 6, 32, seed=5)
    small = native.rf_train(y, x, 4, 8, "sqrt", native.RF_GINI, 6, 32, seed=5)
    cut = big["tree_off"][8]
    for k in INT_KEYS[1:] + F64_KEYS:
        np.testing.assert_array_equal(big[k][:cut], small[k], err_msg=k)
    np.testing.assert_array_equal(big["tree_off"][:9], small["tree_off"])


@pytest.mark.parametrize("kw,y,x", [
    (dict(numClasses=4), [0, 4], [[1.0], [2.0]]),
    (dict(numClasses=4, impurity="entropy"), [0, -1], [[1.0], [2.0]]),
    (dict(), [0, 1], [[1.0], [np.nan]]),
    (dict(), [np.inf, 1], [[1.0], [2.0]]),
    (dict(featureSubsetStrategy="half"), [0, 1], [[1.0], [2.0]]),
    (dict(featureSubsetStrategy="0"), [0, 1], [[1.0], [2.0]]),
    (dict(maxDepth=31), [0, 1], [[1.0], [2.0]]),
    (dict(maxBins=1), [0, 1], [[1.0], [2.0]]),
    (dict(numClasses=65), [0, 1], [[1.0], [2.0]]),
    (dict(numTrees=0), [0, 1], [[1.0], [2.0]]),
    (dict(impurity="variance"), [0, 1], [[1.0], [2.0]]),
    (dict(categoricalFeaturesInfo={0: 3}), [0, 1], [[1.0], [2.0]]),
])
def test_errors_raise_before_device_work(kw, y, x):
    args = dict(numClasses=2, categoricalFeaturesInfo={}, numTrees=3, featureSubsetStrategy="auto", impurity="gini",
                maxDepth=4, maxBins=32)
    args.update(kw)
    y, x = np.array(y, float), np.array(x, float)
    with pytest.raises(ValueError) as want:
        fr.train(y, x, args["numClasses"], args["numTrees"], args["featureSubsetStrategy"], args["impurity"],
                 args["maxDepth"], args["maxBins"], categorical=args["categoricalFeaturesInfo"])
    # device 4096 does not exist: only a check made before any device work can report the argument error
    with pytest.raises(ValueError) as got:
        mllib.RandomForest.trainClassifier(y, x, **args, device=4096)
    assert str(got.value) == str(want.value)


# ---- the classification template -----------------------------------------------------------------------------------
ENGINE_JSON = """{
  "id": "default",
  "description": "Default settings",
  "engineFactory": "org.apache.predictionio.examples.classification.ClassificationEngine",
  "datasource": {
    "params": {
      "appName": "MyApp1"
    }
  },
  "algorithms": [
    {
      "name": "randomforest",
      "params": {
        "numClasses": 4,
        "numTrees": 5,
        "featureSubsetStrategy": "auto",
        "impurity": "gini",
        "maxDepth": 4,
        "maxBins": 100
      }
    }
  ]
}
"""


def _import_users(app, n, seed):
    import datetime as dt
    rng = np.random.default_rng(seed)
    t0 = dt.datetime(2021, 1, 1, tzinfo=dt.timezone.utc).isoformat()
    rows = []
    for _ in range(n):
        a = rng.integers(0, 10, 3)
        p = int(min(3, (a[0] + a[1]) // 5)) if rng.uniform() < 0.9 else int(rng.integers(0, 4))
        rows.append((p, *[int(v) for v in a]))
    s.import_events(app, [dict(event="$set", entityType="user", entityId=f"u{k}", eventTime=t0,
                               properties={"plan": p, "attr0": a, "attr1": b, "attr2": c})
                          for k, (p, a, b, c) in enumerate(rows)])
    return rows


def test_classification_template_randomforest(tmp_path, monkeypatch):
    monkeypatch.setenv("PIO_EVENTDATA_DIR", str(tmp_path / "events"))
    monkeypatch.setenv("PIO_MODELDATA_DIR", str(tmp_path / "models"))
    _import_users("MyApp1", 800, seed=1)
    variant = tmp_path / "engine.json"
    variant.write_text(ENGINE_JSON)
    inst = w.CreateWorkflow.main(["--engine-id", "cls", "--engine-version", "1", "--engine-variant", f"file:{variant}",
                                  "--engine-factory", "pio_b200.templates.classification.ClassificationEngine"])
    assert inst.status == "COMPLETED"
    server = w.deploy(inst.id)
    model = server.models[0]
    assert isinstance(model, mllib.RandomForestModel)

    from pio_b200.templates import classification as cl
    td = cl.DataSource(cl.DataSourceParams(appName="MyApp1")).readTraining(w.WorkflowContext())
    assert td.features64.dtype == np.float64 and np.array_equal(td.features64.astype(np.float32), td.features)
    want = fr.train(td.labels, td.features64, 4, 5, "auto", "gini", 4, 100)
    _assert_same(model.nodes, want)
    again = pickle.loads(pickle.dumps(model))
    _assert_same(again.nodes, want)
    queries = [(float(a), float(b), float(c)) for a in range(0, 10, 3) for b in range(10) for c in (0, 5, 9)]
    got = [server.query({"attr0": a, "attr1": b, "attr2": c})["label"] for a, b, c in queries]
    assert got == list(fr.predict(want, np.array(queries)))


def test_classification_template_trains_both_algorithms(tmp_path, monkeypatch):
    monkeypatch.setenv("PIO_EVENTDATA_DIR", str(tmp_path / "events"))
    rows = _import_users("Both", 400, seed=2)
    from pio_b200.templates import classification as cl
    eng = cl.ClassificationEngine().apply()
    spec = json.loads(ENGINE_JSON)
    spec["datasource"]["params"]["appName"] = "Both"
    spec["algorithms"].insert(0, {"name": "naive", "params": {"lambda": 1.0}})
    ep = eng.jValueToEngineParams(spec)
    nb, rf = eng.train(w.WorkflowContext(), ep, "both")
    assert isinstance(nb, mllib.NaiveBayesModel) and isinstance(rf, mllib.RandomForestModel)
    algo = cl.RandomForestAlgorithm(ep.algorithmParamsList[1][1])
    q = cl.Query(*map(float, rows[0][1:]))
    assert algo.predict(rf, q).label == rf.predict(list(rows[0][1:]))
    assert cl.NaiveBayesAlgorithm(ep.algorithmParamsList[0][1]).predict(nb, q).label in (0.0, 1.0, 2.0, 3.0)
