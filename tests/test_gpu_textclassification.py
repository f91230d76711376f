"""GPU tests (-m gpu) of the text featurizer and Naive Bayes (native.TextModel, pio_text_*) and of the text
classification template (templates/textclassification.py).

The device equals the restatement tests/textclassification_ref.py byte for byte: the TF and TF-IDF COO, df, idf, pi,
theta, the raw scores, the categories and the confidences.  The fixtures are seeded and built here: texts with empty
and blank documents, leading, trailing and doubled spaces, \\n and \\t inside tokens, multibyte UTF-8, \\u escapes,
surrogate pairs and lone surrogates, terms of every byte length mod 4, and stop words that cover whole documents."""
import json
import math
import pickle

import numpy as np
import pytest

from pio_b200 import evaluation as ev
from pio_b200 import native
from pio_b200 import storage as s
from pio_b200 import workflow as w
from pio_b200.templates import textclassification as tc
from tests import textclassification_ref as ref

pytestmark = pytest.mark.gpu

VOCAB = ["a", "ab", "abc", "abcd", "abcde", "spam", "free", "win", "now", "the", "é", "日本", "😀", "x\ny", "t\tab",
         "\ud800", "z\udc00z", "money", "hello", "naïve", "\\", '"q"', "/"]
CORNERS = ["", "   ", " ", " lead", "trail ", "double  space", "a\nb\tc", "é 日本 😀", "lone \ud800 sur",
           "pair 😀 here", "the the the", "the", "x" * 41, "a b c d e f g h"]


def corpus(seed, n, max_words=14):
    rng = np.random.default_rng(seed)
    out = list(CORNERS)
    while len(out) < n:
        k = int(rng.integers(0, max_words))
        words = [VOCAB[int(rng.integers(0, len(VOCAB)))] for _ in range(k)]
        seps = [" " if rng.random() < 0.85 else "  " for _ in range(k)]
        t = "".join(wd + sp for wd, sp in zip(words, seps))
        if rng.random() < 0.5:
            t = t.rstrip(" ")
        out.append(t)
    return out[:n]


def same(a, b):
    """Equal bytes, or both NaN."""
    a, b = np.asarray(a, np.float64), np.asarray(b, np.float64)
    if a.shape != b.shape:
        return False
    nan = np.isnan(a) & np.isnan(b)
    return bool(np.all(nan | (a.view(np.uint64) == b.view(np.uint64))))


def decoded(tb, to):
    return [ref.decode_token(bytes(tb[to[i]:to[i + 1]])) for i in range(to.shape[0] - 1)]


def check(texts, labels, C, n_gram, D, lam, stop, queries=None):
    tm = native.TextModel(stop, n_gram, D)
    tb, to = native.text_tokens(texts)
    dec = decoded(tb, to)
    sb = [w_.encode("utf-8", "replace") for w_ in stop]
    labels = np.asarray(labels, np.int32)
    df, idf, pi, theta = tm.train_nb(tb, to, labels, C, lam)
    rdf, ridf, rpi, rtheta, (rp, rj, rx) = ref.train(dec, labels, C, n_gram, D, lam, sb)
    assert np.array_equal(df, rdf) and same(idf, ridf) and same(pi, rpi) and same(theta, rtheta)
    p, j, v = tm.features(tb, to, use_idf=False)
    tp, tj, tv = ref.features(dec, n_gram, D, sb)
    assert np.array_equal(p, tp) and np.array_equal(j, tj) and same(v, tv)
    tm.set_model(idf, pi, theta)
    p, j, v = tm.features(tb, to, use_idf=True)
    assert np.array_equal(p, rp) and np.array_equal(j, rj) and same(v, rx)
    qs = texts if queries is None else queries
    qb, qo = native.text_tokens(qs)
    raw = tm.scores(qb, qo)
    want = ref.scores(*ref.features(decoded(qb, qo), n_gram, D, sb, idf), pi, theta)
    assert same(raw, want)
    best, conf = tc.confidences(raw)
    rbest, rconf, _ = ref.confidences(want)
    assert np.array_equal(best, rbest) and same(conf, rconf)
    tm.close()
    return raw, theta


@pytest.mark.parametrize("n_gram,D,C,lam", [(1, 7, 2, 1.0), (2, 500, 20, 0.5), (3, 1 << 20, 2, 1.0), (1, 1, 1, 1.0),
                                            (2, 500, 2, 0.0), (3, 500, 3, 2.5), (5, 97, 2, 1.0)])
def test_device_equals_restatement(n_gram, D, C, lam):
    texts = corpus(10 + n_gram + C, 300)
    labels = np.random.default_rng(D).integers(0, C, len(texts))
    labels[:C] = np.arange(C)
    raw, theta = check(texts, labels, C, n_gram, D, lam, ["the", "now", "\ud800"], queries=corpus(77, 60))
    if lam == 0.0:
        assert np.isinf(theta).any() and np.isnan(raw).any()    # the dense fold's 0 * -inf


def test_stop_words_cover_documents_and_empty_token():
    texts = ["the", "the  the", "", "  ", "a the b", " x", "x  y"]
    check(texts, [0, 1, 0, 1, 0, 1, 0], 2, 2, 64, 1.0, ["the", ""])


def test_every_term_length_mod_4():
    texts = [" ".join("q" * k for k in range(1, 13)), "é" * 7 + " " + "日本" * 3, "😀 😀😀 😀😀😀"]
    for n_gram in (1, 2, 3):
        check(texts, [0, 1, 1], 2, n_gram, 1 << 18, 1.0, [])


def test_df_equal_m_gives_idf_zero():
    texts = ["w a", "w b", "w c", "w"]
    tm = native.TextModel([], 1, 50)
    tb, to = native.text_tokens(texts)
    df, idf, pi, theta = tm.train_nb(tb, to, [0, 1, 0, 1], 2, 1.0)
    j = ref.features([b"w"], 1, 50)[1][0]
    assert df[j] == 4 and idf[j] == 0.0
    p, jj, v = tm.features(tb, to, use_idf=False)
    tm.set_model(idf, pi, theta)
    p2, jj2, v2 = tm.features(tb, to, use_idf=True)
    assert np.array_equal(jj, jj2) and (v2[jj2 == j] == 0.0).all()   # entries with idf 0 stay
    tm.close()
    check(texts, [0, 1, 0, 1], 2, 1, 50, 1.0, [])


def test_underflow_gives_nan_and_the_first_label():
    rng = np.random.default_rng(1)
    words = [f"w{k}" for k in range(3000)]
    texts = [" ".join(rng.choice(words, 400)) for _ in range(40)]
    long_q = [" ".join(rng.choice(words, 3000))]
    raw, _ = check(texts, np.arange(40) % 3, 3, 1, 4096, 1.0, [], queries=long_q)
    best, conf = tc.confidences(raw)
    assert (raw < -800).all() and best[0] == 0 and math.isnan(conf[0])


def test_exact_confidence_tie_keeps_the_first_class():
    raw, _ = check(["p q", "p q", "r"], [0, 1, 2], 3, 1, 32, 1.0, [], queries=["p q"])
    best, conf = tc.confidences(raw)
    assert raw[0, 0] == raw[0, 1] and best[0] == 0


@pytest.mark.parametrize("budget,parts", [(1 << 26, 1), (None, 2), (None, 3)])
def test_budgets_give_the_same_bytes(monkeypatch, budget, parts):
    texts = corpus(5, 90)
    tb, to = native.text_tokens(texts)
    total = int(to[-1])
    b = budget or (total + parts - 1) // parts
    labels = np.arange(90) % 4
    monkeypatch.delenv("PIO_TEXT_BUDGET", raising=False)
    base = check(texts, labels, 4, 2, 1000, 0.5, ["the"])
    monkeypatch.setenv("PIO_TEXT_BUDGET", str(b))
    tm = native.TextModel(["the"], 2, 1000)
    df, idf, pi, theta = tm.train_nb(tb, to, labels, 4, 0.5)
    assert native.text_stats()["parts"] >= parts
    tm.set_model(idf, pi, theta)
    assert same(tm.scores(tb, to), base[0])
    tm.close()
    check(texts, labels, 4, 2, 1000, 0.5, ["the"])


def test_document_larger_than_the_budget(monkeypatch):
    texts = ["tiny", " ".join(["long"] * 500) + " end", "small one"]
    monkeypatch.setenv("PIO_TEXT_BUDGET", "64")
    check(texts, [0, 1, 0], 2, 2, 300, 1.0, [])
    assert native.text_stats()["parts"] == 3


def test_rejections():
    for args in ((["x"], 0, 10), (["x"], 1, 0)):
        with pytest.raises(native.NativeError) as e:
            native.TextModel(*args)
        assert e.value.code == native.ERR_ARG
    tm = native.TextModel([], 1, 10)
    tb, to = native.text_tokens(["a", "b"])
    for lam in (-1.0, float("nan")):
        with pytest.raises(native.NativeError) as e:
            tm.train_nb(tb, to, [0, 0], 1, lam)
        assert e.value.code == native.ERR_ARG
    with pytest.raises(native.NativeError) as e:
        tm.train_nb(tb, np.array([0, 3, 2]), [0, 0], 1, 1.0)
    assert e.value.code == native.ERR_ARG
    bad = np.frombuffer(b'"a"5', np.uint8)
    with pytest.raises(native.NativeError) as e:
        tm.features(bad, np.array([0, 3, 4]), use_idf=False)
    assert e.value.code == native.ERR_ARG
    with pytest.raises(native.NativeError) as e:
        tm.scores(tb, to)
    assert e.value.code == native.ERR_STATE
    tm.close()


# ---- the template end to end -------------------------------------------------------------------------------------------
def _events(n, seed):
    rng = np.random.default_rng(seed)
    texts = corpus(seed, n)
    evs = [dict(event="e-mail", entityType="content", entityId=str(i),
                properties={"text": t, "label": "spam" if rng.random() < 0.4 else "ham"}) for i, t in enumerate(texts)]
    evs += [dict(event="stopwords", entityType="resource", entityId=f"s{k}", properties={"word": wd})
            for k, wd in enumerate(["the", "now", "a"])]
    return evs


def _restated(evs, n_gram, D, lam, queries):
    mails = [e for e in evs if e["event"] == "e-mail"]
    stop = [e["properties"]["word"].encode("utf-8", "replace") for e in evs if e["event"] == "stopwords"]
    labels = np.array([1.0 if e["properties"]["label"] == "spam" else 0.0 for e in mails])
    classes = np.unique(labels)
    dec = [ref.decode_token(json.dumps(e["properties"]["text"]).encode()) for e in mails]
    _, idf, pi, theta, _ = ref.train(dec, np.searchsorted(classes, labels), classes.shape[0], n_gram, D, lam, stop)
    qdec = [ref.decode_token(json.dumps(q).encode()) for q in queries]
    raw = ref.scores(*ref.features(qdec, n_gram, D, stop, idf), pi, theta)
    best, conf, _ = ref.confidences(raw)
    cm = {}
    for e, y in zip(mails, labels.tolist()):
        cm[y] = e["properties"]["label"]
    return [(cm[float(classes[b])], c) for b, c in zip(best.tolist(), conf.tolist())]


def test_template_end_to_end(tmp_path, monkeypatch):
    monkeypatch.setenv("PIO_EVENTDATA_DIR", str(tmp_path / "events"))
    monkeypatch.setenv("PIO_MODELDATA_DIR", str(tmp_path / "models"))
    evs = _events(200, 3)
    s.import_events("MyTextApp", evs)
    variant = tmp_path / "engine.json"
    variant.write_text(json.dumps({
        "id": "default", "description": "Default settings",
        "engineFactory": "pio_b200.templates.textclassification.TextClassificationEngine",
        "datasource": {"params": {"appName": "MyTextApp"}},
        "preparator": {"params": {"nGram": 2, "numFeatures": 500}},
        "algorithms": [{"name": "nb", "params": {"lambda": 0.25}}]}))
    inst = w.CreateWorkflow.main(["--engine-id", "tc", "--engine-version", "1", "--engine-variant", f"file:{variant}"])
    assert inst.status == "COMPLETED"
    server = w.deploy(inst.id)
    model = server.models[0]
    queries = corpus(41, 30) + ["free money now", ""]
    want = _restated(evs, 2, 500, 0.25, queries)
    got = [server.query({"text": q}) for q in queries]
    for g, (cat, conf) in zip(got, want):
        assert g["category"] == cat and (g["confidence"] == conf or (math.isnan(conf) and math.isnan(g["confidence"])))
    algo = server.algorithms[0]
    qs = [tc.Query(q) for q in queries]
    many = algo.predictMany(model, qs)
    assert [(p.category, p.confidence) for p in many] == [(p.category, p.confidence) for p in
                                                          (algo.predict(model, q) for q in qs)]
    again = pickle.loads(pickle.dumps(model))
    assert "_handle" not in again.__dict__
    assert [(p.category, p.confidence) for p in algo.predictMany(again, qs)] == \
        [(p.category, p.confidence) for p in many]
    (tmp_path / "in.json").write_text("\n".join(json.dumps({"text": q}) for q in queries) + "\n")
    out = tmp_path / "out.json"
    assert w.BatchPredict.main(["--input", str(tmp_path / "in.json"), "--output", str(out),
                                "--engine-instance-id", inst.id]) == len(queries)
    lines = out.read_text().splitlines()
    assert lines == [json.dumps({"query": {"text": q}, "prediction": w.to_json(algo.predict(model, tc.Query(q)))},
                                separators=(",", ":")) for q in queries]


def test_lr_and_sppmi_are_rejected(tmp_path, monkeypatch):
    monkeypatch.setenv("PIO_EVENTDATA_DIR", str(tmp_path / "events"))
    monkeypatch.setenv("PIO_MODELDATA_DIR", str(tmp_path / "models"))
    s.import_events("MyTextApp", _events(20, 4))
    for prep, algo, what in (({"nGram": 2}, {"name": "lr", "params": {"regParam": 0.1}}, "not supported"),
                             ({"nGram": 2, "SPPMI": True}, {"name": "nb", "params": {"lambda": 1.0}}, "SPPMI")):
        variant = tmp_path / "engine.json"
        variant.write_text(json.dumps({
            "engineFactory": "pio_b200.templates.textclassification.TextClassificationEngine",
            "datasource": {"params": {"appName": "MyTextApp"}}, "preparator": {"params": prep}, "algorithms": [algo]}))
        with pytest.raises(Exception) as e:
            w.CreateWorkflow.main(["--engine-id", "tc", "--engine-version", "1", "--engine-variant", str(variant)])
        assert what in str(e.value)


def test_missing_text_names_the_event(tmp_path, monkeypatch):
    monkeypatch.setenv("PIO_EVENTDATA_DIR", str(tmp_path / "events"))
    evs = _events(5, 6)
    evs.insert(2, dict(event="e-mail", entityType="content", entityId="x", properties={"label": "spam", "text": 5}))
    s.import_events("MyTextApp", evs)
    with pytest.raises(ValueError, match="line 3"):
        tc.DataSource(tc.DataSourceParams(appName="MyTextApp")).readTraining(w.WorkflowContext())


def test_evaluation_writes_best_json(tmp_path, monkeypatch):
    monkeypatch.setenv("PIO_EVENTDATA_DIR", str(tmp_path / "events"))
    monkeypatch.setenv("PIO_MODELDATA_DIR", str(tmp_path / "models"))
    monkeypatch.chdir(tmp_path)
    s.import_events("MyTextApp", _events(150, 8))
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
    best = json.loads((tmp_path / "best.json").read_text())
    assert best["algorithms"][0]["params"]["lambda"] == res.bestEngineParams.algorithmParamsList[0][1].lambda_
    assert 0.0 <= res.bestScore.score <= 1.0
