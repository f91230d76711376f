#!/usr/bin/env python
"""The text classification template's evaluation on one GPU (DESIGN.md 4.18.1).

Corpus: tools/textclassification_bench.py's seeded e-mails (category 0 is "spam", so both labels occur) and its 500
stop words, --docs documents, written as an event file.  Generator: the doc's EngineParamsList (nGram 1, numFeatures
5000, "nb" with lambda 0.5 / 1.5 / 5, evalK 5) under AccuracyEvaluation.

The columnar evaluation is run phase by phase, as Engine.evalColumns runs it, each phase a host clock around work that
ends in a device synchronise:
  read        DataSource._read (the event scan and its host columns)
  create      native.TextFolds over the read's tokens (a host copy of them)
  featurize   one featurization of every document on the device
  train       the 15 fold trainings (Preparator.prepare + NBAlgorithm.train), device and host milliseconds apart
  scores      the 15 fold scorings on the device (TextFolds.scores)
  host_rest   confidences, categories, serveColumns and Accuracy.calculate_columns
and then once more end to end through evaluation.run_evaluation, whose scores must equal the phased run's.  The object
path (Engine.eval + evaluateBase) runs on the first --object-docs documents, where its scores and bestIdx are asserted
equal to the columnar path's.  The card's name and power limit are read in the same run.

    python tools/text_eval_bench.py [--docs 1000000] [--object-docs 3000] [--out DIR]
"""
import argparse
import json
import os
import sys
import tempfile
import time
from pathlib import Path

import numpy as np

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))
sys.path.insert(0, str(ROOT / "tools"))
import pio_b200  # noqa: E402,F401
from pio_b200 import evaluation as ev  # noqa: E402
from pio_b200 import native  # noqa: E402
from pio_b200 import workflow as w  # noqa: E402
from pio_b200 import storage  # noqa: E402
from pio_b200.templates import textclassification as tc  # noqa: E402
import textclassification_bench as tcb  # noqa: E402


def phased(sc, app):
    """The columnar evaluation of EngineParamsList on `app`, phase by phase, with readEvalColumns' steps taken one at a
    time: (timings, scores per parameter set)."""
    gen = tc.EngineParamsList(appName=app)
    ep0 = gen.engineParamsList[0]
    k = ep0.dataSourceParams[1].evalK
    t = {}
    t0 = time.perf_counter()
    td = tc.DataSource(ep0.dataSourceParams[1])._read(sc)
    t["read_s"] = time.perf_counter() - t0
    t0 = time.perf_counter()
    folds = native.TextFolds(*td.tokens, sorted(td.stopWords), k, getattr(sc, "device", 0) or 0)
    t["create_s"] = time.perf_counter() - t0
    folds_cols = []
    for f in range(k):
        fold = tc.TextFold(folds, f, td)
        folds_cols.append((tc.TrainingData(stopWords=td.stopWords, fold=fold), None, fold))
    pp = ep0.preparatorParams[1]
    t0 = time.perf_counter()
    folds.featurize(pp.nGram, pp.numFeatures)
    t["featurize_s"] = time.perf_counter() - t0
    st0 = folds.stats()
    t["featurize_device_s"] = st0["featurize_ms"] / 1e3
    t["entries"] = st0["entries"]
    t["parts"] = st0["parts"]
    t0 = time.perf_counter()
    models = []
    for ep in gen.engineParamsList:
        algo = tc.NBAlgorithm(ep.algorithmParamsList[0][1])
        models.append([algo.train(sc, tc.Preparator(pp).prepare(sc, tdf)) for tdf, _, _ in folds_cols])
    t["train_s"] = time.perf_counter() - t0
    st1 = folds.stats()
    t["train_device_s"] = (st1["train_ms"] - st0["train_ms"]) / 1e3
    t["train_host_s"] = t["train_s"] - t["train_device_s"]
    t0 = time.perf_counter()
    raws = [[folds.scores(q.fold, m.idf, m.pi, m.theta) for m, (_, _, q) in zip(ms, folds_cols)] for ms in models]
    t["scores_s"] = time.perf_counter() - t0
    t["scores_device_s"] = (folds.stats()["scores_ms"] - st1["scores_ms"]) / 1e3
    t0 = time.perf_counter()
    scores = []
    for ms, rs in zip(models, raws):
        served = []
        for m, r, (_, _, q) in zip(ms, rs, folds_cols):
            best, conf = tc.confidences(r)
            cats = np.array([m.categoryMap.get(y, "") for y in m.labels.tolist()], dtype=object)
            served.append((None, q, tc.Serving().serveColumns(q, [tc.PredictedColumns(cats[best], conf)])))
        scores.append(tc.Accuracy().calculate_columns(sc, served))
    t["host_rest_s"] = time.perf_counter() - t0
    t["post_read_s"] = t["create_s"] + t["featurize_s"] + t["train_s"] + t["scores_s"] + t["host_rest_s"]
    t["docs"] = len(td)
    folds.close()
    return t, scores


def _same(a, b):
    return all((x != x and y != y) or x == y for x, y in zip(a, b)) and len(a) == len(b)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--docs", type=int, default=1_000_000)
    ap.add_argument("--object-docs", type=int, default=3000)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    res = {"card": tcb.card(), "docs": a.docs, "object_docs": a.object_docs}
    rng = np.random.default_rng(7)
    out = Path(a.out).resolve() if a.out else None
    cwd = os.getcwd()
    with tempfile.TemporaryDirectory() as tmp:
        os.environ["PIO_EVENTDATA_DIR"] = tmp
        os.chdir(tmp)                                          # AccuracyEvaluation writes best.json here
        path = storage.app_file("MyTextApp", None)
        path.parent.mkdir(parents=True, exist_ok=True)
        t0 = time.perf_counter()
        tcb.write_events(path, rng, a.docs)
        res["event_file_bytes"] = path.stat().st_size
        res["write_s"] = time.perf_counter() - t0
        small = storage.app_file("SmallTextApp", None)
        with open(path, "rb") as src, open(small, "wb") as dst:
            lines = src.read().split(b"\n")
            dst.write(b"\n".join(lines[:a.object_docs] + lines[a.docs:]))
        sc = w.WorkflowContext(mode="Evaluation")
        # the object path on the prefix, against the columnar path there (which also warms every shape up)
        gen = tc.EngineParamsList(appName="SmallTextApp")
        E = tc.AccuracyEvaluation
        t0 = time.perf_counter()
        col = ev.run_evaluation(E, gen, sc)
        res["prefix_columnar_s"] = time.perf_counter() - t0
        t0 = time.perf_counter()
        obj = E.evaluator.evaluateBase(sc, [(ep, E.engine.eval(sc, ep)) for ep in gen.engineParamsList])
        res["prefix_object_s"] = time.perf_counter() - t0
        assert col.bestIdx == obj.bestIdx
        assert _same([s.score for _, s in col.engineParamsScores], [s.score for _, s in obj.engineParamsScores])
        res["prefix_scores"] = [s.score for _, s in col.engineParamsScores]
        res["prefix_equal"] = True
        # the full corpus, phase by phase, then end to end
        t, scores = phased(sc, "MyTextApp")
        res["phased"] = t
        t0 = time.perf_counter()
        full = ev.run_evaluation(E, tc.EngineParamsList(appName="MyTextApp"), sc)
        res["run_evaluation_s"] = time.perf_counter() - t0
        assert _same([s.score for _, s in full.engineParamsScores], scores)
        res["scores"] = scores
        res["bestIdx"] = full.bestIdx
        os.chdir(cwd)
    print(json.dumps(res, indent=1))
    if out:
        out.mkdir(parents=True, exist_ok=True)
        (out / "text_eval_bench.json").write_text(json.dumps(res, indent=1))


if __name__ == "__main__":
    main()
