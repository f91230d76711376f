#!/usr/bin/env python
"""The dimensionality-reduction classification template (DESIGN.md 4.19) on one GPU.

Corpus: seeded synthetic digits (tests/digits.py: 28 x 28 intensities 0-255 from per-class strokes, 10 labels),
written as an event file of digitData events.  Preparator numFeatures 250, "lr" regParam 1.
Timed, each a host clock around work that ends in a device synchronise:
  read      DataSource.readTraining (the event scan on the GPU plus the host columns);
  prepare   PreparedData: the device's parse (with its host-parsed rows), mean + Gramian (achieved fp64 FLOP/s from
            n p (p + 1)), the host SVD and the projection, from pio_fr_data_debug_stats and host clocks;
  train     LRAlgorithm.train: loss-and-gradient calls, iterations per label, device against host time;
  many      predictMany of --queries rows; single: the median of 200 single-query predict calls;
  eval      the doc's pio eval (evalK 3, numFeatures 250, regParam 0.5 / 2.5 / 7.5: 90 trainings) when --eval;
  host      the restatement (tests/featurereduction_ref: mean, transform) on --host-rows rows.
The card's name and power limit are read in the same run.

    python tools/featurereduction_bench.py [--rows 42000] [--queries 28000] [--eval] [--out DIR]
"""
import argparse
import json
import os
import subprocess
import sys
import tempfile
import time
from pathlib import Path

import numpy as np

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))
import pio_b200  # noqa: E402,F401
from pio_b200 import storage  # noqa: E402
from pio_b200 import workflow as w  # noqa: E402
from pio_b200.templates import featurereduction as fr  # noqa: E402
from tests import digits  # noqa: E402
from tests import featurereduction_ref as ref  # noqa: E402


def card():
    out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                         capture_output=True, text=True, timeout=30, check=True).stdout.strip().splitlines()
    if not out:
        raise RuntimeError("nvidia-smi reported no GPU")
    return out[0]


def write_events(path, x, y):
    with open(path, "w") as f:
        for i in range(x.shape[0]):
            f.write('{"event":"digitData","entityType":"digit","entityId":"%d","properties":{"label":%.1f,'
                    '"features":"%s"},"eventTime":"2020-01-01T00:00:00.000Z"}\n'
                    % (i, y[i], ", ".join(map(str, x[i].tolist()))))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rows", type=int, default=42000)
    ap.add_argument("--queries", type=int, default=28000)
    ap.add_argument("--host-rows", type=int, default=2000)
    ap.add_argument("--eval", action="store_true")
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    out_dir = Path(a.out).resolve() if a.out else None
    cwd = os.getcwd()
    res = {"card": card(), "rows": a.rows}
    with tempfile.TemporaryDirectory() as tmp:
        os.environ["PIO_EVENTDATA_DIR"] = tmp
        os.environ["PIO_MODELDATA_DIR"] = os.path.join(tmp, "models")
        x, y = digits.digits(a.rows, seed=7)
        path = storage.app_file("FeatureReduction", None)
        path.parent.mkdir(parents=True, exist_ok=True)
        write_events(path, x, y)
        res["event_file_bytes"] = path.stat().st_size
        sc = w.WorkflowContext()
        ds = fr.DataSource(fr.DataSourceParams(appName="FeatureReduction"))
        t0 = time.perf_counter()
        td = ds.readTraining(sc)
        res["read_s"] = time.perf_counter() - t0
        t0 = time.perf_counter()
        pd = fr.Preparator(fr.PreparatorParams(250)).prepare(sc, td)
        res["prepare_s"] = time.perf_counter() - t0
        st = pd.rows.stats()
        p = pd.rows.p
        res["prepare"] = {k: st[k] for k in ("parts", "host_rows", "parse_ms", "gram_ms", "project_ms", "slices")}
        res["prepare"]["gram_tflops"] = a.rows * p * (p + 1) / (st["gram_ms"] * 1e-3) / 1e12
        res["prepare"]["host_svd_s"] = pd.svd_s
        t0 = time.perf_counter()
        model = fr.LRAlgorithm(fr.LRAlgorithmParams(1.0)).train(sc, pd)
        train_s = time.perf_counter() - t0
        ms = model.stats
        res["train"] = {"wall_s": train_s, "lr_evals": ms["lr_evals"], "iterations": ms["iterations"],
                        "evaluations": ms["evaluations"], "device_s": (ms["lr_ms"] + ms["sigma_ms"]) * 1e-3,
                        "host_s": train_s - (ms["lr_ms"] + ms["sigma_ms"]) * 1e-3}
        algo = fr.LRAlgorithm(fr.LRAlgorithmParams(1.0))
        qs = [fr.Query(digits.feature_string(r)) for r in x[:a.queries]]
        algo.predictMany(model, qs[:10])
        t0 = time.perf_counter()
        pred = algo.predictMany(model, qs)
        res["many_s"] = time.perf_counter() - t0
        res["many_device_ms"] = model.handle().stats()["device_ms"]
        res["train_accuracy_on_queries"] = float(np.mean([q.label == lab for q, lab in zip(pred, y[:a.queries])]))
        lat = []
        for q in qs[:200]:
            t0 = time.perf_counter()
            algo.predict(model, q)
            lat.append(time.perf_counter() - t0)
        res["single_median_ms"] = float(np.median(lat) * 1e3)
        X = x[:a.host_rows].astype(np.float64)
        t0 = time.perf_counter()
        mu = ref.mean(X)
        ref.transform(X, mu, model.pc)
        res["host_restatement_s"] = {"rows": a.host_rows, "mean_transform_s": time.perf_counter() - t0}
        if a.eval:
            from pio_b200 import evaluation as ev  # noqa: F401
            t0 = time.perf_counter()
            os.chdir(tmp)
            variant = Path(tmp) / "engine.json"
            variant.write_text(json.dumps({
                "engineFactory": "pio_b200.templates.featurereduction.ClassificationEngine",
                "datasource": {"params": {"appName": "FeatureReduction"}},
                "preparator": {"params": {"numFeatures": 250}},
                "algorithms": [{"name": "lr", "params": {"regParam": 1.0}}]}))
            r = w.CreateWorkflow.main([
                "--engine-id", "fr", "--engine-version", "1", "--engine-variant", str(variant),
                "--evaluation-class", "pio_b200.templates.featurereduction.AccuracyEvaluation",
                "--engine-params-generator-class", "pio_b200.templates.featurereduction.EngineParamsList"])
            res["eval"] = {"wall_s": time.perf_counter() - t0, "best_score": r.bestScore.score,
                           "best_regParam": r.bestEngineParams.algorithmParamsList[0][1].regParam}
            os.chdir(cwd)
    print(json.dumps(res, indent=1))
    if out_dir:
        out_dir.mkdir(parents=True, exist_ok=True)
        (out_dir / f"featurereduction_bench_{a.rows}.json").write_text(json.dumps(res, indent=1))


if __name__ == "__main__":
    main()
