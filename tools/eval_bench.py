"""`pio eval` measurement: the recommendation template's RecommendationEvaluation x EngineParamsList (3 ranks x 3
iteration counts x kFold 5 = 45 trainings) on a seeded JSON-lines event file, columnar path versus object path.

    python tools/eval_bench.py [--events N] [--object-events M] [--dir DIR]

The file is written by tools/events_bench.write_file (fixed-width lines, zipf users and items, 30 % buy events) into a
temporary directory and removed afterwards.  The columnar path (run_evaluation -> Engine.evalColumns) runs on all N
events and is split into phases by timing the calls that make it up, each of which returns after a device synchronise:
event scan + ids_encode, the per-fold split (native.EvalFolds), ingest (EvalFolds.set_ratings), ALS (NativeALS.run),
top-N (NativeALS.recommend), rank counts (EvalResult.rank_counts); the rest of the wall time (string maps, host means,
Python) is reported as host_rest.  The object path (Engine.eval + MetricEvaluator.evaluateBase, per-rating objects) runs
on the first M events and is extrapolated to N, and labelled so.  Both paths also run on the M-event file, where their
scores must be identical.  Prints one JSON object, with the card name and power limit read in the same run."""
import argparse
import json
import os
import sys
import tempfile
import time
from pathlib import Path

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))
sys.path.insert(0, str(ROOT / "tools"))
import pio_b200  # noqa: E402,F401
from pio_b200 import evaluation as ev, native, storage as s, workflow as w  # noqa: E402
from pio_b200.templates import recommendation as rec  # noqa: E402
from events_bench import machine, write_file  # noqa: E402

PHASES = (("scan_encode", s.PEventStore, "findColumns", True), ("scan_encode", native, "ids_encode", False),
          ("split", native.EvalFolds, "__init__", False), ("ingest", native.EvalFolds, "set_ratings", False),
          ("als", native.NativeALS, "run", False), ("top_n", native.NativeALS, "recommend", False),
          ("rank_counts", native.EvalResult, "rank_counts", False))


def timed_phases():
    """Wraps the calls of PHASES with wall clocks; returns (totals by phase, undo)."""
    tot = {p: 0.0 for p, *_ in PHASES}
    saved = []
    for phase, owner, name, static in PHASES:
        orig = owner.__dict__[name]
        fn = orig.__func__ if static else orig

        def wrap(*a, _fn=fn, _phase=phase, **kw):
            t = time.perf_counter()
            try:
                return _fn(*a, **kw)
            finally:
                tot[_phase] += time.perf_counter() - t
        setattr(owner, name, staticmethod(wrap) if static else wrap)
        saved.append((owner, name, orig))

    def undo():
        for owner, name, orig in reversed(saved):
            setattr(owner, name, orig)
    return tot, undo


def columnar(app, sc):
    evaluation, gen = rec.RecommendationEvaluation(), rec.EngineParamsList(appName=app)
    tot, undo = timed_phases()
    t = time.perf_counter()
    try:
        res = ev.run_evaluation(evaluation, gen, sc)
    finally:
        undo()
    wall = time.perf_counter() - t
    out = {k + "_s": v for k, v in tot.items()}
    out["host_rest_s"] = wall - sum(tot.values())
    out["total_s"] = wall
    return res, out


def object_path(app, sc):
    evaluation, gen = rec.RecommendationEvaluation(), rec.EngineParamsList(appName=app)
    t = time.perf_counter()
    res = evaluation.evaluator.evaluateBase(sc, [(ep, evaluation.engine.eval(sc, ep)) for ep in gen.engineParamsList])
    return res, time.perf_counter() - t


def scores(res):
    return [[x.score, *x.otherScores] for _, x in res.engineParamsScores]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--events", type=int, default=20_000_000)
    ap.add_argument("--object-events", type=int, default=200_000)
    ap.add_argument("--dir", default=None)
    a = ap.parse_args()
    out = {"machine": machine(), "events": a.events, "object_events": a.object_events, "trainings": 45}
    sc = w.WorkflowContext(mode="Evaluation")
    with tempfile.TemporaryDirectory(dir=a.dir) as d:
        os.environ["PIO_EVENTDATA_DIR"] = d
        write_file(s.app_file("Big"), a.events, 1)
        write_file(s.app_file("Small"), a.object_events, 1)
        # equal scores on the small file; this also warms the library and the allocator up
        small_cols, small_split = columnar("Small", sc)
        small_obj, t_obj = object_path("Small", sc)
        out["scores_identical"] = scores(small_cols) == scores(small_obj) and small_cols.bestIdx == small_obj.bestIdx
        out["small_file"] = {"columnar": small_split, "object_s": t_obj, "best_idx": small_cols.bestIdx,
                             "best_score": small_cols.bestScore.score}
        res, split = columnar("Big", sc)
        out["columnar"] = split
        out["columnar"]["best_idx"] = res.bestIdx
        out["object"] = {"events_measured": a.object_events, "measured_s": t_obj,
                         "extrapolated_s_for_events": t_obj / a.object_events * a.events, "label": "extrapolated"}
        out["speedup_vs_object_extrapolated"] = out["object"]["extrapolated_s_for_events"] / split["total_s"]
    print(json.dumps(out))


if __name__ == "__main__":
    main()
