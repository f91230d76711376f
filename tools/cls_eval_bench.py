"""`pio eval` measurement for the classification template: EngineParamsList (NaiveBayes, lambda in 10 / 100 / 1000) and
RandomForestParamsList (maxDepth 4 / 6 / 8), evalK 5, on a seeded `$set` event file of N users with plan / attr0-2
(C5 shape: 4 classes, 3 features), columnar path versus object path.

    python tools/cls_eval_bench.py [--users N] [--object-users M] [--dir DIR]

The file is generated vectorised (fixed-width lines) into a temporary directory and removed afterwards.  The columnar
path (run_evaluation -> Engine.evalColumns) runs on all N users and is split into phases by timing the calls that make
it up, each of which returns after a device synchronise: read (event scan and property fold), fold create
(native.ClsFolds), training (ClsFolds.nb_train / rf_train), predict (ClsFolds.nb_predict / rf_predict) and counts
(ClsResult.counts); the rest of the wall time is host_rest.  The object path (Engine.eval + MetricEvaluator.evaluateBase,
one device call per test row) runs on the first M users and is extrapolated to N, and labelled so.  Both paths also run
on the M-user file, where their scores and bestIdx must be identical.  Prints one JSON object, with the card name and
power limit read in the same run."""
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
from pio_b200 import evaluation as ev, native, storage as s, workflow as w  # noqa: E402
from pio_b200.templates import classification as cl  # noqa: E402
from events_bench import machine  # noqa: E402

W_ID = 9
PHASES = (("read", s.PEventStore, "aggregatePropertyColumns", True), ("fold_create", native.ClsFolds, "__init__", False),
          ("training", native.ClsFolds, "nb_train", False), ("training", native.ClsFolds, "rf_train", False),
          ("predict", native.ClsFolds, "nb_predict", False), ("predict", native.ClsFolds, "rf_predict", False),
          ("counts", native.ClsResult, "counts", False))


def write_users(path: Path, n: int, seed: int, block: int = 1 << 20):
    """n `$set` events, user k: attr0-2 digits 0-9, plan = min(3, (attr0 + attr1) // 5) with 10 % noise; returns the
    line length."""
    tl = (b'{"event": "$set", "entityType": "user", "entityId": "u' + b"0" * W_ID + b'", "properties": {"plan": 0, '
          b'"attr0": 0, "attr1": 0, "attr2": 0}, "eventTime": "2021-03-04T05:06:07.000000+00:00"}\n')
    row = np.frombuffer(tl, np.uint8)
    p_u = tl.index(b'"u0') + 2
    pos = [tl.index(k) + len(k) for k in (b'"plan": ', b'"attr0": ', b'"attr1": ', b'"attr2": ')]
    rng = np.random.default_rng(seed)
    with open(path, "wb") as fh:
        for b0 in range(0, n, block):
            m = min(block, n - b0)
            a = np.tile(row, (m, 1))
            uid = np.arange(b0, b0 + m)
            for k in range(W_ID):
                a[:, p_u + k] = 48 + (uid // 10 ** (W_ID - 1 - k)) % 10
            x = rng.integers(0, 10, (m, 3))
            plan = np.minimum(3, (x[:, 0] + x[:, 1]) // 5)
            noise = rng.random(m) < 0.1
            plan[noise] = rng.integers(0, 4, int(noise.sum()))
            for p, v in zip(pos, (plan, x[:, 0], x[:, 1], x[:, 2])):
                a[:, p] = 48 + v
            fh.write(a.tobytes())
    return len(tl)


def timed_phases():
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


GENERATORS = (("naive", cl.EngineParamsList), ("randomforest", cl.RandomForestParamsList))


def columnar(app, sc):
    out, results = {}, {}
    for name, G in GENERATORS:
        tot, undo = timed_phases()
        t = time.perf_counter()
        try:
            res = ev.run_evaluation(cl.CompleteEvaluation(), G(appName=app), sc)
        finally:
            undo()
        wall = time.perf_counter() - t
        d = {k + "_s": v for k, v in tot.items()}
        d["host_rest_s"] = wall - sum(tot.values())
        d["total_s"] = wall
        d["best_idx"] = res.bestIdx
        out[name], results[name] = d, res
    return results, out


def object_path(app, sc):
    out, results = {}, {}
    evaluation = cl.CompleteEvaluation()
    for name, G in GENERATORS:
        t = time.perf_counter()
        res = evaluation.evaluator.evaluateBase(sc, [(ep, evaluation.engine.eval(sc, ep))
                                                     for ep in G(appName=app).engineParamsList])
        out[name], results[name] = time.perf_counter() - t, res
    return results, out


def scores(res):
    return [[x.score, *x.otherScores] for _, x in res.engineParamsScores]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--users", type=int, default=10_000_000)
    ap.add_argument("--object-users", type=int, default=20_000)
    ap.add_argument("--dir", default=None)
    a = ap.parse_args()
    out = {"machine": machine(), "users": a.users, "object_users": a.object_users, "eval_k": 5,
           "trainings": {"naive": 15, "randomforest": 15}}
    sc = w.WorkflowContext(mode="Evaluation")
    with tempfile.TemporaryDirectory(dir=a.dir) as d:
        os.environ["PIO_EVENTDATA_DIR"] = d
        cwd = os.getcwd()
        os.chdir(d)            # CompleteEvaluation writes best.json into the working directory
        try:
            line = write_users(s.app_file("Big"), a.users, 1)
            with open(s.app_file("Big"), "rb") as src:     # the first M users of the big file
                s.app_file("Small").write_bytes(src.read(line * a.object_users))
            # equal scores on the small file; this also warms the library and the allocator up
            small_cols, small_split = columnar("Small", sc)
            small_obj, t_obj = object_path("Small", sc)
            out["scores_identical"] = all(scores(small_cols[g]) == scores(small_obj[g]) and
                                          small_cols[g].bestIdx == small_obj[g].bestIdx for g, _ in GENERATORS)
            out["small_file"] = {"columnar": small_split, "object_s": t_obj,
                                 "best_idx": {g: small_cols[g].bestIdx for g, _ in GENERATORS},
                                 "scores": {g: scores(small_cols[g]) for g, _ in GENERATORS}}
            _, split = columnar("Big", sc)
            out["columnar"] = split
            out["object"] = {g: {"users_measured": a.object_users, "measured_s": t_obj[g],
                                 "extrapolated_s_for_users": t_obj[g] / a.object_users * a.users,
                                 "label": "extrapolated"} for g, _ in GENERATORS}
            out["speedup_vs_object_extrapolated"] = {
                g: out["object"][g]["extrapolated_s_for_users"] / split[g]["total_s"] for g, _ in GENERATORS}
        finally:
            os.chdir(cwd)
    print(json.dumps(out))


if __name__ == "__main__":
    main()
