#!/usr/bin/env python
"""Training of the lead scoring template on the GPU (RandomForest.trainRegressor, DESIGN.md 4.16), per phase and end to
end, against the NumPy restatement (tests/forest_reg_ref.py) on a subsample.

Workload, seeded: --rows labeled points with three categorical features of arities 1000, 100 and 10 (Zipf-skewed) and
one continuous feature, 0 / 1 labels that depend on them.  Reported, each a host clock around work that ends in a device
synchronise, with the phases of native.rf_train_timing:
  - trainRegressor with the template's parameters (5 trees, "auto", maxDepth 4; maxBins 1000 so that the widest feature
    fits) and with a deeper forest (--deep-trees trees, "all", maxDepth --deep-depth), --rounds times each;
  - end to end from an event file of --sessions sessions: DataSource.readTraining (GPU scan, device session ids and
    sessions) + Preparator + RFAlgorithm.train with the doc's parameters but maxBins 1024 (1000 pages and "" need
    1001 bins);
  - forest_reg_ref.train on a --sample-row subsample, and the device on the same subsample, whose forests must be equal.
Also the card's name and power limit.

    python tools/leadscoring_bench.py [--rows 10000000] [--sessions 300000] [--rounds 2]
"""
import argparse
import datetime as dt
import json
import os
import shutil
import subprocess
import sys
import tempfile
import time
from pathlib import Path

import numpy as np

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))
import pio_b200  # noqa: E402,F401
from pio_b200 import mllib, native  # noqa: E402

ARITIES = (1000, 100, 10)


def card():
    out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                         capture_output=True, text=True, timeout=30, check=True).stdout.strip().splitlines()
    return out[0] if out else "unknown"


def points(n, seed):
    rng = np.random.default_rng(seed)
    cols, score = [], np.zeros(n)
    for a in ARITIES:
        v = np.minimum(rng.zipf(1.2, n) - 1, a - 1)
        v = rng.permutation(a)[v].astype(np.float64)
        cols.append(v)
        score += np.sin(v * 0.37)
    c = np.round(rng.normal(size=n) * 3, 1)
    cols.append(c)
    score += 0.3 * c
    y = (score + rng.normal(size=n) > np.median(score)).astype(np.float64)
    return y, np.stack(cols, axis=1)


def timed_train(y, x, T, strategy, depth, bins, seed=1):
    cat = {k: a for k, a in enumerate(ARITIES)}
    t0 = time.perf_counter()
    m = mllib.RandomForest.trainRegressor(y, x, cat, T, strategy, "variance", depth, bins, seed=seed)
    wall = (time.perf_counter() - t0) * 1e3
    tm = native.rf_train_timing()
    return m, dict(wall_ms=wall, nodes=int(m.totalNumNodes), paths=native.rf_train_paths(),
                   **{k: tm[k] for k in ("h2d_ms", "split_ms", "bin_ms", "hist_ms", "select_ms", "update_ms", "levels")})


def event_file(app, n_sessions, seed):
    from pio_b200 import storage as s
    rng = np.random.default_rng(seed)
    t0 = dt.datetime(2021, 3, 1, tzinfo=dt.timezone.utc)
    lines = []
    for k in range(n_sessions):
        base = t0 + dt.timedelta(seconds=int(rng.integers(0, 10 ** 7)))
        for v in range(int(rng.integers(1, 4))):
            when = (base + dt.timedelta(milliseconds=int(rng.integers(0, 5000)))).isoformat()
            lines.append(json.dumps(dict(
                event="view", entityType="user", entityId=f"u{k % 5000}", targetEntityType="page",
                targetEntityId=f"example.com/page{int(min(rng.zipf(1.3), 1000))}", eventTime=when,
                properties={"sessionId": f"s{k}", "referrerId": f"ref{int(min(rng.zipf(1.5), 100))}.com",
                            "browser": ["Chrome", "Firefox", "Safari", "Edge"][int(rng.integers(0, 4))]})))
        if rng.random() < 0.2:
            when = (base + dt.timedelta(seconds=int(rng.integers(1, 600)))).isoformat()
            lines.append(json.dumps(dict(event="buy", entityType="user", entityId=f"u{k % 5000}",
                                         targetEntityType="item", targetEntityId="i1", eventTime=when,
                                         properties={"sessionId": f"s{k}"})))
    p = s.app_file(app, None)
    p.parent.mkdir(parents=True, exist_ok=True)
    p.write_text("\n".join(lines) + "\n")
    return len(lines), p.stat().st_size


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rows", type=int, default=10_000_000)
    ap.add_argument("--sessions", type=int, default=300_000)
    ap.add_argument("--rounds", type=int, default=2)
    ap.add_argument("--deep-trees", type=int, default=20)
    ap.add_argument("--deep-depth", type=int, default=10)
    ap.add_argument("--sample-rows", type=int, default=20_000)
    a = ap.parse_args()
    out = {"card": card()}
    y, x = points(a.rows, 7)
    for name, (T, strat, depth) in (("template", (5, "auto", 4)), ("deep", (a.deep_trees, "all", a.deep_depth))):
        out[name] = [timed_train(y, x, T, strat, depth, 1000)[1] for _ in range(a.rounds)]
    # end to end from an event file
    from pio_b200 import workflow as w
    from pio_b200.templates import leadscoring as ls
    tmp = tempfile.mkdtemp()
    try:
        os.environ["PIO_EVENTDATA_DIR"] = tmp
        n_ev, n_bytes = event_file("LSB", a.sessions, 3)
        sc = w.WorkflowContext()
        t0 = time.perf_counter()
        td = ls.DataSource(ls.DataSourceParams("LSB")).readTraining(sc)
        t1 = time.perf_counter()
        pd = ls.Preparator().prepare(sc, td)
        t2 = time.perf_counter()
        ls.RFAlgorithm(ls.RFAlgorithmParams(5, "auto", "variance", 4, 1024, 12345)).train(sc, pd)
        t3 = time.perf_counter()
        out["end_to_end"] = dict(events=n_ev, file_bytes=n_bytes, sessions=len(td.features()[0]),
                                 read_ms=(t1 - t0) * 1e3, prepare_ms=(t2 - t1) * 1e3, train_ms=(t3 - t2) * 1e3)
    finally:
        shutil.rmtree(tmp, ignore_errors=True)
    # the restatement on a subsample, and the device on the same rows
    sys.path.insert(0, str(ROOT))
    from tests import forest_reg_ref as rr
    ys, xs = y[:a.sample_rows], x[:a.sample_rows]
    cat = {k: ar for k, ar in enumerate(ARITIES)}
    t0 = time.perf_counter()
    want = rr.train(ys, xs, 5, "auto", "variance", 4, 1000, seed=1, categorical=cat)
    ref_ms = (time.perf_counter() - t0) * 1e3
    m, dev = timed_train(ys, xs, 5, "auto", 4, 1000)
    same = all(np.array_equal(np.asarray(m.nodes[k]), want[k]) for k in
               ("tree_off", "feature", "left", "right", "count", "cat_off", "cat_ids", "threshold", "prediction",
                "impurity", "gain"))
    out["subsample"] = dict(rows=a.sample_rows, restatement_ms=ref_ms, device_ms=dev["wall_ms"], equal=same)
    print(json.dumps(out))


if __name__ == "__main__":
    main()
