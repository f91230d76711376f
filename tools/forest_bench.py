"""Time RandomForest.trainClassifier on the GPU on a seeded set shaped like the classification template's data (rows of
three numeric attributes and a plan label in 0..3), per phase, and the restatement tests/forest_ref.py on a prefix,
extrapolated per row.

Two configurations: the template's engine.json (5 trees, auto, gini, maxDepth 4, maxBins 100) and a larger forest
(100 trees, auto, gini, maxDepth 10, maxBins 32).  The histogram pass's algorithmic bytes come from the shapes: per
level and tree group, every row's bin codes (uint8 per feature), its class (uint8) and one int32 node id per tree of
the group; bootstrap weights are recomputed from the counter hash and read nothing.  Prints one JSON line with the
card's name and power limit (and writes it to --out when given).

    python tools/forest_bench.py [--rows 10000000] [--host-rows 100000] [--out result.json]
"""
import argparse
import json
import subprocess
import sys
import time
from pathlib import Path

import numpy as np

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))
import pio_b200  # noqa: E402,F401
from pio_b200 import mllib, native  # noqa: E402
from tests import forest_ref as fr  # noqa: E402

HBM_BYTES_PER_S = 3.35e12      # H100 SXM data sheet


def make_set(n, seed):
    rng = np.random.default_rng(seed)
    x = np.round(rng.normal(size=(n, 3)) * [3.0, 2.0, 5.0] + [5.0, 0.0, 10.0], 2)
    score = x[:, 0] + 1.5 * x[:, 1] - 0.4 * x[:, 2] + rng.normal(size=n)
    y = np.digitize(score, np.quantile(score, [0.25, 0.5, 0.75])).astype(np.float64)
    return y, x


def run(y, x, cfg, host_rows):
    T, strategy, depth, bins = cfg["numTrees"], cfg["featureSubsetStrategy"], cfg["maxDepth"], cfg["maxBins"]
    n, F = x.shape
    t0 = time.perf_counter()
    m = mllib.RandomForest.trainClassifier(y, x, 4, {}, T, strategy, "gini", depth, bins)
    train_s = time.perf_counter() - t0
    tm = native.rf_train_timing()
    m.predictBatch(x[:1000])
    t0 = time.perf_counter()
    pred = m.predictBatch(x)
    pred_s = time.perf_counter() - t0
    # algorithmic bytes of the histogram passes: per level, each group reads bins + class once and its node ids
    levels = tm["levels"]
    hist_bytes = levels * (tm["groups"] * n * (F + 1) + 4 * n * T)
    t0 = time.perf_counter()
    want = fr.train(y[:host_rows], x[:host_rows], 4, T, strategy, "gini", depth, bins)
    host_s = (time.perf_counter() - t0) * n / host_rows
    # the same prefix on the GPU must give the restatement's forest, node for node
    got = native.rf_train(y[:host_rows], x[:host_rows], 4, T, strategy, native.RF_GINI, depth, bins)
    prefix_equal = all(np.array_equal(got[k], want[k]) for k in got)
    return {
        "config": cfg, "train_s": round(train_s, 3), "nodes": m.totalNumNodes, "depth": [int(d) for d in m.depth[:5]],
        "phase_ms": {k: round(v, 2) for k, v in tm.items() if isinstance(v, float)},
        "hist_level_ms": [round(v, 2) for v in tm["hist_level_ms"]],
        "select_level_ms": [round(v, 2) for v in tm["select_level_ms"]],
        "levels": levels, "groups": tm["groups"],
        "hist_bytes": hist_bytes,
        "hist_bytes_per_s": hist_bytes / (tm["hist_ms"] / 1e3) if tm["hist_ms"] else None,
        "hist_share_of_hbm": hist_bytes / (tm["hist_ms"] / 1e3) / HBM_BYTES_PER_S if tm["hist_ms"] else None,
        "predict_rows_per_s": n / pred_s, "train_accuracy": float((pred == y).mean()),
        "restatement_s_extrapolated": round(host_s, 1), "restatement_rows": host_rows,
        "prefix_equals_restatement": prefix_equal,
    }


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rows", type=int, default=10_000_000)
    ap.add_argument("--host-rows", type=int, default=100_000, help="prefix timed on the NumPy restatement")
    ap.add_argument("--seed", type=int, default=1)
    ap.add_argument("--out")
    args = ap.parse_args()
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                         text=True).stdout.strip().splitlines()
    y, x = make_set(args.rows, args.seed)
    mllib.RandomForest.trainClassifier(y[:100_000], x[:100_000], 4, {}, 5, "auto", "gini", 4, 100)   # warm-up
    out = {"gpu": gpu, "rows": args.rows, "runs": []}
    for cfg in (dict(numTrees=5, featureSubsetStrategy="auto", maxDepth=4, maxBins=100),
                dict(numTrees=100, featureSubsetStrategy="auto", maxDepth=10, maxBins=32)):
        out["runs"].append(run(y, x, cfg, min(args.host_rows, args.rows)))
    line = json.dumps(out)
    print(line)
    if args.out:
        Path(args.out).write_text(line + "\n")


if __name__ == "__main__":
    main()
