#!/usr/bin/env python
"""The similarproduct engine's BatchPredict on the column path (predictManyColumns + serveManyColumns, the z-score merge
on the GPU) against the object path (predictMany + Serving.serve per query).

Workload (DESIGN.md 4.9.1): seeded events of 1 M users over 100 k items (1-8 views and 0-3 likes / dislikes per user,
item popularity skewed); ALSAlgorithm (views), LikeAlgorithm (likes) and CooccurrenceAlgorithm (n = 50) trained on
them; 1 M queries of 1-5 items mixing every filter field, written as BatchPredict writes them in chunks of 16 384.
Nothing is read from outside the tree; the output lines are hashed, not written.

The object path is forced with a Serving that lacks serveManyColumns.  Reported, each a host clock around work that
ends in a device synchronise: per path the end-to-end time, in alternated runs on one card; for the column path its
stages summed over the chunks (the algorithms' calls, the item numbering, the merge call, the rest of
serveManyColumns with the remap, the output lines) and the merge's device time (CUDA events, first upload to last copy back); whether
both paths wrote the same bytes; and the card's name, power limit and SM clock, read in the same run.

    python tools/serve_merge_bench.py [--users 1000000] [--items 100000] [--queries 1000000] [--rounds 1]
"""
import argparse
import hashlib
import json
import subprocess
import sys
import time
from pathlib import Path
from types import SimpleNamespace

import numpy as np

sys.path.insert(0, str(Path(__file__).resolve().parent.parent))
import pio_b200  # noqa: E402,F401
from pio_b200 import native  # noqa: E402

CHUNK = 16384   # workflow.BatchPredict.QUERY_CHUNK


def card():
    out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True, timeout=30, check=True).stdout.strip().splitlines()
    if not out:
        raise RuntimeError("nvidia-smi reported no GPU")
    return out[0]


def queries(rng, ni, n):
    from pio_b200.templates import similarproduct as sp
    cats = [f"c{c}" for c in range(20)]

    def names(k):
        return [f"i{x}" for x in rng.integers(0, ni, k)]
    qs = []
    for j in range(n):
        items = names(int(rng.integers(1, 6))) + (["nope"] if j % 17 == 0 else [])
        qs.append(sp.Query(items=items, num=int((10, 20, 50, 1)[j % 4]),
                           categories={cats[j % 20], cats[(j * 7) % 20]} if j % 3 == 0 else None,
                           categoryBlackList={cats[j % 5]} if j % 4 == 0 else None,
                           whiteList=set(names(200)) if j % 10 == 0 else None,
                           blackList=set(names(10)) if j % 2 else None))
    return qs


def models(rng, nu, ni):
    from pio_b200.mllib import ALS
    from pio_b200.storage import BiMap
    from pio_b200.templates import similarproduct as sp
    views = rng.integers(1, 9, nu)
    u = np.repeat(np.arange(nu, dtype=np.int32), views)
    i = np.minimum((rng.random(u.shape[0]) ** 3 * ni).astype(np.int32), ni - 1)
    likes = rng.integers(0, 4, nu)
    lu = np.repeat(np.arange(nu, dtype=np.int32), likes)
    li = np.minimum((rng.random(lu.shape[0]) ** 2 * ni).astype(np.int32), ni - 1)
    lv = np.where(rng.random(lu.shape[0]) < 0.7, 1.0, -1.0).astype(np.float32)
    lt = np.arange(lu.shape[0], dtype=np.int64)
    cats = [f"c{c}" for c in range(20)]
    props = {k: sp.Item(categories=None if k % 11 == 0 else [cats[k % 20], cats[(k * 3) % 20]]) for k in range(ni)}
    names = BiMap({f"i{k}": k for k in range(ni)})
    als = ALS.trainImplicit((u, i, np.ones(u.shape[0], np.float32)), rank=10, iterations=10, lambda_=0.01, blocks=-1,
                            alpha=1.0, seed=1, dedup="sum", n_users=nu, n_products=ni)
    like = ALS.trainImplicit((lu, li, lv, lt), rank=10, iterations=10, lambda_=0.01, blocks=-1, alpha=1.0, seed=2,
                             dedup="keep_last", n_users=nu, n_products=ni)
    ti, tc, tn = native.cooc_train(u, i, nu, ni, 50)
    return ([sp.ALSAlgorithm(sp.ALSAlgorithmParams(10, 10)), sp.LikeAlgorithm(sp.ALSAlgorithmParams(10, 10)),
             sp.CooccurrenceAlgorithm(sp.CooccurrenceAlgorithmParams(n=50))],
            [sp.ALSModel(als, names, props), sp.ALSModel(like, names, props),
             sp.CooccurrenceModel(ti, tc, tn, names, props)], int(u.shape[0]), int(lu.shape[0]))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--users", type=int, default=1_000_000)
    ap.add_argument("--items", type=int, default=100_000)
    ap.add_argument("--queries", type=int, default=1_000_000)
    ap.add_argument("--rounds", type=int, default=1)
    a = ap.parse_args()
    native.build()
    print(json.dumps({"card": card()}), flush=True)
    from pio_b200 import workflow as w
    from pio_b200.controller import LServing
    from pio_b200.templates import similarproduct as sp

    class ObjectServing(LServing):   # Serving without serveManyColumns: BatchPredict takes the object path
        serve = sp.Serving.serve

    rng = np.random.default_rng(0)
    algorithms, models_, n_views, n_likes = models(rng, a.users, a.items)
    qs = queries(rng, a.items, a.queries)
    pairs = [(None, q) for q in qs]
    print(json.dumps({"what": "workload", "users": a.users, "items": a.items, "views": n_views, "likes": n_likes,
                      "queries": a.queries}), flush=True)
    col = SimpleNamespace(algorithms=algorithms, models=models_, serving=sp.Serving())
    obj = SimpleNamespace(algorithms=algorithms, models=models_, serving=ObjectServing())
    assert w.BatchPredict.columnar(col) and not w.BatchPredict.columnar(obj)

    # column-path stages: wrappers that add host time per stage
    stage = {"algorithms_ms": 0.0, "numbering_ms": 0.0, "merge_call_ms": 0.0, "merge_device_ms": 0.0, "serve_ms": 0.0}

    def timed(key, f):
        def g(*args, **kw):
            t = time.perf_counter()
            r = f(*args, **kw)
            stage[key] += (time.perf_counter() - t) * 1e3
            if key == "merge_call_ms":
                stage["merge_device_ms"] += native.serve_merge_stats()["device_ms"]
            return r
        return g
    for alg in algorithms:
        alg.predictManyColumns = timed("algorithms_ms", alg.predictManyColumns)
    col.serving._numbering = timed("numbering_ms", col.serving._numbering)
    col.serving.serveManyColumns = timed("serve_ms", col.serving.serveManyColumns)
    merge = native.serve_zscore_merge
    native.serve_zscore_merge = timed("merge_call_ms", merge)

    def run(server):   # the digest of the lines, not the lines: both paths' output would not fit in memory together
        t = time.perf_counter()
        h = hashlib.sha256()
        for line in w.BatchPredict.lines(server, pairs, CHUNK):
            h.update(line.encode() + b"\n")
        return h.hexdigest(), (time.perf_counter() - t) * 1e3

    for server in (col, obj):                                              # warm-up: uploads, first launches
        list(w.BatchPredict.lines(server, pairs[:CHUNK], CHUNK))
    times = {"column": [], "object": []}
    same = True
    for r in range(a.rounds):
        for k in stage:
            stage[k] = 0.0
        lines_c, ms_c = run(col)
        times["column"].append(round(ms_c, 1))
        st = dict(stage)
        lines_o, ms_o = run(obj)
        times["object"].append(round(ms_o, 1))
        same = same and lines_c == lines_o
        print(json.dumps({"what": f"round {r}", "column_ms": round(ms_c, 1), "object_ms": round(ms_o, 1)}), flush=True)
    native.serve_zscore_merge = merge
    serve_rest = st["serve_ms"] - st["numbering_ms"] - st["merge_call_ms"]
    out_ms = times["column"][-1] - st["algorithms_ms"] - st["serve_ms"]
    print(json.dumps({"what": f"BatchPredict of {a.queries} queries in chunks of {CHUNK}, last round",
                      "column_ms": times["column"], "object_ms": times["object"], "same_bytes": same,
                      "column_stages_ms": {"algorithms": round(st["algorithms_ms"], 1),
                                           "numbering": round(st["numbering_ms"], 1),
                                           "merge_call": round(st["merge_call_ms"], 1),
                                           "merge_device": round(st["merge_device_ms"], 1),
                                           "rest_of_serveManyColumns": round(serve_rest, 1),
                                           "output_lines": round(out_ms, 1)},
                      "merge_share_of_column_path": round(st["merge_call_ms"] / times["column"][-1], 4),
                      "card": card()}), flush=True)


if __name__ == "__main__":
    main()
