#!/usr/bin/env python
"""CooccurrenceAlgorithm.predictMany (pio_cooc_predict_filtered) against the predict loop.

Workload: seeded view events of 1 M users over 100 k items (1-8 views per user, item popularity skewed), trained with
pio_cooc_train at n = 50; then 1 M similarproduct queries of 1-5 items that mix every filter field (blackList,
whiteList, categories, an ignored categoryBlackList, unknown ids), scored in BatchPredict-sized chunks of 16 384.
Nothing is read from outside the tree.

Reported, each a host clock around work that ends in a device synchronise (the library call synchronises before it
returns): the device calls (pio_cooc_predict_filtered, uploads and downloads included) and the host work of
predictMany around them (query maps, filter lists, category rows, result objects), summed over the chunks after a
warm-up chunk; the predict loop over a prefix, extrapolated to all queries and flagged as such; whether both paths agree
exactly on that prefix; and the card's name and power limit, read in the same run (a failing nvidia-smi is an error).

    python tools/cooc_predict_bench.py [--users 1000000] [--items 100000] [--queries 1000000] [--prefix 5000]
"""
import argparse
import json
import subprocess
import sys
import time
from pathlib import Path

import numpy as np

sys.path.insert(0, str(Path(__file__).resolve().parent.parent))
import pio_b200  # noqa: E402,F401
from pio_b200 import native  # noqa: E402

CHUNK = 16384   # workflow.BatchPredict.QUERY_CHUNK


def card():
    out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                         text=True, timeout=30, check=True).stdout.strip().splitlines()
    if not out:
        raise RuntimeError("nvidia-smi reported no GPU")
    return out[0]


def workload(rng, nu, ni):
    per_user = rng.integers(1, 9, nu)
    u = np.repeat(np.arange(nu, dtype=np.int32), per_user)
    i = np.minimum((rng.random(u.shape[0]) ** 3 * ni).astype(np.int32), ni - 1)
    return u, i


def queries(rng, ni, n):
    from pio_b200.templates import similarproduct as sp
    cats = [f"c{c}" for c in range(20)]

    def names(k):
        return [f"i{x}" for x in rng.integers(0, ni, k)]
    qs = []
    for j in range(n):
        items = names(int(rng.integers(1, 6))) + (["nope"] if j % 17 == 0 else [])
        qs.append(sp.Query(items=items, num=int((10, 20, 50)[j % 3]),
                           categories={cats[j % 20], cats[(j * 7) % 20]} if j % 3 == 0 else None,
                           categoryBlackList={cats[j % 5]} if j % 4 == 0 else None,
                           whiteList=set(names(200)) if j % 10 == 0 else None,
                           blackList=set(names(10)) if j % 2 else None))
    return qs


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--users", type=int, default=1_000_000)
    ap.add_argument("--items", type=int, default=100_000)
    ap.add_argument("--queries", type=int, default=1_000_000)
    ap.add_argument("--prefix", type=int, default=5000)
    ap.add_argument("--n", type=int, default=50)
    a = ap.parse_args()
    native.build()
    print(json.dumps({"card": card()}), flush=True)
    from pio_b200.storage import BiMap
    from pio_b200.templates import similarproduct as sp
    rng = np.random.default_rng(0)
    u, i = workload(rng, a.users, a.items)
    t0 = time.perf_counter()
    ti, tc, tn = native.cooc_train(u, i, a.users, a.items, a.n)
    train_ms = (time.perf_counter() - t0) * 1e3
    cats = [f"c{c}" for c in range(20)]
    props = {k: sp.Item(categories=None if k % 11 == 0 else [cats[k % 20], cats[(k * 3) % 20]]) for k in range(a.items)}
    model = sp.CooccurrenceModel(ti, tc, tn, BiMap({f"i{k}": k for k in range(a.items)}), props)
    algo = sp.CooccurrenceAlgorithm(sp.CooccurrenceAlgorithmParams(n=a.n))
    qs = queries(rng, a.items, a.queries)
    print(json.dumps({"what": "workload", "users": a.users, "items": a.items, "views": int(u.shape[0]), "n": a.n,
                      "train_ms": round(train_ms, 1), "mean_top_n": round(float(tn.mean()), 2),
                      "queries": a.queries}), flush=True)

    dev = model.device_model()
    device_ms = [0.0]
    call = dev.predict_filtered

    def timed(*args, **kw):
        t = time.perf_counter()
        r = call(*args, **kw)
        device_ms[0] += (time.perf_counter() - t) * 1e3
        return r
    dev.predict_filtered = timed
    algo.predictMany(model, qs[:CHUNK])                                     # warm-up: upload, first launches
    device_ms[0] = 0.0
    expanded = rows = 0
    t0 = time.perf_counter()
    many = []
    for c in range(0, len(qs), CHUNK):
        many.extend(algo.predictMany(model, qs[c:c + CHUNK]))
        st = dev.stats()
        expanded += st["last_expanded"]
        rows += st["last_rows"]
    total_ms = (time.perf_counter() - t0) * 1e3
    t0 = time.perf_counter()
    each = [algo.predict(model, q) for q in qs[:a.prefix]]
    loop_ms = (time.perf_counter() - t0) * 1e3
    print(json.dumps({"what": f"predictMany of {a.queries} queries in chunks of {CHUNK}", "total_ms": round(total_ms, 1),
                      "device_call_ms": round(device_ms[0], 1), "host_ms": round(total_ms - device_ms[0], 1),
                      "queries_per_s": round(a.queries / total_ms * 1e3), "expanded_entries": expanded,
                      "rows_after_filters": rows}), flush=True)
    print(json.dumps({"what": f"predict loop over the first {a.prefix} queries", "ms": round(loop_ms, 1),
                      "queries_per_s": round(a.prefix / loop_ms * 1e3),
                      "extrapolated_ms_for_all_queries": round(loop_ms * a.queries / a.prefix, 1),
                      "extrapolated": True, "equal_on_prefix": many[:a.prefix] == each}), flush=True)
    dev.predict_filtered = call
    dev.close()


if __name__ == "__main__":
    main()
