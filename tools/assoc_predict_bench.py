#!/usr/bin/env python
"""Batch predict of the complementary purchase template on the GPU (pio_assoc_predict, DESIGN.md 4.15.1) against its
host paths.

Model: trained as tools/assoc_bench.py trains one (--events 10 M seeded buys over 1 M users and 100 k Zipf-popular
items, minSupport 1e-5, no confidence or lift cut), once per --length (maxRuleLength 3 and 4).
Queries, seeded: --queries (1 M) short queries of 1 to 8 items drawn Zipf over the items, about 5 % of them unknown
ids and about 10 % of the queries repeating an item, num 1 to 5; plus --long (200) queries of 100 to 1000 items.

Reported per length, each a host clock around work that ends in a device synchronise (or in host objects built from
arrays the device returned):
  - predictMany on all queries, split into string mapping (query_arrays), the device call (AssocIndex.predict, with the
    device milliseconds of native.assoc_predict_stats) and object building (rule_results);
  - BatchPredict.lines on the column path, and BatchPredict.run + json.dumps (the object path);
  - the predict loop on the first --prefix short queries, and that time scaled to all short queries, labelled
    extrapolated (the long queries are out of its reach: a 1000-item query has C(1000, 3) = 1.7e8 subsets).
Checked in the same run: the column path's lines equal the object path's byte for byte, and both equal the predict loop
on the prefix.  Also the card's name and power limit.

    python tools/assoc_predict_bench.py [--events 10000000] [--queries 1000000] [--long 200] [--lengths 3 4]
"""
import argparse
import json
import sys
import time
from pathlib import Path
from types import SimpleNamespace

import numpy as np

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))
sys.path.insert(0, str(ROOT / "tools"))
import pio_b200  # noqa: E402,F401
from assoc_bench import buys, card  # noqa: E402
from pio_b200 import native  # noqa: E402
from pio_b200 import storage as s  # noqa: E402
from pio_b200 import workflow as w  # noqa: E402
from pio_b200.templates import complementarypurchase as cp  # noqa: E402


def queries(n_short, n_long, n_items, seed):
    """(query JSON, Query) pairs, as BatchPredict.read_queries gives them."""
    rng = np.random.default_rng(seed)
    lens = rng.integers(1, 9, n_short)
    ids = (rng.zipf(1.3, int(lens.sum())) - 1) % n_items
    ids = np.where(rng.random(ids.shape[0]) < 0.05, n_items + ids, ids)   # unknown ids
    names = [f"i{x}" for x in ids.tolist()]
    out, at = [], 0
    rep = rng.random(n_short) < 0.1
    num = rng.integers(1, 6, n_short).tolist()
    for j, L in enumerate(lens.tolist()):
        items = names[at:at + L]
        at += L
        if rep[j]:
            items.append(items[0])
        out.append({"items": items, "num": num[j]})
    for L in rng.integers(100, 1001, n_long).tolist():
        out.append({"items": [f"i{x}" for x in rng.choice(n_items, L, replace=False).tolist()], "num": 3})
    return [(q, cp.Query(**q)) for q in out]


def timed(f):
    t0 = time.perf_counter()
    r = f()
    return time.perf_counter() - t0, r


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--events", type=int, default=10_000_000)
    ap.add_argument("--users", type=int, default=1_000_000)
    ap.add_argument("--items", type=int, default=100_000)
    ap.add_argument("--lengths", type=int, nargs="+", default=[3, 4])
    ap.add_argument("--min-support", type=float, default=1e-5)
    ap.add_argument("--queries", type=int, default=1_000_000)
    ap.add_argument("--long", type=int, default=200)
    ap.add_argument("--prefix", type=int, default=20_000)
    a = ap.parse_args()
    print(f"card: {card()}")
    native.lib()
    u, i, t = buys(a.events, a.users, a.items, a.events)
    itemMap = s.BiMap({f"i{k}": k for k in range(a.items)})
    qs = queries(a.queries, a.long, a.items, 11)
    objs = [q for _, q in qs]
    print(f"queries: {a.queries} short + {a.long} long, {sum(len(q.items) for q in objs)} items", flush=True)
    failed = False
    for length in a.lengths:
        p = {"basketWindow": 120, "maxRuleLength": length, "minSupport": a.min_support, "minConfidence": 0.0,
             "minLift": 0.0, "minBasketSize": 2, "maxNumRulesPerCond": 5}
        arrays = native.assoc_train(u, i, t, a.users, a.items, p["basketWindow"], length, p["minSupport"], 0.0, 0.0, 2, 5)
        model = cp.Model(arrays, itemMap, length)
        algo, serving = cp.Algorithm(cp.AlgorithmParams(**p)), cp.Serving()
        server = SimpleNamespace(algorithms=[algo], models=[model], serving=serving)
        print(f"maxRuleLength {length}: sets {np.diff(arrays['level_off']).tolist()}, rules "
              f"{arrays['rule_cond'].shape[0]}", flush=True)
        algo.predictMany(model, objs[:1000])                                 # warm-up: the index's device copy
        # predictMany, by phase, in BatchPredict's chunks
        chunk = w.BatchPredict.QUERY_CHUNK
        t_map = t_dev = t_obj = dev_ms = 0.0
        n_conds = 0
        for c0 in range(0, len(objs), chunk):
            part = objs[c0:c0 + chunk]
            dt, arr = timed(lambda: cp.query_arrays(model, part))
            t_map += dt
            dt, res = timed(lambda: model.device_index().predict(*arr, length - 1))
            t_dev += dt
            dev_ms += native.assoc_predict_stats()["device_ms"]
            n_conds += res[3].shape[0]
            cols = native.RuleColumns(*res, model.rule_conseq, model.support, model.confidence, model.lift,
                                      model.item_names(), 0)
            dt, _ = timed(lambda: cp.rule_results(cols))
            t_obj += dt
        print(f"  predictMany: mapping {t_map:.2f} s, device call {t_dev:.2f} s (device {dev_ms / 1e3:.2f} s), "
              f"objects {t_obj:.2f} s; {n_conds} conds", flush=True)
        t_col, col = timed(lambda: list(w.BatchPredict.lines(server, qs, chunk)))
        print(f"  BatchPredict: column path {t_col:.2f} s ({len(col)} lines, {sum(map(len, col)) / 1e6:.1f} MB)",
              flush=True)
        t_objp, objl = timed(lambda: [json.dumps(r, separators=(",", ":")) for r in w.BatchPredict.run(server, qs, chunk)])
        print(f"  BatchPredict: object path {t_objp:.2f} s", flush=True)
        n = min(a.prefix, a.queries)
        t_loop, loop = timed(lambda: [json.dumps({"query": w.to_json(q), "prediction": w.to_json(
            serving.serve(q, [algo.predict(model, q)]))}, separators=(",", ":")) for q in objs[:n]])
        print(f"  predict loop: {t_loop:.2f} s for {n} short queries; {t_loop * a.queries / n:.1f} s for "
              f"{a.queries} (extrapolated)", flush=True)
        same_cols, same_loop = col == objl, col[:n] == loop
        print(f"  column bytes == object bytes: {same_cols}; == predict loop on the prefix: {same_loop}", flush=True)
        failed |= not (same_cols and same_loop)
        model.device_index().close()
    if failed:
        raise SystemExit("the column path, the object path and the predict loop disagree")


if __name__ == "__main__":
    main()
