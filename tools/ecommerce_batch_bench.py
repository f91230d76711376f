#!/usr/bin/env python
"""The ecommerce engine's BatchPredict on the column path (predictManyColumns + LFirstServing.serveManyColumns) against
the object path (predictMany + serveBase per query), and the popularity rule of its cold users on the GPU
(pio_popular_predict_filtered) against the host loop it replaced.

Workload (DESIGN.md 4.14), seeded, written to a temporary event store: 1 M users over 100 k items in 50 categories
(five items also in a category "rare"); rate events of 40 % of the users (the known users), view events of the next
30 % (unknown users with recent items), buy events skewed to popular items plus 3 000 buys each for 20 cold users (long
seen lists), `unavailableItems` and `weightedItems` (weights 0, -1 and 50).  ECommAlgorithm is trained through
CreateWorkflow (unseenOnly, seenEvents buy, similarEvents view), then 200 k queries mix known, recent-view and cold users
with category, white and black lists; one in 20 is the worst case, a heavy cold user asking for the "rare" category.

Reported, each a host clock around work that ends in a device synchronise: BatchPredict.lines over all queries in
chunks of 16 384, column path against object path, alternated, with the SHA-256 of both outputs compared; the
pio_popular_predict_filtered calls of the column path (time, rows, last_walked); and the host loop predictMany ran for
the default rows before (dense mask, candidate list, sort), timed on a prefix of those rows and extrapolated to all of
them -- labelled as extrapolated, it is not run in full.  That prefix is timed inside the column run, so the column
path is also reported without it.  Also the card's name and power limit.

    python tools/ecommerce_batch_bench.py [--users 1000000] [--items 100000] [--queries 200000] [--rounds 2]
"""
import argparse
import hashlib
import json
import os
import shutil
import subprocess
import sys
import tempfile
import time
from pathlib import Path

import numpy as np

sys.path.insert(0, str(Path(__file__).resolve().parent.parent))
import pio_b200  # noqa: E402,F401
from pio_b200 import native  # noqa: E402

CHUNK = 16384   # workflow.BatchPredict.QUERY_CHUNK
N_CATS, N_HEAVY, HEAVY_BUYS = 50, 20, 3000


def card():
    out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True, timeout=30, check=True).stdout.strip().splitlines()
    if not out:
        raise RuntimeError("nvidia-smi reported no GPU")
    return out[0]


def write_events(path, nu, ni, rng):
    """The shop's event file; returns the user ranges (known, recent-view, cold) and the heavy cold users."""
    known, recent = int(nu * 0.4), int(nu * 0.7)
    heavy = list(range(recent, recent + N_HEAVY))
    lines = [f'{{"event": "$set", "entityType": "user", "entityId": "u{k}", "eventTime": "2021-01-01T00:00:00Z"}}\n'
             for k in range(nu)]
    for k in range(ni):
        cats = [f"c{k % N_CATS}"] + (["rare"] if k % (ni // 5) == 3 else [])
        lines.append(f'{{"event": "$set", "entityType": "item", "entityId": "i{k}", "properties": '
                     f'{{"categories": {json.dumps(cats)}}}, "eventTime": "2021-01-01T00:00:00Z"}}\n')

    def events(name, users, items, ratings=None):
        secs = rng.integers(0, 86400, users.shape[0]).tolist()
        ratings = [None] * users.shape[0] if ratings is None else ratings.tolist()
        for u, i, v, t in zip(users.tolist(), items.tolist(), ratings, secs):
            props = "" if v is None else f', "properties": {{"rating": {v}}}'
            lines.append(f'{{"event": "{name}", "entityType": "user", "entityId": "u{u}", "targetEntityType": "item", '
                         f'"targetEntityId": "i{i}"{props}, '
                         f'"eventTime": "2021-01-02T{t // 3600:02d}:{t // 60 % 60:02d}:{t % 60:02d}Z"}}\n')

    ru = np.repeat(np.arange(known), rng.integers(1, 7, known))
    events("rate", ru, np.minimum((rng.random(ru.shape[0]) ** 2 * ni).astype(np.int64), ni - 1),
           rng.integers(1, 6, ru.shape[0]))
    vu = np.repeat(np.arange(known, recent), rng.integers(1, 4, recent - known))
    events("view", vu, rng.integers(0, ni, vu.shape[0]))
    bu = rng.integers(0, nu, 300_000)
    events("buy", bu, np.minimum((rng.random(bu.shape[0]) ** 3 * ni).astype(np.int64), ni - 1))
    hu = np.repeat(np.array(heavy), HEAVY_BUYS)
    events("buy", hu, rng.integers(0, ni, hu.shape[0]))
    unavailable = [f"i{k}" for k in rng.choice(ni, 100, replace=False)]
    weights = [{"items": [f"i{k}" for k in range(0, ni, 7)], "weight": 0.0},
               {"items": [f"i{k}" for k in range(1, ni, 5)], "weight": -1.0},
               {"items": [f"i{k}" for k in range(2, ni // 10, 3)], "weight": 50.0}]
    for eid, props in (("unavailableItems", {"items": unavailable}), ("weightedItems", {"weights": weights})):
        lines.append(json.dumps({"event": "$set", "entityType": "constraint", "entityId": eid, "properties": props,
                                 "eventTime": "2021-01-03T00:00:00Z"}) + "\n")
    path.parent.mkdir(parents=True, exist_ok=True)
    path.write_text("".join(lines))
    return known, recent, heavy, len(lines)


def queries(rng, nu, ni, known, recent, heavy, n):
    from pio_b200.templates import ecommerce as ec
    qs = []
    for j in range(n):
        kind = j % 20
        if kind == 0:        # the worst case: a heavy cold user (3 000 seen items), a category of five items
            qs.append(ec.Query(user=f"u{heavy[j % len(heavy)]}", num=20, categories={"rare"}))
            continue
        user = (f"u{rng.integers(0, known)}" if kind < 8 else f"u{rng.integers(known, recent)}" if kind < 13 else
                f"u{rng.integers(recent, nu)}" if kind < 17 else f"ghost{j}")
        qs.append(ec.Query(user=user, num=int((10, 20, 50, 1)[j % 4]),
                           categories={f"c{j % N_CATS}", f"c{(j * 7) % N_CATS}"} if j % 3 == 0 else None,
                           whiteList={f"i{x}" for x in rng.integers(0, ni, 200)} if j % 10 == 1 else None,
                           blackList={f"i{x}" for x in rng.integers(0, ni, 10)} if j % 2 else None))
    return qs


def host_default_rows(scores, qf, rows, nums):
    """The host loop predictMany ran for default rows before: per row a dense mask, a candidate list, a sort."""
    n_items = scores.shape[0]
    for r in rows:
        mask = np.zeros(n_items, bool)
        if qf.has_wl is not None and qf.has_wl[r]:
            mask[:] = True
            mask[qf.wl_items[qf.wl_ptr[r]:qf.wl_ptr[r + 1]]] = False
        mask[qf.ex_items[qf.ex_ptr[r]:qf.ex_ptr[r + 1]]] = True
        if qf.set_ix is not None and qf.set_ix[r] >= 0:
            mask |= qf.item_sets[qf.set_ix[r]].astype(bool)
        cand = [(int(i), float(scores[i])) for i in np.flatnonzero(~mask)]
        cand.sort(key=lambda kv: (-kv[1], kv[0]))
        cand[:nums[r]]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--users", type=int, default=1_000_000)
    ap.add_argument("--items", type=int, default=100_000)
    ap.add_argument("--queries", type=int, default=200_000)
    ap.add_argument("--rounds", type=int, default=2)
    ap.add_argument("--host-rows", type=int, default=300, help="default rows of the host-loop prefix")
    a = ap.parse_args()
    native.build()
    print(json.dumps({"card": card()}), flush=True)
    tmp = Path(tempfile.mkdtemp(prefix="ecomm_bench_"))
    try:
        run_bench(a, tmp)
    finally:
        shutil.rmtree(tmp, ignore_errors=True)


def run_bench(a, tmp):
    os.environ["PIO_EVENTDATA_DIR"] = str(tmp / "events")
    os.environ["PIO_MODELDATA_DIR"] = str(tmp / "models")
    from pio_b200 import storage as s
    from pio_b200 import workflow as w
    rng = np.random.default_rng(0)
    t = time.perf_counter()
    known, recent, heavy, n_events = write_events(s.app_file("Shop"), a.users, a.items, rng)
    variant = tmp / "engine.json"
    variant.write_text(json.dumps({
        "id": "default", "engineFactory": "pio_b200.templates.ecommerce.ECommerceRecommendationEngine",
        "datasource": {"params": {"appName": "Shop"}},
        "algorithms": [{"name": "ecomm", "params": {"appName": "Shop", "unseenOnly": True, "seenEvents": ["buy"],
                                                    "similarEvents": ["view"], "rank": 10, "numIterations": 10,
                                                    "lambda": 0.01, "seed": 3}}]}))
    inst = w.CreateWorkflow.main(["--engine-id", "shop", "--engine-version", "1", "--engine-variant", str(variant)])
    server = w.deploy(inst.id)
    qs = queries(rng, a.users, a.items, known, recent, heavy, a.queries)
    pairs = [(None, q) for q in qs]
    print(json.dumps({"what": "workload", "users": a.users, "items": a.items, "events": n_events,
                      "queries": a.queries, "setup_s": round(time.perf_counter() - t, 1)}), flush=True)
    assert w.BatchPredict.columnar(server)

    # the popularity calls of the column path: host clock around each call (it ends in a stream synchronise)
    calls = {"ms": 0.0, "rows": 0, "walked": 0, "listed": 0, "host_ms": 0.0, "host_rows": 0}
    predict = native.PopularModel.predict_filtered

    def timed(self, n, topk, qf=None):
        t0 = time.perf_counter()
        r = predict(self, n, topk, qf)
        calls["ms"] += (time.perf_counter() - t0) * 1e3
        st = self.stats()
        calls["rows"] += n
        calls["walked"] += st["last_walked"]
        calls["listed"] += st["last_listed"]
        if calls["host_rows"] < a.host_rows:      # the host loop on a prefix of the same rows
            rows = list(range(min(n, a.host_rows - calls["host_rows"])))
            t0 = time.perf_counter()
            host_default_rows(timed.scores, qf, rows, [topk] * n)
            calls["host_ms"] += (time.perf_counter() - t0) * 1e3
            calls["host_rows"] += len(rows)
        return r

    model = server.models[0]

    def run(columnar):
        orig = w.BatchPredict.columnar
        if not columnar:
            w.BatchPredict.columnar = staticmethod(lambda server: False)
        try:
            t0 = time.perf_counter()
            h = hashlib.sha256()
            for line in w.BatchPredict.lines(server, pairs, CHUNK):
                h.update(line.encode() + b"\n")
            return h.hexdigest(), (time.perf_counter() - t0) * 1e3
        finally:
            w.BatchPredict.columnar = orig

    list(w.BatchPredict.lines(server, pairs[:CHUNK], CHUNK))          # warm-up: uploads, indexes, first launches
    w_ = server.algorithms[0]._weights(model)
    timed.scores = model.popularity() if w_ is None else model.popularity() * w_
    times = {"column": [], "object": []}
    same = True
    for r in range(a.rounds):
        for k in calls:
            calls[k] = 0 if isinstance(calls[k], int) else 0.0
        native.PopularModel.predict_filtered = timed
        digest_c, ms_c = run(True)
        native.PopularModel.predict_filtered = predict
        st = dict(calls)
        digest_o, ms_o = run(False)
        same = same and digest_c == digest_o
        times["column"].append(round(ms_c, 1))
        times["object"].append(round(ms_o, 1))
        print(json.dumps({"what": f"round {r}", "column_ms": round(ms_c, 1), "object_ms": round(ms_o, 1),
                          "same_bytes": digest_c == digest_o}), flush=True)
    per_row = st["host_ms"] / max(st["host_rows"], 1)
    print(json.dumps({"what": f"BatchPredict.lines of {a.queries} queries in chunks of {CHUNK}",
                      "column_ms": times["column"], "object_ms": times["object"], "same_bytes": same,
                      "column_ms_less_host_prefix_last_round": round(times["column"][-1] - st["host_ms"], 1),
                      "popular_calls_last_round": {"ms": round(st["ms"], 1), "rows": st["rows"],
                                                   "last_walked_sum": st["walked"], "last_listed_sum": st["listed"]},
                      "host_default_loop": {"timed_rows": st["host_rows"], "timed_ms": round(st["host_ms"], 1),
                                            "extrapolated_ms_for_all_rows": round(per_row * st["rows"], 1),
                                            "note": "extrapolated from the timed prefix, not run in full"},
                      "card": card()}), flush=True)
    assert same


if __name__ == "__main__":
    main()
