"""Time the ecommerce template's serving lookups through the GPU event index (LEventStore.entityIndex) on seeded
ecommerce-shaped event files of two sizes, against the host path (LEventStore.findByEntity, one json.loads per line)
timed on a prefix and reported per event.

Per size: the index build split into file read, device scan and sort / merge; p50 / p99 of single-id `find` calls
(limit=10 and no limit); an append of 1 and of 10 000 events with the next `find`; the delta -> main merges of the
build; and ECommAlgorithm.predict p50 for a known user (unseenOnly) and for an unknown user with recent views.
Prints one JSON line with the card's name and power limit.

    python tools/event_index_bench.py [--sizes 2000000,20000000] [--finds 1000] [--host-lines 100000]
"""
import argparse
import datetime as dt
import json
import os
import subprocess
import sys
import tempfile
import time
from pathlib import Path

import numpy as np

sys.path.insert(0, str(Path(__file__).resolve().parent.parent))
import pio_b200  # noqa: E402,F401
from pio_b200 import native  # noqa: E402
from pio_b200 import storage as s  # noqa: E402
from pio_b200 import workflow as w  # noqa: E402
from pio_b200.templates import ecommerce as ec  # noqa: E402

N_USERS, N_ITEMS = 200_000, 20_000
T0 = np.datetime64("2015-01-01T00:00:00", "s")


def write_file(path, n, seed, mode="w"):
    """n events: user $set (1 %), item $set (0.1 %), and view / buy / rate events of users on items."""
    rng = np.random.default_rng(seed)
    kind = rng.choice(4, n, p=[0.01, 0.001, 0.8, 0.189]).tolist()
    u, i = rng.integers(0, N_USERS, n).tolist(), rng.integers(0, N_ITEMS, n).tolist()
    r = rng.integers(1, 6, n).tolist()
    times = np.datetime_as_string(T0 + rng.integers(0, 10 ** 8, n).astype("timedelta64[s]"), unit="s").tolist()
    with open(path, mode) as f:
        buf = []
        for j in range(n):
            k, t = kind[j], times[j]
            if k == 0:
                buf.append(f'{{"event": "$set", "entityType": "user", "entityId": "u{u[j]}", "properties": {{}}, '
                           f'"eventTime": "{t}Z"}}\n')
            elif k == 1:
                buf.append(f'{{"event": "$set", "entityType": "item", "entityId": "i{i[j]}", "properties": '
                           f'{{"categories": ["c{i[j] % 20}"]}}, "eventTime": "{t}Z"}}\n')
            else:
                ev = "view" if k == 2 else "buy" if r[j] < 3 else "rate"
                buf.append(f'{{"event": "{ev}", "entityType": "user", "entityId": "u{u[j]}", "targetEntityType": '
                           f'"item", "targetEntityId": "i{i[j]}", "properties": {{"rating": {r[j]}}}, '
                           f'"eventTime": "{t}Z"}}\n')
            if len(buf) >= 1 << 16:
                f.write("".join(buf))
                buf = []
        f.write("".join(buf))


def pct(xs, q):
    return float(np.percentile(np.asarray(xs) * 1e3, q))


def build_breakdown(app, view):
    """The build of one view's index piece by piece: file read, scan (chunk loop) and sort + merge, summed."""
    mode, tet = s._target_filter(view.get("targetEntityType", s._UNSET))
    ix = native.EventsIndex(view["entityType"], view["eventNames"], mode, tet)
    read_s, scan_ms, sort_ms, merges = 0.0, 0.0, 0.0, []
    t0 = time.perf_counter()
    with open(s.app_file(app), "rb") as fh:
        pieces = s._line_pieces(fh, s.FIND_COLUMNS_CHUNK)
        while True:
            r0 = time.perf_counter()
            p = next(pieces, None)
            read_s += time.perf_counter() - r0
            if p is None:
                break
            ix.append(p[1], p[0])
            st = ix.stats()
            scan_ms += st["scan_ms"]
            sort_ms += st["sort_ms"]
            if st["merge_ms"]:
                merges.append({"ms": round(st["merge_ms"], 2), "n_main_after": st["n_main"]})
    total = time.perf_counter() - t0
    st = ix.stats()
    ix.close()
    return {"total_s": round(total, 3), "read_s": round(read_s, 3), "scan_s": round(scan_ms / 1e3, 3),
            "sort_merge_s": round(sort_ms / 1e3, 3), "entries": st["n_main"] + st["n_delta"], "merges": merges}


def one_size(n, args, tmp):
    os.environ["PIO_EVENTDATA_DIR"] = str(tmp / f"ev{n}")
    app = "Big"
    p = s.app_file(app)
    p.parent.mkdir(parents=True, exist_ok=True)
    t = time.perf_counter()
    write_file(p, n, 1)
    out = {"events": n, "file_mb": round(p.stat().st_size / 2 ** 20, 1), "generate_s": round(time.perf_counter() - t, 1)}
    seen = dict(entityType="user", eventNames=["buy", "view"], targetEntityType="item")
    out["build"] = build_breakdown(app, seen)
    ix = s.LEventStore.entityIndex(app, **seen)
    t = time.perf_counter()
    ix.find("u0")
    out["first_find_s"] = round(time.perf_counter() - t, 3)
    rng = np.random.default_rng(2)
    for limit in (10, None):
        ts, n_ev = [], 0
        for k in rng.integers(0, N_USERS, args.finds).tolist():
            t = time.perf_counter()
            n_ev += len(ix.find(f"u{k}", limit))
            ts.append(time.perf_counter() - t)
        out[f"find_limit_{limit}_ms"] = {"p50": round(pct(ts, 50), 3), "p99": round(pct(ts, 99), 3),
                                         "events_per_find": round(n_ev / args.finds, 1)}
    t0 = dt.datetime(2020, 1, 1, tzinfo=dt.timezone.utc)
    for m in (1, 10000):
        s.import_events(app, [dict(event="view", entityType="user", entityId=f"u{k % N_USERS}", targetEntityType="item",
                                   targetEntityId="i1", eventTime=t0.isoformat()) for k in range(m)])
        t = time.perf_counter()
        ix.find("u1")
        out[f"append_{m}_then_find_ms"] = round((time.perf_counter() - t) * 1e3, 3)
        out[f"append_{m}_stats"] = {k: (round(v, 3) if isinstance(v, float) else v) for k, v in ix.stats().items()}
    ix.close()
    # predict: a model trained on a small app with the same ids, serving from this file
    small = "Small"
    s.import_events(small, [dict(event="$set", entityType="user", entityId=f"u{k}", eventTime=t0.isoformat())
                            for k in range(2000)] +
                    [dict(event="$set", entityType="item", entityId=f"i{k}", eventTime=t0.isoformat(),
                          properties={"categories": [f"c{k % 20}"]}) for k in range(500)] +
                    [dict(event="rate", entityType="user", entityId=f"u{k % 2000}", targetEntityType="item",
                          targetEntityId=f"i{(k * 7919) % 500}", properties={"rating": float(k % 5 + 1)},
                          eventTime=t0.isoformat()) for k in range(40000)])
    eng = ec.ECommerceRecommendationEngine().apply()
    params = {"appName": small, "unseenOnly": True, "seenEvents": ["buy", "view"], "similarEvents": ["view"],
              "rank": 10, "numIterations": 5, "lambda": 0.01, "seed": 3}
    ep = eng.jValueToEngineParams({"datasource": {"params": {"appName": small}},
                                   "algorithms": [{"name": "ecomm", "params": params}]})
    sc = w.WorkflowContext()
    model = eng.prepareDeploy(sc, ep, "bench", eng.train(sc, ep, "bench"))[0]
    ap = ep.algorithmParamsList[0][1]
    ap.appName = app
    algo = ec.ECommAlgorithm(ap)
    s.import_events(app, [dict(event="view", entityType="user", entityId=f"new{k}", targetEntityType="item",
                               targetEntityId=f"i{k % 500}", eventTime=t0.isoformat()) for k in range(200)])
    algo.predict(model, ec.Query(user="u0", num=10))   # builds the indexes
    for name, users in (("known_user", [f"u{k}" for k in range(200)]), ("unknown_user_recent", [f"new{k}" for k in
                                                                                                range(200)])):
        ts = []
        for u in users:
            t = time.perf_counter()
            algo.predict(model, ec.Query(user=u, num=10))
            ts.append(time.perf_counter() - t)
        out[f"predict_{name}_ms"] = {"p50": round(pct(ts, 50), 3), "p99": round(pct(ts, 99), 3)}
    for v in algo._indexes.values():
        v.close()
    p.unlink()
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--sizes", default="2000000,20000000")
    ap.add_argument("--finds", type=int, default=1000)
    ap.add_argument("--host-lines", type=int, default=100_000)
    args = ap.parse_args()
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                         text=True).stdout.strip().splitlines()
    res = {"gpu": gpu[0] if gpu else None, "sizes": []}
    with tempfile.TemporaryDirectory() as d:
        tmp = Path(d)
        os.environ["PIO_EVENTDATA_DIR"] = str(tmp / "host")
        p = s.app_file("Host")
        p.parent.mkdir(parents=True)
        write_file(p, args.host_lines, 1)
        t = time.perf_counter()
        s.LEventStore.findByEntity("Host", "user", "u1", eventNames=["buy", "view"], targetEntityType="item")
        res["host_findByEntity_us_per_event"] = round((time.perf_counter() - t) / args.host_lines * 1e6, 2)
        for n in (int(x) for x in args.sizes.split(",")):
            res["sizes"].append(one_size(n, args, tmp))
    print(json.dumps(res))


if __name__ == "__main__":
    main()
