"""Time the similarproduct template's DataSource.readTraining from event columns on the GPU, split into the keyed scans,
the folds, the view-event scan and the host materialisation of the training data, against the host path
(aggregateProperties + find, one json.loads per line) timed on a prefix of the same file and extrapolated per event.

The file is generated from a seed: n_users user $set events, n_items item $set events with "categories", and n_views
view events, in a seeded order.  Prints one JSON line with the card's name and power limit.

    python tools/properties_bench.py [--users 1000000] [--items 100000] [--views 20000000] [--host-lines 200000]
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

sys.path.insert(0, str(Path(__file__).resolve().parent.parent))
import pio_b200  # noqa: E402,F401
from pio_b200 import native  # noqa: E402
from pio_b200 import storage as s  # noqa: E402
from pio_b200.templates import similarproduct as sp  # noqa: E402


def write_file(path, n_users, n_items, n_views, seed):
    rng = np.random.default_rng(seed)
    kinds = np.concatenate([np.zeros(n_users, np.int8), np.ones(n_items, np.int8), np.full(n_views, 2, np.int8)])
    rng.shuffle(kinds)
    vu, vi = rng.integers(0, n_users, n_views).tolist(), rng.integers(0, n_items, n_views).tolist()
    t0 = np.datetime64("2015-01-01T00:00:00", "s")
    times = np.datetime_as_string(t0 + rng.integers(0, 10 ** 8, kinds.shape[0]).astype("timedelta64[s]"),
                                  unit="s").tolist()
    cats = ['["c%d"]' % k for k in range(20)] + ['["c1", "c2"]', "null"]
    cat_pick = rng.integers(0, len(cats), n_items).tolist()
    nu = ni = nv = 0
    with open(path, "w") as f:
        buf = []
        for j, k in enumerate(kinds.tolist()):
            t = times[j]
            if k == 0:
                buf.append(f'{{"event": "$set", "entityType": "user", "entityId": "u{nu}", "properties": {{}}, '
                           f'"eventTime": "{t}Z"}}\n')
                nu += 1
            elif k == 1:
                buf.append(f'{{"event": "$set", "entityType": "item", "entityId": "i{ni}", "properties": '
                           f'{{"categories": {cats[cat_pick[ni]]}}}, "eventTime": "{t}Z"}}\n')
                ni += 1
            else:
                buf.append(f'{{"event": "view", "entityType": "user", "entityId": "u{vu[nv]}", "targetEntityType": '
                           f'"item", "targetEntityId": "i{vi[nv]}", "properties": {{}}, "eventTime": "{t}Z"}}\n')
                nv += 1
            if len(buf) >= 1 << 16:
                f.write("".join(buf))
                buf = []
        f.write("".join(buf))


def timed(fn, what=""):
    t0 = time.perf_counter()
    out = fn()
    dt = time.perf_counter() - t0
    if what:
        print(f"{what}: {dt:.2f} s", file=sys.stderr, flush=True)
    return out, dt


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--users", type=int, default=1_000_000)
    ap.add_argument("--items", type=int, default=100_000)
    ap.add_argument("--views", type=int, default=20_000_000)
    ap.add_argument("--host-lines", type=int, default=200_000, help="prefix of the file timed on the host path")
    ap.add_argument("--seed", type=int, default=1)
    args = ap.parse_args()
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                         text=True).stdout.strip().splitlines()
    with tempfile.TemporaryDirectory() as d:
        os.environ["PIO_EVENTDATA_DIR"] = d
        path = s.app_file("Bench")
        path.parent.mkdir(parents=True, exist_ok=True)
        _, gen_s = timed(lambda: write_file(path, args.users, args.items, args.views, args.seed), "generate")
        n_lines = args.users + args.items + args.views

        class Ctx:
            device = 0
        ds = sp.DataSource(sp.DataSourceParams(appName="Bench"))
        timed(lambda: ds.readTraining(Ctx()), "warm-up readTraining")   # module load, allocator, page cache
        # time spent inside the native calls, summed per name (the device work of each step)
        spent = {}
        for name in ("events_scan_keys", "events_scan", "events_fold", "ids_encode"):
            def wrap(f, name=name):
                def g(*a, **k):
                    t0 = time.perf_counter()
                    try:
                        return f(*a, **k)
                    finally:
                        spent[name] = spent.get(name, 0.0) + time.perf_counter() - t0
                return g
            setattr(native, name, wrap(getattr(native, name)))
        # the calls readTraining makes, one by one, then the materialisation the algorithms need
        users, t_users = timed(lambda: s.PEventStore.aggregatePropertyColumns("Bench", "user", ["categories"], sc=Ctx()),
                               "users")
        in_users = dict(spent)
        items, t_items = timed(lambda: s.PEventStore.aggregatePropertyColumns("Bench", "item", ["categories"], sc=Ctx()),
                               "items")
        in_agg = dict(spent)
        views, t_views = timed(lambda: s.PEventStore.findColumns("Bench", entityType="user",
                                                                 eventNames=["view", "like", "dislike"],
                                                                 targetEntityType="item", sc=Ctx()), "views")
        c = s.EntityEventColumns(users, items, views, 0)

        def materialise():
            c.user_map(), c.item_map(), sp._item_index(c), c.event_users(), c.event_items(), c.millis()
        _, t_mat = timed(materialise, "materialise")
        _, t_read = timed(lambda: ds.readTraining(Ctx()), "readTraining")
        file_bytes = path.stat().st_size
        # host path on a prefix, extrapolated per line
        prefix = s.app_file("Prefix")
        with open(path, "rb") as src, open(prefix, "wb") as dst:
            for _ in range(min(args.host_lines, n_lines)):
                dst.write(src.readline())

        def host_read():
            users_h = {k: sp.User() for k, _ in s.PEventStore.aggregateProperties("Prefix", "user")}
            items_h = {k: sp.Item(categories=pm.getOpt("categories"))
                       for k, pm in s.PEventStore.aggregateProperties("Prefix", "item")}
            evs = s.PEventStore.find("Prefix", entityType="user", eventNames=["view", "like", "dislike"],
                                     targetEntityType="item")
            return users_h, items_h, evs
        _, t_host = timed(host_read, "host prefix")
        host_per_line = t_host / min(args.host_lines, n_lines)
    print(json.dumps({
        "gpu": gpu, "lines": n_lines, "file_bytes": file_bytes, "generate_s": round(gen_s, 1),
        "device": {"aggregate_users_s": round(t_users, 2), "aggregate_items_s": round(t_items, 2),
                   "users_keyed_scan_s": round(in_users.get("events_scan_keys", 0.0), 2),
                   "users_fold_s": round(in_users.get("events_fold", 0.0), 3),
                   "items_keyed_scan_s": round(in_agg.get("events_scan_keys", 0.0) -
                                               in_users.get("events_scan_keys", 0.0), 2),
                   "items_fold_s": round(in_agg.get("events_fold", 0.0) - in_users.get("events_fold", 0.0), 3),
                   "find_views_s": round(t_views, 2), "host_materialise_s": round(t_mat, 2),
                   "of_which_ids_encode_s": round(spent.get("ids_encode", 0.0) - in_agg.get("ids_encode", 0.0), 3),
                   "readTraining_s": round(t_read, 2),
                   "n_users": len(users), "n_items": len(items), "n_view_events": len(views)},
        "host": {"prefix_lines": min(args.host_lines, n_lines), "prefix_s": round(t_host, 2),
                 "us_per_line": round(host_per_line * 1e6, 2),
                 "extrapolated_readTraining_s": round(host_per_line * n_lines, 1)},
    }))


if __name__ == "__main__":
    main()
