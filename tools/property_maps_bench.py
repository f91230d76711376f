"""Time PEventStore.aggregatePropertyMaps("user") and ("item") on the GPU, split into the whole-map scan calls, the
fold and the rest (file read, merge and the host materialisation of the PropertyMaps), against aggregateProperties
(one json.loads per line) timed on a prefix of the same file and extrapolated per line.

The file is tools/properties_bench.py's: generated from a seed, n_users user $set events, n_items item $set events with
"categories", and n_views view events, in a seeded order.  Prints one JSON line with the card's name and power limit.

    python tools/property_maps_bench.py [--users 1000000] [--items 100000] [--views 20000000] [--host-lines 200000]
"""
import argparse
import json
import os
import subprocess
import sys
import tempfile
import time
from pathlib import Path

sys.path.insert(0, str(Path(__file__).resolve().parent.parent))
sys.path.insert(0, str(Path(__file__).resolve().parent))
import pio_b200  # noqa: E402,F401
from pio_b200 import native  # noqa: E402
from pio_b200 import storage as s  # noqa: E402
from properties_bench import timed, write_file  # noqa: E402


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
    out = {"gpu": gpu}
    with tempfile.TemporaryDirectory() as d:
        os.environ["PIO_EVENTDATA_DIR"] = d
        path = s.app_file("Bench")
        path.parent.mkdir(parents=True, exist_ok=True)
        _, gen_s = timed(lambda: write_file(path, args.users, args.items, args.views, args.seed), "generate")
        n_lines = args.users + args.items + args.views
        out.update(lines=n_lines, file_bytes=path.stat().st_size, generate_s=round(gen_s, 1))
        timed(lambda: s.PEventStore.aggregatePropertyMaps("Bench", "item"), "warm-up")   # module load, page cache
        spent = {}   # time inside the native calls, per name
        for name in ("events_scan_props", "events_fold_props"):
            def wrap(f, name=name):
                def g(*a, **k):
                    t0 = time.perf_counter()
                    try:
                        return f(*a, **k)
                    finally:
                        spent[name] = spent.get(name, 0.0) + time.perf_counter() - t0
                return g
            setattr(native, name, wrap(getattr(native, name)))
        dev = {}
        for et in ("user", "item"):
            spent.clear()
            maps, t = timed(lambda: s.PEventStore.aggregatePropertyMaps("Bench", et), et)
            scan, fold = spent.get("events_scan_props", 0.0), spent.get("events_fold_props", 0.0)
            dev[et] = {"total_s": round(t, 2), "scan_calls_s": round(scan, 2), "fold_s": round(fold, 3),
                       "read_merge_materialise_s": round(t - scan - fold, 2), "n_maps": len(maps)}
        out["device"] = dev
        prefix = s.app_file("Prefix")
        k = min(args.host_lines, n_lines)
        with open(path, "rb") as src, open(prefix, "wb") as dst:
            for _ in range(k):
                dst.write(src.readline())
        host = {"prefix_lines": k}
        for et in ("user", "item"):
            _, t = timed(lambda: s.PEventStore.aggregateProperties("Prefix", et), f"host prefix {et}")
            host[et] = {"prefix_s": round(t, 2), "us_per_line": round(t / k * 1e6, 2),
                        "extrapolated_s": round(t / k * n_lines, 1)}
        out["host"] = host
    print(json.dumps(out))


if __name__ == "__main__":
    main()
