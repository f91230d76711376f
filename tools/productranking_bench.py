#!/usr/bin/env python
"""pio_als_rank_lists (the product ranking template's predict on batches, DESIGN.md 4.17) on one GPU.

Model: imported factors (pio_als_model_import), rank 64, 1 M users x 100 k items, seeded; 2 % of the rows of each side
have no factor.  Workloads:
  A   16 384 queries, lists of 7 to 200 items with repeats and 5 % unknown ids (the tile path);
  A'  the same number of entries in lists of RL_TILE + 1 items (the radix path), to compare the two paths on lists of
      the same content;
  B   64 queries, lists of 50 k to 100 k items (the radix path);
  C   200 single-query calls with the doc's 7-item list: the latency a deployed predict pays (median).
Reported per workload, each a host clock around a call that ends in a device synchronise (best and median of the timed
rounds after a warm-up): the call time, entries per second, the factor bytes gathered (entries x rank x 4) over the time,
and the device milliseconds of pio_rank_lists_debug_stats.  Every timed output is checked byte for byte against
tests/productranking_ref.rank_lists, whose time on a prefix of A is the host baseline.  The card's name and power limit
are read in the same run.

    python tools/productranking_bench.py [--users 1000000] [--items 100000] [--rank 64] [--rounds 5] [--out DIR]
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
from pio_b200 import native  # noqa: E402
from tests import productranking_ref as ref  # noqa: E402


def card():
    out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True, timeout=30, check=True).stdout.strip().splitlines()
    if not out:
        raise RuntimeError("nvidia-smi reported no GPU")
    return out[0]


def lists(rng, n_users, n_items, lengths, unknown=0.05):
    users = rng.integers(0, n_users, len(lengths)).astype(np.int32)
    ptr = np.concatenate([[0], np.cumsum(lengths)]).astype(np.int64)
    items = rng.integers(0, n_items, int(ptr[-1])).astype(np.int32)
    items[rng.random(items.shape[0]) < unknown] = -1
    rep = rng.random(items.shape[0]) < 0.05                      # repeats of the entry before
    rep[ptr[:-1]] = False
    items[rep] = items[np.flatnonzero(rep) - 1]
    return users, ptr, items


def timed(h, batch, rounds):
    h.rank_lists(*batch)                                       # warm-up of this shape
    ts, dev = [], []
    for _ in range(rounds):
        t0 = time.perf_counter()
        out = h.rank_lists(*batch)
        ts.append(time.perf_counter() - t0)
        dev.append(native.rank_lists_stats()["device_ms"])
    return out, ts, dev


def report(name, batch, ts, dev, rank, stats):
    entries = int(batch[1][-1])
    best, med = min(ts), float(np.median(ts))
    return {"workload": name, "queries": int(batch[0].shape[0]), "entries": entries, "best_ms": best * 1e3,
            "median_ms": med * 1e3, "device_ms_median": float(np.median(dev)), "entries_per_s": entries / best,
            "gathered_GB_per_s": entries * rank * 4 / best / 1e9, "tile_queries": stats["tile_queries"],
            "radix_queries": stats["radix_queries"], "parts": stats["parts"]}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--users", type=int, default=1_000_000)
    ap.add_argument("--items", type=int, default=100_000)
    ap.add_argument("--rank", type=int, default=64)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--seed", type=int, default=11)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    info = card()
    rng = np.random.default_rng(a.seed)
    uf = rng.standard_normal((a.users, a.rank), np.float32)
    itf = rng.standard_normal((a.items, a.rank), np.float32)
    uh = (rng.random(a.users) >= 0.02).astype(np.uint8)
    ih = (rng.random(a.items) >= 0.02).astype(np.uint8)
    h = native.NativeALS.from_factors(uf, itf, uh, ih)
    f = (uf, uh, itf, ih)
    work = {
        "A": lists(rng, a.users, a.items, rng.integers(7, 201, 16384)),
        "B": lists(rng, a.users, a.items, rng.integers(50_000, 100_001, 64)),
    }
    n_a = int(work["A"][1][-1])
    work["A_radix"] = lists(rng, a.users, a.items, [ref.TILE + 1] * (n_a // (ref.TILE + 1)))
    results, ok = [], True
    for name, batch in work.items():
        out, ts, dev = timed(h, batch, a.rounds)
        st = native.rank_lists_stats()
        want = ref.rank_lists(*f, *batch)
        same = (np.array_equal(out[0], want[0]) and np.array_equal(out[1].view(np.uint64), want[1].view(np.uint64))
                and np.array_equal(out[2], want[2]))
        ok &= same
        results.append(dict(report(name, batch, ts, dev, a.rank, st), equal_to_restatement=same))
    # C: one 7-item query per call, as a deployed predict sends it
    one = lists(rng, a.users, a.items, [7])
    h.rank_lists(*one)
    ts, same = [], True
    for k in range(200):
        batch = (np.array([(k * 7919) % a.users], np.int32), one[1], one[2])
        t0 = time.perf_counter()
        out = h.rank_lists(*batch)
        ts.append(time.perf_counter() - t0)
        want = ref.rank_lists(*f, *batch)
        same &= np.array_equal(out[0], want[0]) and np.array_equal(out[1].view(np.uint64), want[1].view(np.uint64))
    ok &= same
    results.append({"workload": "C", "queries": 1, "entries": 7, "calls": 200, "median_us": float(np.median(ts)) * 1e6,
                    "p90_us": float(np.percentile(ts, 90)) * 1e6, "equal_to_restatement": bool(same)})
    # the host baseline: the restatement on a prefix of A
    pre = 2048
    ua, pa, ia = work["A"]
    t0 = time.perf_counter()
    ref.rank_lists(*f, ua[:pre], pa[:pre + 1], ia[:pa[pre]])
    host_s = time.perf_counter() - t0
    results.append({"workload": "host restatement (A prefix)", "queries": pre, "entries": int(pa[pre]),
                    "ms": host_s * 1e3, "entries_per_s": int(pa[pre]) / host_s})
    doc = {"card": info, "users": a.users, "items": a.items, "rank": a.rank, "rounds": a.rounds, "results": results,
           "all_equal": bool(ok)}
    print(json.dumps(doc, indent=1))
    if a.out:
        Path(a.out).mkdir(parents=True, exist_ok=True)
        (Path(a.out) / "productranking_bench.json").write_text(json.dumps(doc, indent=1))
    h.close()
    return 0 if ok else 1


if __name__ == "__main__":
    sys.exit(main())
