#!/usr/bin/env python
"""Training of the complementary purchase template on the GPU (pio_assoc_train, DESIGN.md 4.15), per phase and end to
end, against the plain-Python restatement (tests/assoc_ref.py) on a subsample.

Workload, seeded: about 1 M users and 100 k items with Zipf-skewed popularity; sessions of 2 to 5 buys, 0 to 3 minutes
apart, on random days of a year, so that consecutive sessions of a user are days apart.  Parameters are the doc's
engine.json (basketWindow 120, minBasketSize 2, maxNumRulesPerCond 5) with maxRuleLength --length (3), minSupport
--min-support (1e-5; the doc's 0.1 keeps no set of this workload) and minConfidence / minLift --min-confidence /
--min-lift (0: every rule of a frequent set is scored and ranked; the items of this workload are independent, so the
doc's 0.6 / 1.0 keep none).

Reported, each a host clock around work that ends in a device synchronise:
  - for each --events size (10 M and 100 M): native.assoc_train from arrays, --rounds times, with its phases
    (native.assoc_train_timing) and the model's size;
  - end to end from an event file for the first size: DataSource.readTraining (the GPU scan) + Algorithm.train;
  - assoc_ref.train on a --sample-event subsample, and the device on the same subsample, whose models must be equal.
Also the card's name and power limit.

    python tools/assoc_bench.py [--events 10000000 100000000] [--users 1000000] [--items 100000] [--rounds 3]
"""
import argparse
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
sys.path.insert(0, str(ROOT / "tests"))
import pio_b200  # noqa: E402,F401
from pio_b200 import native  # noqa: E402


def card():
    out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True, timeout=30, check=True).stdout.strip().splitlines()
    if not out:
        raise RuntimeError("nvidia-smi reported no GPU")
    return out[0]


def buys(n, n_users, n_items, seed):
    """(user, item, t_ms) of about n seeded buys, in random order."""
    rng = np.random.default_rng(seed)
    size = rng.integers(2, 6, n // 3 + 1)
    size = size[:np.searchsorted(np.cumsum(size), n) + 1]
    ns = size.shape[0]
    user = rng.integers(0, n_users, ns)
    start = (rng.integers(0, 365, ns) * 86_400_000 + rng.integers(0, 86_400_000, ns)
             + 1_609_459_200_000)                                       # 2021-01-01
    su = np.repeat(user, size)
    first = np.repeat(np.cumsum(size) - size, size)
    gap = rng.integers(0, 181, su.shape[0]) * 1000
    gap[first] = 0
    csum = np.cumsum(gap)
    t = np.repeat(start, size) + csum - csum[first]
    item = (rng.zipf(1.3, su.shape[0]) - 1) % n_items
    perm = rng.permutation(su.shape[0])[:n]
    return su[perm].astype(np.int32), item[perm].astype(np.int32), t[perm].astype(np.int64)


def train(u, i, t, n_users, n_items, p):
    t0 = time.perf_counter()
    out = native.assoc_train(u, i, t, n_users, n_items, p["basketWindow"], p["maxRuleLength"], p["minSupport"],
                             p["minConfidence"], p["minLift"], p["minBasketSize"], p["maxNumRulesPerCond"])
    return time.perf_counter() - t0, out


def write_events(path, u, i, t):
    stamp = np.datetime_as_string(t.astype("datetime64[ms]"), unit="ms")
    path.parent.mkdir(parents=True, exist_ok=True)
    with open(path, "w") as fh:
        step = 1_000_000
        for a in range(0, u.shape[0], step):
            fh.write("".join(
                f'{{"event":"buy","entityType":"user","entityId":"u{x}","targetEntityType":"item",'
                f'"targetEntityId":"i{y}","eventTime":"{z}Z"}}\n'
                for x, y, z in zip(u[a:a + step].tolist(), i[a:a + step].tolist(), stamp[a:a + step].tolist())))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--events", type=int, nargs="+", default=[10_000_000, 100_000_000])
    ap.add_argument("--users", type=int, default=1_000_000)
    ap.add_argument("--items", type=int, default=100_000)
    ap.add_argument("--length", type=int, default=3)
    ap.add_argument("--min-support", type=float, default=1e-5)
    ap.add_argument("--min-confidence", type=float, default=0.0)
    ap.add_argument("--min-lift", type=float, default=0.0)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--sample-events", type=int, default=300_000)
    ap.add_argument("--no-file", action="store_true")
    a = ap.parse_args()
    p = {"basketWindow": 120, "maxRuleLength": a.length, "minSupport": a.min_support, "minConfidence": a.min_confidence,
         "minLift": a.min_lift, "minBasketSize": 2, "maxNumRulesPerCond": 5}
    print(f"card: {card()}")
    print(f"params: {json.dumps(p)}")
    native.lib()
    train(*buys(10_000, 1000, 100, 0), 1000, 100, p)     # warm-up: context, allocator
    for n in a.events:
        u, i, t = buys(n, a.users, a.items, n)
        for r in range(a.rounds):
            sec, out = train(u, i, t, a.users, a.items, p)
            tm = native.assoc_train_timing()
            phases = {k: round(v, 1) for k, v in tm.items() if k.endswith("_ms")}
            print(f"events {n}: round {r}: {sec * 1e3:.1f} ms wall; phases {phases}; baskets {tm['baskets']}, "
                  f"transactions {tm['transactions']}, candidates {tm['candidates']}; sets "
                  f"{np.diff(out['level_off']).tolist()}, rules {out['rule_cond'].shape[0]}", flush=True)
        del u, i, t
    # end to end from an event file: the GPU scan of the buys, the id numbering and the training
    if not a.no_file:
        n = a.events[0]
        u, i, t = buys(n, a.users, a.items, n)
        tmp = Path(tempfile.mkdtemp(prefix="assoc_bench_"))
        try:
            os.environ["PIO_EVENTDATA_DIR"] = str(tmp / "events")
            from pio_b200 import storage as s
            from pio_b200 import workflow as w
            from pio_b200.templates import complementarypurchase as cp
            t0 = time.perf_counter()
            write_events(s.app_file("Bench"), u, i, t)
            print(f"event file: {n} buys written in {time.perf_counter() - t0:.1f} s "
                  f"({s.app_file('Bench').stat().st_size / 1e9:.2f} GB)", flush=True)
            sc = w.WorkflowContext()
            algo = cp.Algorithm(cp.AlgorithmParams(**p))
            for r in range(a.rounds):
                t0 = time.perf_counter()
                td = cp.DataSource(cp.DataSourceParams("Bench")).readTraining(sc)
                t1 = time.perf_counter()
                model = algo.train(sc, td)
                t2 = time.perf_counter()
                tm = native.assoc_train_timing()
                print(f"end to end {n}: round {r}: readTraining {(t1 - t0) * 1e3:.0f} ms, train {(t2 - t1) * 1e3:.0f} ms "
                      f"(assoc_train {tm['total_ms']:.0f} ms), total {(t2 - t0) * 1e3:.0f} ms; rules "
                      f"{model.rule_cond.shape[0]}", flush=True)
        finally:
            shutil.rmtree(tmp, ignore_errors=True)
    # the restatement on a subsample, and the device on the same events
    import assoc_ref as ref
    u, i, t = buys(a.sample_events, a.users, a.items, 7)
    sec_dev, got = train(u, i, t, a.users, a.items, p)
    t0 = time.perf_counter()
    want = ref.flat(*ref.train(list(zip(u.tolist(), i.tolist(), t.tolist())), **p))
    sec_ref = time.perf_counter() - t0
    same = all(got[k].tolist() == list(want[k]) for k in native.ASSOC_ARRAYS)
    print(f"subsample {a.sample_events}: assoc_ref {sec_ref * 1e3:.0f} ms, device {sec_dev * 1e3:.1f} ms, "
          f"models equal: {same}", flush=True)
    if not same:
        raise SystemExit("the device model differs from the restatement")


if __name__ == "__main__":
    main()
