"""Event ingest measurement: the recommendation template's DataSource on a seeded JSON-lines event file, host path
versus the device scanner (PEventStore.findColumns + ids_encode).

    python tools/events_bench.py [--events N] [--host-events M] [--dir DIR]

The file is generated vectorised (fixed-width lines, 30 % buy events, the rest rate events with a rating) into a
temporary directory and removed afterwards.  The host path (find -> Rating -> BiMap.stringInt -> np.fromiter) runs on
the first M events and is extrapolated to N, and labelled so.  The device path runs on the whole file, once with the
shared-memory parse kernel and once with the global-memory one, and is split into file read, the scan calls (within
them: host copy into pinned staging, host-to-device copy, kernels and device-to-host copy, from pio_events_debug_timing),
ids_encode and the COO build.
Prints one JSON object, with the card name, power limit and CPU model of the same run."""
import argparse
import json
import os
import subprocess
import sys
import tempfile
import time
from pathlib import Path

import numpy as np

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))
import pio_b200  # noqa: E402,F401
from pio_b200 import native, storage as s  # noqa: E402

W_ID = 8


def template_line():
    return (b'{"event": "rate", "entityType": "user", "entityId": "u' + b"0" * W_ID + b'", "targetEntityType": "item", '
            b'"targetEntityId": "i' + b"0" * W_ID + b'", "properties": {"rating": 0}, '
            b'"eventTime": "2021-03-04T05:06:07.000000+00:00"}\n')


def write_file(path: Path, n: int, seed: int, block: int = 1 << 20):
    tl = template_line()
    L = len(tl)
    row = np.frombuffer(tl, np.uint8)
    p_u = tl.index(b'"u0') + 2
    p_i = tl.index(b'"i0') + 2
    p_r = tl.index(b'"rating": ') + 10
    p_f = tl.index(b".000000") + 1
    p_ev = tl.index(b'"rate"')
    rng = np.random.default_rng(seed)
    with open(path, "wb") as fh:
        for b0 in range(0, n, block):
            m = min(block, n - b0)
            a = np.tile(row, (m, 1))
            u = rng.zipf(1.3, m) % 2_000_000
            it = rng.zipf(1.2, m) % 500_000
            for base, v in ((p_u, u), (p_i, it)):
                for k in range(W_ID):
                    a[:, base + k] = 48 + (v // 10 ** (W_ID - 1 - k)) % 10
            a[:, p_r] = 48 + rng.integers(1, 6, m)
            us = np.arange(b0, b0 + m) % 1_000_000
            for k in range(6):
                a[:, p_f + k] = 48 + (us // 10 ** (5 - k)) % 10
            buy = rng.random(m) < 0.3
            a[buy, p_ev:p_ev + 6] = np.frombuffer(b'"buy" ', np.uint8)   # same width: a space before the comma
            fh.write(a.tobytes())
    return L


def host_path(app):
    from pio_b200.templates import recommendation as rec
    t0 = time.perf_counter()
    out = []
    for e in s.PEventStore.find(appName=app, entityType="user", eventNames=["rate", "buy"], targetEntityType="item"):
        out.append(rec.Rating(e.entityId, e.targetEntityId, e.properties.get("rating", float) if e.event == "rate" else 4.0))
    t1 = time.perf_counter()
    um = s.BiMap.stringInt(r.user for r in out)
    im = s.BiMap.stringInt(r.item for r in out)
    n = len(out)
    np.fromiter((um(r.user) for r in out), np.int32, n)
    np.fromiter((im(r.item) for r in out), np.int32, n)
    np.fromiter((r.rating for r in out), np.float32, n)
    return n, t1 - t0, time.perf_counter() - t1


def machine():
    info = {}
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                           text=True, timeout=30).stdout.strip().splitlines()
        info["gpu"], info["power_limit"] = [x.strip() for x in q[0].split(",")]
    except Exception as e:  # noqa: BLE001
        info["gpu"] = f"unknown ({e})"
    try:
        info["cpu"] = next(ln.split(":", 1)[1].strip() for ln in open("/proc/cpuinfo") if ln.startswith("model name"))
    except Exception:  # noqa: BLE001
        info["cpu"] = "unknown"
    return info


def h2d_gbs():
    import torch
    x = torch.empty(1 << 30, dtype=torch.uint8).pin_memory()
    y = torch.empty_like(x, device="cuda")
    y.copy_(x, non_blocking=True)
    torch.cuda.synchronize()
    t = time.perf_counter()
    for _ in range(5):
        y.copy_(x, non_blocking=True)
    torch.cuda.synchronize()
    return 5 * x.numel() / (time.perf_counter() - t) / 1e9


def device_path(n_events, nbytes, t_read):
    """findColumns -> ids_encode -> COO on the whole file, split into its phases."""
    split = {"h2d_ms": 0.0, "kernel_ms": 0.0, "d2h_ms": 0.0, "stage_ms": 0.0, "chunks": 0}
    t_scan = [0.0]
    orig = native.events_scan

    def timed(*args, **kw):
        t0 = time.perf_counter()
        r = orig(*args, **kw)
        t_scan[0] += time.perf_counter() - t0
        for k, v in native.events_scan_timing().items():
            split[k] += v
        return r
    native.events_scan = timed
    t = time.perf_counter()
    try:
        cols = s.PEventStore.findColumns("Big", entityType="user", eventNames=["rate", "buy"], targetEntityType="item",
                                         property="rating")
    finally:
        native.events_scan = orig
    t_find = time.perf_counter() - t
    t = time.perf_counter()
    u, uf = native.ids_encode(cols.entityId)
    i, itf = native.ids_encode(cols.targetEntityId)
    t_ids = time.perf_counter() - t
    t = time.perf_counter()
    v = np.where(cols.code == 0, cols.value, 4.0).astype(np.float32)
    users = s.string_list(s.take_strings(*cols.entityId, uf))
    items = s.string_list(s.take_strings(*cols.targetEntityId, itf))
    t_coo = time.perf_counter() - t
    assert len(cols) == n_events and cols.n_fallback == 0 and v.shape[0] == n_events
    k_s = split["kernel_ms"] / 1e3
    return {
        "file_read_s": t_read, "find_columns_s": t_find, "scan_calls_s": t_scan[0],
        "scan_h2d_s": split["h2d_ms"] / 1e3, "scan_kernels_s": k_s, "scan_d2h_s": split["d2h_ms"] / 1e3,
        "scan_pinned_staging_s": split["stage_ms"] / 1e3, "device_chunks": split["chunks"],
        "h2d_GB_per_s": nbytes / max(split["h2d_ms"] / 1e3, 1e-9) / 1e9, "kernel_GB_per_s": nbytes / k_s / 1e9,
        "ids_encode_s": t_ids, "coo_and_maps_s": t_coo, "n_users": len(users), "n_items": len(items),
        "scan_events_per_s": n_events / t_scan[0], "scan_GB_per_s": nbytes / t_scan[0] / 1e9,
        "find_columns_events_per_s": n_events / t_find, "total_s": t_find + t_ids + t_coo,
    }


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--events", type=int, default=20_000_000)
    ap.add_argument("--host-events", type=int, default=1_000_000)
    ap.add_argument("--dir", default=None)
    a = ap.parse_args()
    res = {"machine": machine()}
    with tempfile.TemporaryDirectory(dir=a.dir) as d:
        os.environ["PIO_EVENTDATA_DIR"] = d
        L = write_file(s.app_file("Big"), a.events, 1)
        write_file(s.app_file("Small"), a.host_events, 1)
        nbytes = s.app_file("Big").stat().st_size
        res.update(events=a.events, file_bytes=nbytes, line_bytes=L)
        n, t_find, t_maps = host_path("Small")
        res["host"] = {"events_measured": n, "find_rating_s": t_find, "bimap_coo_s": t_maps,
                       "us_per_event": 1e6 * (t_find + t_maps) / n,
                       "extrapolated_s_for_file": (t_find + t_maps) / n * a.events, "label": "extrapolated"}
        # device path, phase by phase (the first call warms the library up)
        native.events_scan(b'{"event":"x","entityType":"y","entityId":"z","eventTime":"2021-01-01T00:00:00"}\n')
        t = time.perf_counter()
        with open(s.app_file("Big"), "rb") as fh:
            while fh.read(256 << 20):
                pass
        t_read = time.perf_counter() - t
        pcie = h2d_gbs()
        res["pcie_h2d_pinned_GB_per_s_measured"] = pcie
        res["hbm_GB_per_s_nominal"] = 3350.0
        for smem in ("1", "0"):      # the parse kernel with and without shared-memory staging of its lines
            os.environ["PIO_EVENTS_SMEM"] = smem
            res["device_smem" if smem == "1" else "device_global"] = device_path(a.events, nbytes, t_read)
        os.environ.pop("PIO_EVENTS_SMEM")
        res["device"] = res["device_smem"]
        res["speedup_vs_host_extrapolated"] = res["host"]["extrapolated_s_for_file"] / res["device"]["total_s"]
    print(json.dumps(res))


if __name__ == "__main__":
    main()
