"""Throughput of the lockstep Cholesky alone (debug entry pio_als_debug_lockstep): n dense systems, fill + solve
repeated `reps` times per matrix slot.  Run on the GPU box: python tools/bench_solver.py"""
import ctypes as C
import json
import sys
from pathlib import Path

import numpy as np

sys.path.insert(0, str(Path(__file__).resolve().parent.parent))
import pio_b200  # noqa: E402,F401
from pio_b200 import native  # noqa: E402


def main():
    out = {}
    for N, n in ((64, 132 * 24 * 4), (128, 132 * 6 * 4)):   # four waves of the 132 SMs of an H100
        rng = np.random.default_rng(0)
        Y = rng.standard_normal((64, 2 * N, N)).astype(np.float32)
        A = np.einsum("nri,nrj->nij", Y, Y).astype(np.float32)
        A = np.ascontiguousarray(np.resize(A, (n, N, N)))
        b = rng.standard_normal((n, N)).astype(np.float32)
        x = np.zeros((n, N), np.float32)
        ms, fail = C.c_float(0), C.c_int(0)
        f = native.lib().pio_als_debug_lockstep
        for reps in (1, 9):
            rc = f(C.c_int(0), C.c_int(N), C.c_int(n), A.ctypes.data_as(C.c_void_p), b.ctypes.data_as(C.c_void_p),
                   C.c_float(0.1), x.ctypes.data_as(C.c_void_p), C.c_int(reps), C.byref(ms), C.byref(fail))
            assert rc == 0
            out[f"N{N}_reps{reps}_ms"] = ms.value
        per = (out[f"N{N}_reps9_ms"] - out[f"N{N}_reps1_ms"]) / 8.0
        out[f"N{N}_solves_per_s"] = n / (per / 1e3)
        out[f"N{N}_us_per_1M_rows"] = per / n * 1e6 * 1e3
    print(json.dumps(out))


if __name__ == "__main__":
    main()
