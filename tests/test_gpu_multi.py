"""Multi-GPU parity (-m gpu, needs >= 2 H100s; skipped otherwise): row-sharded training with the NCCL factor
all-gather gives bit-identical factors to the single-GPU run (every row's arithmetic is independent of the
sharding), and therefore the same parity with the oracle."""
import os
import socket
import subprocess
import sys
import textwrap
from pathlib import Path

import numpy as np
import pytest

pytestmark = pytest.mark.gpu
ROOT = Path(__file__).resolve().parent.parent

WORKER = textwrap.dedent("""
    import os, sys
    sys.path.insert(0, {root!r})
    import numpy as np, torch, torch.distributed as dist
    import pio_b200
    from pio_b200 import native, synth
    rank, world = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"])
    torch.cuda.set_device(rank)
    dist.init_process_group("nccl", device_id=torch.device("cuda", rank))
    def fresh_id():      # one ncclUniqueId per communicator (= per handle)
        t = torch.zeros(128, dtype=torch.uint8, device="cuda")
        if rank == 0:
            t = torch.tensor(list(native.nccl_unique_id()), dtype=torch.uint8, device="cuda")
        dist.broadcast(t, 0)
        return bytes(t.cpu().tolist())
    # (rank, implicit, users, items, ratings, PIO_ALS_TC, dedup, sharded input): rank 64 runs the pair kernel (mma.sync +
    # lockstep Cholesky) or, with PIO_ALS_TC=1, the wgmma kernel; the 30-item cases have heavy item rows (parts + finish
    # kernels); rank 128 runs the FP32 Gramian + lockstep finish path.  sharded: every rank passes only its slice of the
    # events (pio_als_set_ratings_coo_sharded) -- the result must still be bit-identical to the single-GPU run.
    cases = ((64, True, 6000, 900, 150000, "", 1, False), (10, False, 3000, 500, 40000, "", 0, False),
             (64, True, 20000, 30, 300000, "", 1, False), (64, True, 20000, 30, 300000, "1", 1, False),
             (64, True, 6000, 900, 150000, "", 1, True), (10, False, 3000, 500, 40000, "", 0, True),
             (12, False, 3000, 500, 60000, "", 2, True), (128, True, 4000, 300, 80000, "", 1, True),
             (64, True, 20000, 30, 300000, "", 1, True))
    for (rk, implicit, nu, ni, nnz, tc, dd, sharded) in cases:
        os.environ.pop("PIO_ALS_TC", None)
        if tc:
            os.environ["PIO_ALS_TC"] = tc
        u, i, r = synth.synth_ratings(nu, ni, nnz, seed=3, implicit=implicit)
        ts = np.random.default_rng(7).integers(0, 1000, nnz).astype(np.int64) if dd == 2 else None
        u0 = synth.synth_init_factors(nu, rk, 5, 0)
        m = native.NativeALS(rk, nu, ni, lam=0.01, implicit=implicit, device=rank, world_size=world, world_rank=rank,
                             nccl_id=fresh_id())
        if sharded:
            # uneven slices, one of them empty when there are more than two ranks
            cuts = [0] + [int(nnz * f) for f in np.linspace(0.3, 1.0, world)]
            if world > 2:
                cuts[2] = cuts[1]
            lo, hi = cuts[rank], cuts[rank + 1]
            m.set_ratings_sharded(u[lo:hi], i[lo:hi], r[lo:hi], dedup=dd, ts=None if ts is None else ts[lo:hi])
        else:
            m.set_ratings(u, i, r, dedup=dd, ts=ts)
        m.set_init(u0)
        m.run(3)
        uf, itf, uh, ih = m.get_factors()
        if rank == 0:
            s = native.NativeALS(rk, nu, ni, lam=0.01, implicit=implicit, device=0)
            s.set_ratings(u, i, r, dedup=dd, ts=ts)
            s.set_init(u0)
            s.run(3)
            suf, sitf, suh, sih = s.get_factors()
            assert m.stats()["nnz"] == s.stats()["nnz"]
            du, di = float(np.abs(uf - suf).max()), float(np.abs(itf - sitf).max())
            assert np.array_equal(uf, suf) and np.array_equal(itf, sitf), (
                "sharded != single GPU: rank %d implicit %s sharded-input %s: max |du| %.3g (%d rows differ), max |di| %.3g (%d rows differ)"
                % (rk, implicit, sharded, du, int((uf != suf).any(1).sum()), di, int((itf != sitf).any(1).sum())))
            assert np.array_equal(uh, suh) and np.array_equal(ih, sih)
            assert m.stats()["last_comm_ms"] > 0
        dist.barrier()
        m.close()
    dist.destroy_process_group()
    print("rank", rank, "ok")
""")


def test_sharded_equals_single_gpu(native, tmp_path):
    n = native.device_count()
    if n < 2:
        pytest.skip("needs >= 2 GPUs")
    world = 2 if n < 4 else 4
    script = tmp_path / "worker.py"
    script.write_text(WORKER.format(root=str(ROOT)))
    with socket.socket() as s:
        s.bind(("127.0.0.1", 0))
        port = s.getsockname()[1]
    out = subprocess.run([sys.executable, "-m", "torch.distributed.run", "--nnodes=1", f"--nproc-per-node={world}",
                          "--master-addr", "127.0.0.1", "--master-port", str(port), str(script)],
                         capture_output=True, text=True, timeout=600)
    assert out.returncode == 0, out.stdout[-3000:] + out.stderr[-6000:]
    assert out.stdout.count("ok") == world
