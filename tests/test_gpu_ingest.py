"""GPU tests (-m gpu): the ALS rating ingest (pio_als.cu: dedup, degrees, renumbering, both CSR orientations, heavy-row
parts) read back with NativeALS.debug_side and held to tests/ingest_ref.py exactly: integers equal, ratings and ridge
counts equal as bits.  Every case asserts what makes it a boundary case (key widths, run lengths, distinct-pair counts,
heavy rows), so it fails if a change stops it from straddling its boundary."""
import ctypes as C

import numpy as np
import pytest

import halfstep_ref as H
import ingest_ref as ref
from pio_b200 import mllib, synth
from test_gpu_halfstep import ALPHA, ENV_VARS, LAM, TAU, check_rows

pytestmark = pytest.mark.gpu

I64_MIN, I64_MAX = np.iinfo(np.int64).min, np.iinfo(np.int64).max
WIDTHS = (1, 2, 255, 256, 257, 65536, 65537, (1 << 24) + 1)


@pytest.fixture(autouse=True)
def _default_switches(monkeypatch):
    for v in ENV_VARS:
        monkeypatch.delenv(v, raising=False)


def _handle(native, nu, ni, rank=10, implicit=False):
    return native.NativeALS(rank, nu, ni, lam=LAM, implicit=implicit, alpha=ALPHA, init_mode=native.INIT_HASH)


def assert_ingest(m, u, i, r, nu, ni, mode, ts=None, implicit=False, rank=10):
    """debug_side of both sides == the restatement; returns the restatement."""
    want = ref.ingest(u, i, r, nu, ni, mode, ts, implicit, 1, rank)
    for name in ("user", "item"):
        got = m.debug_side(name)
        bad = ref.differences(got, want[name][0])
        assert not bad, (name, mode, bad)
    return want


def ingest_case(native, u, i, r, nu, ni, mode, ts=None, implicit=False, rank=10):
    m = _handle(native, nu, ni, rank, implicit)
    try:
        m.set_ratings(u, i, r, dedup=ref.MODES[mode], ts=ts)
        return assert_ingest(m, u, i, r, nu, ni, mode, ts, implicit, rank)
    finally:
        m.close()


# ---- key widths ---------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("nu,ni", list(zip(WIDTHS, WIDTHS[::-1])) + [(WIDTHS[-1], WIDTHS[-1])])
def test_key_widths(native, nu, ni):
    """Dedup key bu + bi and CSR key row.bits + col.bits from 2 to 50 bits: ids 0 and n - 1 on both sides, repeated
    pairs, in every dedup mode on one handle."""
    rng = np.random.default_rng(nu * 7 + ni)
    pool_u = np.concatenate([[0, nu - 1], rng.integers(0, nu, 3000)])
    pool_i = np.concatenate([[ni - 1, 0], rng.integers(0, ni, 3000)])
    pick = rng.integers(0, pool_u.shape[0], 20000)
    u, i = pool_u[pick], pool_i[pick]
    r = rng.choice(np.array([-1.5, 0.0, 0.5, 1.0, 3.0, 1e7], np.float32), u.shape[0])
    ts = rng.integers(0, 4, u.shape[0])
    bu, bi = ref.ceil_log2(nu), ref.ceil_log2(ni)
    m = _handle(native, nu, ni)
    try:
        for mode in ("none", "sum", "keep_last"):
            m.set_ratings(u, i, r, dedup=ref.MODES[mode], ts=ts)
            want = assert_ingest(m, u, i, r, nu, ni, mode, ts)
            assert (want["user"][0]["bits"], want["item"][0]["bits"]) == (bu, bi)
            if mode != "none":
                assert want["user"][0]["nnz"] < u.shape[0]                      # duplicates were folded
        bits = dict(zip(WIDTHS, (1, 1, 8, 8, 9, 16, 17, 25)))
        assert (bu, bi) == (bits[nu], bits[ni])
        if nu == ni == WIDTHS[-1]:
            assert bu + bi == 50                                                # the widest keys: 50 bits
    finally:
        m.close()


# ---- runs and the order of the sum --------------------------------------------------------------------------------------
RUNS = (1, 2, 4095, 4096, 4097, 1 << 20)


@pytest.mark.parametrize("mode", ["sum", "keep_last"])
def test_long_runs_of_one_pair(native, mode):
    """One pair repeated up to 2^20 times (one thread folds a whole run), interleaved with the other runs."""
    rng = np.random.default_rng(11)
    u = np.repeat(np.arange(len(RUNS)), RUNS)
    i = np.repeat(np.arange(len(RUNS))[::-1], RUNS)
    order = rng.permutation(u.shape[0])
    u, i = u[order], i[order]
    r = rng.choice(np.array([1e8, 1.0, 0.1, -1e8, 3.0, -0.0], np.float32), u.shape[0])
    ts = rng.integers(0, 3, u.shape[0])
    _, cnt = np.unique(u * 8 + i, return_counts=True)
    assert sorted(cnt.tolist()) == sorted(RUNS)
    want = ingest_case(native, u, i, r, len(RUNS), len(RUNS), mode, ts, implicit=True)
    assert want["user"][0]["nnz"] == len(RUNS)


def test_sum_order_and_zeros(native):
    """Runs whose fp32 sum depends on the order, runs that cancel to +0, runs of -0.0 (-0.0) and single NaN, 0 and
    -0.0 ratings: none of those is positive."""
    runs = [[1e8] + [1.0] * 40, [1.0] * 40 + [1e8], [0.1] * 37, [0.1, 0.2, 0.3, -0.6], [1.0, -1.0], [0.1, -0.1],
            [-0.0], [-0.0, -0.0, -0.0], [np.nan], [0.0], [-0.0, 0.0], [3.0]]
    u = np.concatenate([np.full(len(x), k) for k, x in enumerate(runs)])
    r = np.concatenate([np.asarray(x, np.float32) for x in runs])
    i = u % 3
    want = ingest_case(native, u, i, r, len(runs), 3, "sum", implicit=True)
    d = want["user"][0]
    val_of = {int(d["inv"][row]): d["val"][d["ptr"][row]] for row in range(d["R"]) if d["deg"][d["inv"][row]]}
    assert val_of[0] == np.float32(1e8) and val_of[1] != val_of[0]
    assert [val_of[k].view(np.uint32) for k in (4, 5, 6, 7, 10)] == [0, 0, 0x80000000, 0x80000000, 0]
    assert np.isnan(val_of[8]) and d["npos"][4:11].tolist() == [0] * 7 and d["npos"][11] == 1


# ---- keep_last timestamps -----------------------------------------------------------------------------------------------
@pytest.mark.parametrize("kind", ["equal", "decreasing", "extremes", "negative", "absent"])
def test_keep_last_timestamps(native, kind):
    """Every event rating distinct, so the winner of every pair is visible; ties (equal ts, absent ts) go to the later
    event."""
    rng = np.random.default_rng(5)
    n = 20000
    u, i = rng.integers(0, 300, n), rng.integers(0, 40, n)
    r = np.arange(n, dtype=np.float32) - 7000.0          # distinct, some negative, one 0
    ts = {"equal": np.full(n, 1_600_000_000_000), "decreasing": np.arange(n, 0, -1),
          "extremes": rng.choice(np.array([I64_MIN, I64_MIN + 1, -1, 0, I64_MAX - 1, I64_MAX]), n),
          "negative": -rng.integers(1, 50, n), "absent": None}[kind]
    want = ingest_case(native, u, i, r, 300, 40, "keep_last", ts, implicit=True)
    assert want["user"][0]["nnz"] < n
    if kind in ("equal", "absent"):
        # the last event of every pair won
        last = {}
        for e in range(n):
            last[(int(u[e]), int(i[e]))] = r[e]
        du, di, dr = ref.dedup(u, i, r, "keep_last", ts)
        assert all(last[(a, b)] == v for a, b, v in zip(du.tolist(), di.tolist(), dr.tolist()))


def test_nan_and_zero_ratings_pass_through(native):
    """NaN, 0 and -0.0 kept bit for bit by none and keep_last; none of them counts as positive."""
    rng = np.random.default_rng(8)
    n = 5000
    u, i = rng.integers(0, 70, n), rng.integers(0, 50, n)
    r = rng.choice(np.array([np.nan, 0.0, -0.0, 2.0, -2.0], np.float32), n)
    for mode in ("none", "keep_last"):
        want = ingest_case(native, u, i, r, 70, 50, mode, rng.integers(0, 5, n), implicit=True)
        assert np.isnan(want["user"][0]["val"]).any()


# ---- distinct-pair counts at the scan and sort tiles --------------------------------------------------------------------
@pytest.mark.parametrize("n2", [2047, 2048, 2049, 4095, 4096, 4097])
@pytest.mark.parametrize("mode", ["sum", "keep_last"])
def test_distinct_pair_counts(native, n2, mode):
    """n2 distinct pairs (SCAN_TILE 2048, RS_TILE 4096), each one to three times; 4096 is the full 64 x 64 grid, so
    every row has the same degree and the permutation is decided by row id alone."""
    rng = np.random.default_rng(n2)
    grid = np.arange(64 * 64)
    pairs = grid if n2 == 4096 else np.sort(rng.choice(100 * 100 if n2 > 4096 else 64 * 64, n2, replace=False))
    width = 100 if n2 > 4096 else 64
    rep = rng.integers(1, 4, n2)
    e = rng.permutation(np.repeat(pairs, rep))
    u, i = e // width, e % width
    r = rng.standard_normal(e.shape[0]).astype(np.float32)
    want = ingest_case(native, u, i, r, width, width, mode, rng.integers(0, 3, e.shape[0]))
    assert want["user"][0]["nnz"] == n2 and e.shape[0] > n2
    if n2 == 4096:
        for name in ("user", "item"):
            d = want[name][0]
            assert (d["deg"] == 64).all() and np.array_equal(d["inv"], np.arange(64))


# ---- heavy rows and their parts -----------------------------------------------------------------------------------------
@pytest.mark.parametrize("rank,heavy", [(16, 2), (64, 4), (128, None)])
def test_heavy_rows(native, rank, heavy):
    """Items with 9000, 4097, 1537, 1025 distinct users and a tail: above and below the FP32 (4096) and pair (1024)
    heavy-row thresholds; at rank 65..128 every active row is heavy."""
    rng = np.random.default_rng(rank)
    nu, ni = 10000, 60
    lens = [9000, 4097, 1537, 1025, 1024, 600] + [40] * (ni - 6)
    i = np.repeat(np.arange(ni), lens)
    u = np.concatenate([rng.choice(nu, d, replace=False) for d in lens])
    r = rng.standard_normal(u.shape[0]).astype(np.float32)
    want = ingest_case(native, u, i, r, nu, ni, "none", implicit=False, rank=rank)
    d = want["item"][0]
    assert d["n_heavy"] == (d["n_active"] if heavy is None else heavy) and d["n_parts"] > d["n_heavy"]
    if heavy is None:
        assert want["user"][0]["n_heavy"] == want["user"][0]["n_active"]


# ---- input routes ---------------------------------------------------------------------------------------------------------
def test_device_input_equals_host_input(native):
    torch = pytest.importorskip("torch")
    rng = np.random.default_rng(3)
    n, nu, ni = 50000, 3000, 700
    u, i = rng.integers(0, nu, n).astype(np.int32), rng.integers(0, ni, n).astype(np.int32)
    r = rng.standard_normal(n).astype(np.float32)
    ts = rng.integers(0, 10, n)
    for mode in ("none", "sum", "keep_last"):
        dev = [torch.from_numpy(x).cuda() for x in (u, i, r, ts)]
        m = _handle(native, nu, ni, implicit=True)
        try:
            m.set_ratings_device(dev[0].data_ptr(), dev[1].data_ptr(), dev[2].data_ptr(), n, dedup=ref.MODES[mode],
                                 d_ts=dev[3].data_ptr())
            torch.cuda.synchronize()
            assert_ingest(m, u, i, r, nu, ni, mode, ts, implicit=True)
        finally:
            m.close()


@pytest.mark.parametrize("dedup", ["sum", "keep_last"])
def test_mllib_route(native, dedup):
    """ALS.trainImplicit(..., dedup=...) ingests through pio_als_train; the model keeps the handle."""
    rng = np.random.default_rng(4)
    n, nu, ni = 30000, 800, 150
    u, i = rng.integers(0, nu, n).astype(np.int32), rng.integers(0, ni, n).astype(np.int32)
    r = rng.choice(np.array([0.5, 1.0, 2.0, -1.0, 0.0], np.float32), n)
    ts = rng.integers(1_600_000_000_000, 1_600_000_000_010, n)
    model = mllib.ALS.trainImplicit((u, i, r, ts), 8, 2, 0.01, alpha=0.5, seed=3, dedup=dedup,
                                       n_users=nu, n_products=ni)
    try:
        assert_ingest(model._h, u, i, r, nu, ni, dedup, ts, implicit=True, rank=8)
    finally:
        model._h.close()


def test_second_set_ratings_shows_only_the_second_input(native):
    rng = np.random.default_rng(6)
    nu, ni = 500, 90
    m = _handle(native, nu, ni)
    try:
        u1, i1 = rng.integers(0, nu, 9000), rng.integers(0, ni, 9000)
        m.set_ratings(u1, i1, rng.standard_normal(9000).astype(np.float32), dedup=ref.MODES["sum"])
        u2, i2 = rng.integers(0, nu // 2, 3000), rng.integers(0, ni, 3000)
        r2 = rng.standard_normal(3000).astype(np.float32)
        m.set_ratings(u2, i2, r2, dedup=ref.MODES["keep_last"])
        assert_ingest(m, u2, i2, r2, nu, ni, "keep_last")
        m.run(1)
        assert_ingest(m, u2, i2, r2, nu, ni, "keep_last")      # training reads the ingest, changes none of it
    finally:
        m.close()


def test_oversized_and_bad_mode_calls_are_refused_before_staging(native):
    """nnz = 2^32 with one-element host arrays, and a bad dedup mode: ERR_ARG before any copy, and the handle keeps its
    ratings and still trains."""
    rng = np.random.default_rng(2)
    nu, ni = 200, 50
    u, i = rng.integers(0, nu, 4000), rng.integers(0, ni, 4000)
    r = rng.standard_normal(4000).astype(np.float32)
    m = _handle(native, nu, ni)
    try:
        m.set_ratings(u, i, r, dedup=ref.MODES["sum"])
        one_i, one_f, one_t = np.zeros(1, np.int32), np.ones(1, np.float32), np.zeros(1, np.int64)
        lib = native.lib()
        p = lambda a, t: a.ctypes.data_as(C.POINTER(t))   # noqa: E731
        for nnz, mode in (((1 << 32), 0), ((1 << 32), 2), (1 << 40, 1), (1, 3), (1, -1)):
            rc = lib.pio_als_set_ratings_coo(m._h, p(one_i, C.c_int32), p(one_i, C.c_int32), p(one_f, C.c_float),
                                             C.c_int64(nnz), C.c_int(mode), p(one_t, C.c_int64))
            assert rc == native.ERR_ARG, (nnz, mode)
        assert_ingest(m, u, i, r, nu, ni, "sum")
        m.run(2)
        uf, itf, uh, ih = m.get_factors()
        assert np.isfinite(uf).all() and uh.sum() == np.unique(u).shape[0]
    finally:
        m.close()


# ---- scale ----------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("mode", ["sum", "keep_last"])
def test_zipf_view_log(native, mode):
    """20 M view events on Zipf-distributed users and items (heavy duplication), millisecond timestamps with ties."""
    rng = np.random.default_rng(20)
    n, nu, ni = 20_000_000, 400_000, 60_000
    u = (np.minimum(rng.zipf(1.3, n), nu) - 1).astype(np.int32)
    i = (np.minimum(rng.zipf(1.2, n), ni) - 1).astype(np.int32)
    r = rng.choice(np.array([1.0, 0.5, 2.0, 0.1], np.float32), n)
    ts = 1_600_000_000_000 + rng.integers(0, 5_000_000, n)
    want = ingest_case(native, u, i, r, nu, ni, mode, ts, implicit=True)
    d = want["item"][0]
    assert want["user"][0]["nnz"] < n // 2 and d["n_heavy"] > 0


# ---- the dedup output solves right ----------------------------------------------------------------------------------------
@pytest.mark.parametrize("mode,implicit", [("sum", True), ("keep_last", False)])
def test_half_step_on_the_deduplicated_ratings(native, mode, implicit):
    """One iteration after a dedup ingest: every item row against halfstep_ref on the restated, deduplicated COO from
    the initial user factors, every user row from the GPU's item rows."""
    nu, ni, rank = 2000, 300, 10
    u, i, r = synth.synth_ratings(nu, ni, 30000, seed=9, implicit=implicit)
    rng = np.random.default_rng(9)
    pick = rng.integers(0, u.shape[0], 15000)                                  # repeat half the events
    u, i = np.concatenate([u, u[pick]]), np.concatenate([i, i[pick]])
    r = np.concatenate([r, rng.standard_normal(15000).astype(np.float32) + (2.0 if not implicit else 0.0)])
    ts = rng.integers(0, 4, u.shape[0])
    m = native.NativeALS(rank, nu, ni, lam=LAM, implicit=implicit, alpha=ALPHA)
    try:
        m.set_ratings(u, i, r, dedup=ref.MODES[mode], ts=ts)
        assert_ingest(m, u, i, r, nu, ni, mode, ts, implicit, rank)
        src = synth.synth_init_factors(nu, rank, 5, 0)
        m.set_init(src)
        m.run(1)
        uf, itf, uh, ih = m.get_factors()
        assert m.phase_ms()["item_kernel"] == "fp32"
    finally:
        m.close()
    du, di, dr = ref.dedup(u, i, r, mode, ts)
    assert du.shape[0] < u.shape[0]
    src[np.bincount(du, minlength=nu) == 0] = 0
    check_rows("item", H.half_step(di, du, dr, ni, src, LAM, implicit, ALPHA, cand=itf), itf, ih, TAU["fp32-16"], 4096)
    check_rows("user", H.half_step(du, di, dr, nu, itf, LAM, implicit, ALPHA, cand=uf), uf, uh, TAU["fp32-16"], 4096)
