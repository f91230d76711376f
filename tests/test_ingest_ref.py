"""tests/ingest_ref.py (the restatement of the ALS rating ingest that test_gpu_ingest.py holds the device to) against
independent constructions: oracle.dedup_coo's per-run loops for the dedup rules, scipy.sparse for both CSR orientations,
and itself on 1 GPU for the deal to 2, 4 and 8 ranks."""
import numpy as np
import pytest
import scipy.sparse as sp

import ingest_ref as ref


def _events(seed, n, nu, ni, ties=True):
    rng = np.random.default_rng(seed)
    u = rng.integers(0, nu, n)
    i = rng.integers(0, ni, n)
    r = rng.choice(np.array([-2.0, -0.0, 0.0, 0.1, 1.0, 1e8, 3.5], np.float32), n)
    ts = rng.integers(0, 20 if ties else 1 << 40, n)
    return u, i, r, ts


@pytest.mark.parametrize("seed,n,nu,ni", [(1, 3000, 30, 20), (2, 500, 7, 300), (3, 4000, 3, 2), (4, 100, 1, 1)])
@pytest.mark.parametrize("mode", ["sum", "keep_last"])
@pytest.mark.parametrize("with_ts", [True, False])
def test_dedup_equals_the_oracle(oracle, seed, n, nu, ni, mode, with_ts):
    u, i, r, ts = _events(seed, n, nu, ni)
    ts = ts if with_ts else None
    gu, gi, gr = ref.dedup(u, i, r, mode, ts)
    ou, oi, orr = oracle.dedup_coo(u, i, r, mode, ts)
    assert np.array_equal(gu, ou) and np.array_equal(gi, oi)
    assert np.array_equal(gr.view(np.uint32), orr.view(np.uint32))


def test_sum_reduces_in_event_order_past_the_vectorised_prefix(oracle):
    """Runs of 1 .. 300 events (the restatement folds the first 64 positions across runs, the rest per run) whose fp32
    sums depend on the order, runs of -0.0 that keep their sign and runs that cancel to +0."""
    rng = np.random.default_rng(9)
    lens = np.array([1, 2, 63, 64, 65, 127, 300], np.int64)
    u = np.repeat(np.arange(lens.shape[0]), lens)
    vals = rng.choice(np.array([1e8, 1.0, 0.1, -1e8, 3.0], np.float32), u.shape[0])
    u = np.concatenate([u, [10, 10, 11, 12, 12]])
    r = np.concatenate([vals, np.array([-0.0, -0.0, -0.0, 1.0, -1.0], np.float32)])
    order = rng.permutation(u.shape[0])
    u, r = u[order], r[order]
    r[u == 6] = np.r_[np.float32(1e8), np.ones(299, np.float32)]   # the ones vanish one by one, not in reverse order
    i = np.zeros_like(u)
    gu, _, gr = ref.dedup(u, i, r, "sum")
    ou, _, orr = oracle.dedup_coo(u, i, r, "sum")
    assert np.array_equal(gu, ou) and np.array_equal(gr.view(np.uint32), orr.view(np.uint32))
    bits = dict(zip(gu.tolist(), gr.view(np.uint32).tolist()))
    assert bits[10] == bits[11] == 0x80000000 and bits[12] == 0
    rev = np.float32(0)
    for v in r[u == 6][::-1]:
        rev = np.float32(rev + v)
    assert rev != gr[gu == 6][0]             # the 300-event run's sum depends on the order


def _csr_rows(side, cinv):
    """Per external row: (external columns, values) in CSR order, from every rank's slice."""
    rows = {}
    for k, d in enumerate(side):
        for r in range(d["R"]):
            ext = int(d["inv"][k * d["R"] + r])
            if ext < 0:
                continue
            b, e = d["ptr"][r], d["ptr"][r + 1]
            rows[ext] = (cinv[d["idx"][b:e]], d["val"][b:e])
    return rows


@pytest.mark.parametrize("mode", ["none", "sum", "keep_last"])
@pytest.mark.parametrize("implicit", [False, True])
def test_both_csr_orientations_equal_scipy(mode, implicit):
    nu, ni = 50, 37
    u, i, r, ts = _events(5, 2500, nu, ni)
    out = ref.ingest(u, i, r, nu, ni, mode, ts, implicit)
    du, di, dr = ref.dedup(u, i, r, mode, ts)
    for name, rows, cols, n, m in (("user", du, di, nu, ni), ("item", di, du, ni, nu)):
        (d,), (c,) = out[name], out["item" if name == "user" else "user"]
        assert d["n_internal"] == d["R"] == n and d["nnz"] == d["nnz_local"] == du.shape[0]
        # scipy: row x event incidence (no duplicate coordinates, so duplicates of a pair stay apart), and the
        # row x column multiplicities
        k = rows.shape[0]
        mat = sp.coo_matrix((np.ones(k), (rows, np.arange(k))), shape=(n, k)).tocsr()
        mat.sort_indices()
        assert np.array_equal(np.diff(mat.indptr), d["deg"].astype(np.int64))
        mult = sp.coo_matrix((np.ones(k), (rows, cols)), shape=(n, m)).tocsr()
        assert np.array_equal(np.asarray(mult.sum(axis=1)).ravel(), d["deg"])
        if mode != "none":
            assert mult.max() == 1
        pos = sp.csr_matrix(((dr > 0).astype(np.float64), (rows, cols)), shape=(n, m))
        assert np.array_equal(np.asarray(pos.sum(axis=1)).ravel().astype(np.int64), d["npos"].astype(np.int64))
        got = _csr_rows(out[name], c["inv"])
        for x in range(n):
            ent = mat.indices[mat.indptr[x]:mat.indptr[x + 1]].astype(np.int64)   # entries of row x, in input order
            ent = ent[np.lexsort((ent, c["rpos"][cols[ent]]))]                  # by column position, then event
            if ent.shape[0] == 0:
                assert x not in got
                continue
            gc, gv = got[x]
            assert np.array_equal(gc, cols[ent]) and np.array_equal(gv.view(np.uint32), dr[ent].view(np.uint32)), x
        # internal order is degree-descending; nreg follows implicit
        ext = d["inv"]
        assert (np.diff(d["deg"][ext[ext >= 0]].astype(np.int64)) <= 0).all()
        assert np.array_equal(d["nreg"][ext >= 0], (d["npos"] if implicit else d["deg"])[ext[ext >= 0]].astype(np.float32))


@pytest.mark.parametrize("W", [2, 4, 8])
@pytest.mark.parametrize("mode,rank", [("none", 64), ("sum", 16), ("keep_last", 128)])
def test_rank_slices_reassemble_the_single_gpu_result(W, mode, rank):
    """The deal: every external row lands on exactly one rank with the same entries, bit for bit, and the same parts."""
    rng = np.random.default_rng(W)
    nu, ni = 20003, 61                                   # not multiples of W: padding rows on the last ranks
    u = np.concatenate([rng.integers(0, nu, 30000), np.full(1500, 7), np.full(5000, 11)])
    i = np.concatenate([rng.integers(0, ni, 30000), rng.integers(0, ni, 1500), rng.integers(0, ni, 5000)])
    i[:6000] = 3                                         # one item above the FP32 threshold (4096) after dedup
    r = rng.standard_normal(u.shape[0]).astype(np.float32)
    one = ref.ingest(u, i, r, nu, ni, mode, None, True, 1, rank)
    many = ref.ingest(u, i, r, nu, ni, mode, None, True, W, rank)
    for name, other in (("user", "item"), ("item", "user")):
        (d1,), (c1,) = one[name], one[other]
        rows1 = _csr_rows(one[name], c1["inv"])
        rowsW = _csr_rows(many[name], many[other][0]["inv"])
        assert rows1.keys() == rowsW.keys()
        for x, (cols, vals) in rows1.items():
            assert np.array_equal(rowsW[x][0], cols) and np.array_equal(rowsW[x][1].view(np.uint32), vals.view(np.uint32))
        assert sum(d["nnz_local"] for d in many[name]) == d1["nnz_local"]
        assert sum(d["n_active"] for d in many[name]) == d1["n_active"]
        assert sum(d["n_heavy"] for d in many[name]) == d1["n_heavy"] > (0 if name == "item" else -1)
        # the part lengths of every heavy row are the same wherever it lives
        def parts(side):
            got = {}
            for k, d in enumerate(side):
                for h in range(d["n_heavy"]):
                    ext = int(d["inv"][k * d["R"] + h])
                    a, b = d["row_part_ptr"][h], d["row_part_ptr"][h + 1]
                    got[ext] = (d["part_end"][a:b] - d["part_beg"][a:b]).tolist()
            return got
        assert parts(many[name]) == parts(one[name])
        for d in many[name]:
            assert d["R"] == -(-d1["n"] // W) and d["n_internal"] == d["R"] * W
            assert (d["inv"] == -1).sum() == d["n_internal"] - d["n"]
            assert np.array_equal(d["rpos"], d1["rpos"])   # degree-rank positions do not depend on W


def test_plan_follows_the_solve_plan_switches():
    c = ref.plan_constants()
    assert ref.side_plan(16, 100, 1000) == (c["HEAVY_T"], c["PART"])
    assert ref.side_plan(64, 100, 1000) == (c["PAIR_SEG_T"], c["PAIR_PART"])
    assert ref.side_plan(128, 100, 1000) == (0, c["PART"])
    assert ref.side_plan(64, 100, 1000, {"PIO_ALS_TC": "1"}) == (c["HEAVY_T_TC"], c["PART"])
    assert ref.side_plan(64, 100, 1000, {"PIO_ALS_MMA": "1"}) == (c["HEAVY_T_TC"], c["PART"])
    assert ref.side_plan(64, 100, 1000, {"PIO_ALS_MMA": "0"}) == (c["HEAVY_T"], c["PART"])
    assert ref.side_plan(64, 100, 1000, {"PIO_ALS_SEG_T": "40", "PIO_ALS_PART": "13"}) == (40, 16)
    assert ref.side_plan(64, 100, 1000, {"PIO_ALS_TC": "1", "PIO_ALS_TC_MIN_DEG": "11"})[0] == c["PAIR_SEG_T"]
