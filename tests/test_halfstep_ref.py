"""CPU tests of tests/halfstep_ref.py (the fp64 half-step reference the row-by-row GPU tests check against) and of the
degree ladder those tests use: the reference agrees with both oracle restatements, and the ladder straddles every
row-length threshold the CUDA sources define."""
import numpy as np
import pytest

import halfstep_ref as H
import test_gpu_halfstep as G
from pio_b200 import synth


def _problem(nu, ni, nnz, seed, implicit, rank):
    u, i, r = synth.synth_ratings(nu, ni, nnz, seed=seed, implicit=implicit)
    if implicit:
        r = r.copy()
        r[::5] = -r[::5]
        r[::7] = 0.0
        r[np.isin(u, [3, 4])] = -1.0      # two users whose preferences are all negative: ridge lambda * n+ = 0
    u0 = synth.synth_init_factors(nu, rank, 5, 0)
    u0[np.bincount(u, minlength=nu) == 0] = 0
    return u, i, r, u0


@pytest.mark.parametrize("implicit", [False, True])
@pytest.mark.parametrize("rank", [1, 4, 13])
def test_reference_matches_oracles(oracle, implicit, rank):
    nu, ni, nnz, lam, alpha = 60, 25, 500, 0.05, 1.5
    u, i, r, u0 = _problem(nu, ni, nnz, 7, implicit, rank)
    src = u0
    # item rows from the user factors, then user rows from those item rows (the second includes the users whose
    # preferences are all negative)
    for dst, col, n_dst in ((i, u, ni), (u, i, nu)):
        ref = H.half_step(dst, col, r, n_dst, src, lam, implicit, alpha)
        # dense NumPy/SciPy restatement
        dense = oracle.numpy_half_step(n_dst, dst, col, r, src, np.zeros((n_dst, rank), np.float32), lam, implicit, alpha)
        assert np.abs(ref.x - dense).max() <= 1e-6 * max(1.0, np.abs(ref.x).max())
        # C restatement (fp64 accumulation, fp32 output)
        ptr, idx, val = oracle.csr_build(n_dst, dst, col, r)
        yty = oracle.gram(src) if implicit else None
        out, fails = oracle.half_step_rows(ptr, idx, val, src, np.arange(n_dst, dtype=np.int32), lam, implicit, alpha,
                                           yty)
        assert fails == 0
        assert np.abs(ref.x - out).max() <= 1e-6 * max(1.0, np.abs(ref.x).max())
        assert np.array_equal(ref.deg, np.bincount(dst, minlength=n_dst))
        if implicit:
            assert np.array_equal(ref.npos, np.bincount(dst, weights=r > 0, minlength=n_dst).astype(np.int64))
        src = ref.x.astype(np.float32)
    if implicit:
        assert (ref.npos[[3, 4]] == 0).all() and (ref.deg[[3, 4]] > 0).all() and (ref.x[[3, 4]] == 0).all()


@pytest.mark.parametrize("implicit", [False, True])
def test_backward_error_measures(implicit):
    """eta of the exact solution is at rounding level; dropping one rating of a row or perturbing one coordinate
    shows up as a backward error far above it; the forward error obeys the perturbation bound."""
    nu, ni, nnz, rank, lam, alpha = 300, 40, 6000, 8, 0.02, 0.7
    u, i, r, u0 = _problem(nu, ni, nnz, 3, implicit, rank)
    ref = H.half_step(i, u, r, ni, u0, lam, implicit, alpha)
    good = H.half_step(i, u, r, ni, u0, lam, implicit, alpha, cand=ref.x)
    act = good.deg > 0
    assert good.eta[act].max() <= 1e-14
    f32 = H.half_step(i, u, r, ni, u0, lam, implicit, alpha, cand=ref.x.astype(np.float32))
    assert f32.eta[act].max() <= 1e-7 and (f32.eta[act] > 0).all()
    assert (f32.fwd[act] <= f32.fwd_bound[act] * 1.01 + 1e-15).all()
    # one rating dropped from the row of the most ratings
    row = int(np.argmax(ref.deg))
    drop = np.flatnonzero(i == row)[np.argmax(np.abs(r[i == row]))]
    keep = np.ones(i.shape[0], bool)
    keep[drop] = False
    wrong = H.half_step(i[keep], u[keep], r[keep], ni, u0, lam, implicit, alpha).x
    bad = H.half_step(i, u, r, ni, u0, lam, implicit, alpha, cand=wrong)
    assert bad.eta[row] >= 1e-4 and np.delete(bad.eta, row)[np.delete(act, row)].max() <= 1e-14
    # one coordinate off by 1e-3 relative
    x = ref.x.copy()
    x[row, 0] += 1e-3 * np.linalg.norm(x[row])
    assert H.half_step(i, u, r, ni, u0, lam, implicit, alpha, cand=x).eta[row] >= 1e-5


def test_degree_ladder_straddles_every_planner_threshold():
    """Moving a row-length threshold in the solve planner (solve_plan.h) or the CUDA sources without moving the GPU
    tests' degree ladder fails here."""
    host, tc = G.source_constants("solve_plan.h"), G.source_constants("als_tc_kernel.cuh")
    assert G.HEAVY == {"pair": host["PAIR_SEG_T"], "mma": host["HEAVY_T_TC"], "wgmma": host["HEAVY_T_TC"],
                       "fp32": host["HEAVY_T"]}
    ladder = set(G.DEGREE_LADDER)

    def straddles(t):
        return {t - 1, t, t + 1} <= ladder

    for name in ("PAIR_SEG_T", "PAIR_PART", "HEAVY_T", "HEAVY_T_TC", "PART"):
        assert straddles(host[name]), (name, host[name])
    assert straddles(2 * host["PART"])                                 # a row of exactly two parts, and one more
    assert {host["PAIR_SEG_T"] + host["PAIR_PART"], host["PAIR_SEG_T"] + host["PAIR_PART"] + 1} <= ladder
    assert straddles(tc["STAGE_RATINGS"]) and straddles(tc["SEG"]), (tc["STAGE_RATINGS"], tc["SEG"])
    assert max(ladder) > host["HEAVY_T_TC"] + host["PART"]              # several parts on every path
    assert set(range(1, 10)) <= ladder and {15, 16, 17} <= ladder
    # the rank 65..128 case has more active rows on one side than one tile of the work-list launch
    assert G.SCALE_ROWS > host["LS128_TILE_ROWS"]
    assert max(G.SCALE_HEAVY) > 2 * host["PART"]
