"""GPU tests (-m gpu): every ALS solve path checked row by row against the fp64 half-step reference (halfstep_ref.py).

One iteration isolates each half-step: after set_init(u0) and run(1), every active item row is checked against the
reference built from u0 (rows without ratings zeroed), and every active user row against the reference built from the
GPU's own item rows, so no error carries over from the first half-step.  A second variant runs a few iterations first
and checks the next one, on near-converged factors.  Each row must have a normwise backward error
eta = ||A x - b|| / (||A|| ||x|| + ||b||) below the path's tolerance; eta does not grow with the row's condition number,
so it stays tight on the ill-conditioned explicit rows (halfstep_ref.py: b enters with the magnitude of its terms).
The forward error ||x - x*|| / ||x*|| is checked against the bound ||A^-1|| ||A x - b|| / ||x*|| its residual allows.  Every case asserts the kernel labels of phase_ms(), so it provably ran the path it names.

Which kernel solves a row depends on the padded rank (16 / 32 / 64 / 128), the path switches (PIO_ALS_TC, PIO_ALS_MMA)
and the row's rating count: rows longer than the path's heavy-row threshold are cut into parts whose partial normal
equations a finish kernel sums (at rank 65..128 every row is).  The degree ladder puts rows just below, at and above
every such threshold, the part lengths and the wgmma stage and segment sizes (test_halfstep_ref.py keeps it in step
with the constants in the CUDA sources).

Tolerances (TAU) are about 4x the largest eta measured on an H100 80GB HBM3, listed beside each.
"""
import itertools
import re
from pathlib import Path

import numpy as np
import pytest

import halfstep_ref as H
from pio_b200 import synth

pytestmark = pytest.mark.gpu

CSRC = Path(__file__).resolve().parent.parent / "incubator-predictionio_b200" / "csrc"

# row lengths of the degree ladder: 1..9 and 15..17 (chunk tails of the 8 / 4 / 8 / 9-rating FP32 chunks and the
# 8-rating mma chunks), then below / at / above the wgmma stage (24) and segment (504), the pair part (512) and
# whole-row limit (1024, 1024 + 512), the 2016-rating part (one and two parts), the FP32 heavy-row threshold (4096),
# the tensor-core heavy-row threshold (8192), and one row of six parts
DEGREE_LADDER = (1, 2, 3, 4, 5, 6, 7, 8, 9, 15, 16, 17, 23, 24, 25, 503, 504, 505, 511, 512, 513,
                 1023, 1024, 1025, 1536, 1537, 2015, 2016, 2017, 4031, 4032, 4033, 4095, 4096, 4097,
                 8191, 8192, 8193, 12000)
LADDER_USERS = 12500
LADDER_FILL = 160
SCALE_ROWS = 34000                 # active rows of the large side in the rank 65..128 case (> one 32768-row tile)
SCALE_HEAVY = (2017, 4033, 6000)   # its long rows: two, three and three parts of 2016 ratings
# heavy-row threshold of each rank-1..64 kernel (rows with more ratings are solved in parts); rank 65..128: every row
HEAVY = {"pair": 1024, "mma": 8192, "wgmma": 8192, "fp32": 4096}
LAM, ALPHA = 0.02, 0.7

# path -> tolerance, about 4x the largest eta measured over this module's cases on an H100 80GB HBM3 (400 W power
# limit): rows solved whole / rows solved in parts
TAU = {
    "fp32-16": 8e-7,     # 2.0e-7 / 9.2e-8
    "fp32-32": 7e-7,     # 1.7e-7 / 9.1e-8
    "fp32-64": 5e-7,     # 1.3e-7 / 6.3e-8
    "pair": 6.5e-7,      # 1.6e-7 / 8.6e-8 (40-rating parts: 8.6e-8)
    "mma": 1.8e-6,       # 4.4e-7 / 5.8e-8 (whole rows of up to 8192 ratings, accumulated in one level)
    "wgmma": 1.4e-6,     # 3.5e-7 / 5.1e-8
    "ls128": 1.1e-6,     # every row in parts: 2.6e-7
}
ENV_VARS = ("PIO_ALS_TC", "PIO_ALS_TC_MIN_DEG", "PIO_ALS_TC_SPLIT", "PIO_ALS_MMA", "PIO_ALS_PAIR_WARPS",
            "PIO_ALS_PIECES", "PIO_ALS_SEG_T", "PIO_ALS_PART")


def source_constants(name):
    """`constexpr int NAME = expr;` definitions of one CUDA source, evaluated in order (later ones may use earlier)."""
    env = {}
    for key, expr in re.findall(r"constexpr\s+int\s+(\w+)\s*=\s*([^;]+);", (CSRC / name).read_text()):
        try:
            env[key] = int(eval(expr.replace("/", "//"), {"__builtins__": {}}, dict(env)))
        except (NameError, SyntaxError, TypeError):
            pass
    return env


def path_of(rank, env):
    """(phase_ms kernel label, heavy-row threshold, TAU key) of the half-steps at this rank and switch setting."""
    kp = 16 if rank <= 16 else 32 if rank <= 32 else 64 if rank <= 64 else 128
    if kp == 128:
        return "fp32", 0, "ls128"
    if kp < 64:
        return "fp32", HEAVY["fp32"], f"fp32-{kp}"
    if env.get("PIO_ALS_TC") == "1":
        return "wgmma", HEAVY["wgmma"], "wgmma"
    if env.get("PIO_ALS_MMA") == "1":
        return "mma", HEAVY["mma"], "mma"
    if env.get("PIO_ALS_MMA") == "0":
        return "fp32", HEAVY["fp32"], "fp32-64"
    return "pair", int(env.get("PIO_ALS_SEG_T", HEAVY["pair"])), "pair"


def set_env(monkeypatch, env):
    for v in ENV_VARS:
        monkeypatch.delenv(v, raising=False)
    for k, v in env.items():
        monkeypatch.setenv(k, v)


def implicit_prefs(u, i, r, seed, users_allneg=True):
    """Implicit preferences with negative and zero values, and a few items (and users) whose preferences are all <= 0:
    their ridge lambda * n+ is 0 and the row is solved from YtY and the confidence terms alone.  Such a row is positive
    definite only when YtY is, so users get them only where there are at least rank item rows."""
    rng = np.random.default_rng(seed)
    r = np.abs(np.asarray(r, np.float32)) + rng.random(r.shape[0]).astype(np.float32)
    r[::5] = -r[::5]
    r[::7] = 0.0
    allneg = (i % 97 == 5) | ((u % 23 == 4) & users_allneg)
    r[allneg] = -np.abs(r[allneg])
    return r


def check_rows(side, ref, out, has, tau, heavy_t):
    """Assert every row of one half-step; returns the largest eta of the whole rows and of the rows solved in parts."""
    act = ref.deg > 0
    assert np.array_equal(has.astype(bool), act), side
    assert (out[~act] == 0).all(), side
    eta = ref.eta[act]
    worst = np.flatnonzero(act)[np.argsort(-eta)[:5]]
    report = [(int(w), int(ref.deg[w]), float(ref.eta[w]), float(ref.kappa[w]), float(ref.fwd[w])) for w in worst]
    assert np.isfinite(out[act]).all() and eta.max() <= tau, (side, "worst rows (row, degree, eta, kappa, fwd)", report)
    assert (ref.fwd[act] <= 1.01 * ref.fwd_bound[act] + 1e-12 * ref.kappa[act]).all(), (side, report)
    parts = act & (ref.deg > heavy_t)
    return float(ref.eta[act & ~parts].max(initial=0)), float(ref.eta[parts].max(initial=0))


def one_iteration(native, monkeypatch, nu, ni, u, i, r, rank, implicit, env, warm=0, seed=5, tag=""):
    label, heavy_t, key = path_of(rank, env)
    set_env(monkeypatch, env)
    m = native.NativeALS(rank, nu, ni, lam=LAM, implicit=implicit, alpha=ALPHA)
    m.set_ratings(u, i, r, dedup=0)
    src = synth.synth_init_factors(nu, rank, seed, 0)
    m.set_init(src)
    src[np.bincount(u, minlength=nu) == 0] = 0
    if warm:
        m.run(warm)
        src = m.get_factors()[0]
    m.run(1)
    uf, itf, uh, ih = m.get_factors()
    ph = m.phase_ms()
    m.close()
    assert (ph["item_kernel"], ph["user_kernel"]) == (label, label), (ph, env)
    ri = H.half_step(i, u, r, ni, src, LAM, implicit, ALPHA, cand=itf)
    ei = check_rows("item", ri, itf, ih, TAU[key], heavy_t)
    ru = H.half_step(u, i, r, nu, itf, LAM, implicit, ALPHA, cand=uf)
    eu = check_rows("user", ru, uf, uh, TAU[key], heavy_t)
    print(f"\nETA {key} {tag} rank={rank} implicit={int(implicit)} warm={warm} env={env} "
          f"item_whole={ei[0]:.3e} item_parts={ei[1]:.3e} user_whole={eu[0]:.3e} user_parts={eu[1]:.3e} "
          f"item_deg_max={int(ri.deg.max())} user_deg_max={int(ru.deg.max())}")
    return ri, ru


# ---- rank ladder ------------------------------------------------------------------------------------------------------
def ladder_problem(implicit):
    nu, ni = 2000, 300
    u, i, r = synth.synth_ratings(nu, ni, 30000, seed=3, implicit=implicit)
    if implicit:
        r = implicit_prefs(u, i, r, 1)
    return nu, ni, u, i, r


@pytest.mark.parametrize("implicit", [False, True])
@pytest.mark.parametrize("rank", [1, 2, 15, 16, 17, 31, 32, 33, 40, 47, 63, 64, 65, 96, 127, 128])
def test_rank_ladder_default_paths(native, monkeypatch, rank, implicit):
    """Default path of every padded rank; rank 33..63 exercises the padded lanes of the pair kernel's Gramian and of the
    lockstep solver (unit diagonal beyond k), which matter most on implicit rows whose ridge lambda * n+ is 0.  The head
    item (~1700 ratings) is solved in parts on the pair path and at rank 65..128."""
    nu, ni, u, i, r = ladder_problem(implicit)
    one_iteration(native, monkeypatch, nu, ni, u, i, r, rank, implicit, {})


@pytest.mark.parametrize("env", [{"PIO_ALS_TC": "1"}, {"PIO_ALS_MMA": "1"}, {"PIO_ALS_MMA": "0"}],
                         ids=["wgmma", "mma", "fp32"])
@pytest.mark.parametrize("implicit", [False, True])
@pytest.mark.parametrize("rank", [33, 48, 63, 64])
def test_rank_ladder_alternative_paths(native, monkeypatch, rank, implicit, env):
    nu, ni, u, i, r = ladder_problem(implicit)
    one_iteration(native, monkeypatch, nu, ni, u, i, r, rank, implicit, env)


@pytest.mark.parametrize("rank,env", [(16, {}), (32, {}), (64, {}), (64, {"PIO_ALS_TC": "1"}), (128, {})],
                         ids=["fp32-16", "fp32-32", "pair", "wgmma", "ls128"])
@pytest.mark.parametrize("implicit", [False, True])
def test_near_converged_factors(native, monkeypatch, rank, env, implicit):
    """run(4) then run(1): the checked half-steps start from near-converged factors (run is resumable)."""
    nu, ni, u, i, r = ladder_problem(implicit)
    one_iteration(native, monkeypatch, nu, ni, u, i, r, rank, implicit, env, warm=4)


# ---- degree ladder ----------------------------------------------------------------------------------------------------
def degree_ladder_problem(transpose, implicit, seed=17):
    """Long side: one row per DEGREE_LADDER entry with exactly that many distinct partners, plus LADDER_FILL rows of 10
    (so that the short side's YtY has full rank at rank 128 and its implicit rows without a positive preference are
    well posed); short side: LADDER_USERS rows of about six ratings.  transpose=False puts the ladder on the item side
    (first half-step, sourced from the initial factors), transpose=True on the user side (second half-step, sourced
    from the GPU's item rows)."""
    rng = np.random.default_rng(seed)
    degs = DEGREE_LADDER + (10,) * LADDER_FILL
    long_rows = np.repeat(np.arange(len(degs), dtype=np.int32), degs)
    short_rows = np.concatenate([rng.choice(LADDER_USERS, d, replace=False) for d in degs]).astype(np.int32)
    r = rng.integers(1, 6, long_rows.shape[0]).astype(np.float32)
    if transpose:
        u, i, nu, ni = long_rows, short_rows, len(degs), LADDER_USERS
    else:
        u, i, nu, ni = short_rows, long_rows, LADDER_USERS, len(degs)
    if implicit:
        r = implicit_prefs(u, i, r, seed)
    return nu, ni, u, i, r


LADDER_PATHS = {
    "fp32-16": (16, {}), "fp32-32": (32, {}), "fp32-64": (64, {"PIO_ALS_MMA": "0"}), "pair": (64, {}),
    "pair-short-parts": (40, {"PIO_ALS_SEG_T": "64", "PIO_ALS_PART": "40"}), "mma": (64, {"PIO_ALS_MMA": "1"}),
    "wgmma": (64, {"PIO_ALS_TC": "1"}), "ls128": (128, {}), "ls128-k100": (100, {}),
}


@pytest.mark.parametrize("transpose", [False, True], ids=["items", "users"])
@pytest.mark.parametrize("path", list(LADDER_PATHS))
def test_degree_ladder(native, monkeypatch, path, transpose):
    """Rows just below, at and above every threshold of every path, on both half-steps.  pair-short-parts cuts every
    row above 64 ratings into 40-rating parts: rows of up to 300 parts through als_finish_pair_kernel."""
    rank, env = LADDER_PATHS[path]
    implicit = not transpose
    nu, ni, u, i, r = degree_ladder_problem(transpose, implicit)
    ri, ru = one_iteration(native, monkeypatch, nu, ni, u, i, r, rank, implicit, env, tag=path)
    ladder = ru if transpose else ri
    assert sorted(ladder.deg[:len(DEGREE_LADDER)].tolist()) == sorted(DEGREE_LADDER)


# ---- rank 65..128 at scale -------------------------------------------------------------------------------------------
@pytest.mark.parametrize("rank,implicit", [(96, True), (128, False)])
def test_rank128_tiles_at_scale(native, monkeypatch, rank, implicit):
    """More active user rows than one 32768-row tile of the work-list launch (the partial buffer is sized for the
    largest tile), with users of 2017, 4033 and 6000 ratings (two and three 2016-rating parts) in the first tile."""
    rng = np.random.default_rng(29)
    nu, ni = SCALE_ROWS, 6500
    u = [np.repeat(np.arange(nu, dtype=np.int32), 3)]
    i = [rng.integers(0, ni, 3 * nu).astype(np.int32)]
    for j, d in enumerate(SCALE_HEAVY):
        u.append(np.full(d, j, np.int32))
        i.append(rng.choice(ni, d, replace=False).astype(np.int32))
    u, i = np.concatenate(u), np.concatenate(i)
    r = rng.integers(1, 6, u.shape[0]).astype(np.float32)
    if implicit:
        r = implicit_prefs(u, i, r, 3)
    _, ru = one_iteration(native, monkeypatch, nu, ni, u, i, r, rank, implicit, {})
    assert (ru.deg > 0).sum() == SCALE_ROWS and ru.deg.max() > 2 * 2016


# ---- tiny sides ----------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("n_items,env", [(n, {"PIO_ALS_TC": "1"}) for n in (1, 2, 3, 7, 8, 9)] +
                         [(n, {}) for n in (1, 3, 5)],
                         ids=[f"wgmma-{n}" for n in (1, 2, 3, 7, 8, 9)] + [f"pair-{n}" for n in (1, 3, 5)])
def test_tiny_sides(native, monkeypatch, n_items, env):
    """Fewer item rows than the wgmma kernel holds in flight per CTA (8), and odd row counts on the pair kernel (the
    last warp's second matrix is a dummy).  Item 0 has 1100 ratings: three wgmma segments, three pair parts.  Explicit
    ratings: the user rows see at most nine item rows, too few for an implicit row without a positive preference."""
    rng = np.random.default_rng(n_items)
    nu, ni = 2000, n_items + 3          # three items never rated
    degs = [1100] + list(rng.integers(1, 700, n_items - 1))
    i = np.repeat(np.arange(n_items, dtype=np.int32), degs)
    u = np.concatenate([rng.choice(nu, d, replace=False) for d in degs]).astype(np.int32)
    r = rng.integers(1, 6, u.shape[0]).astype(np.float32)
    ri, _ = one_iteration(native, monkeypatch, nu, ni, u, i, r, 64, False, env)
    assert (ri.deg > 0).sum() == n_items


# ---- launch-partition invariance ---------------------------------------------------------------------------------
def test_pair_kernel_partition_invariance(native, monkeypatch):
    """Each row's arithmetic on the pair kernel depends on that row alone: the warps per CTA and the pieces the row
    range is launched in (which change how rows are paired inside a warp) leave every factor bit-identical."""
    nu, ni, rank = 3000, 300, 48
    u, i, r = synth.synth_ratings(nu, ni, 40000, seed=5, implicit=True)
    r = implicit_prefs(u, i, r, 5)
    u0 = synth.synth_init_factors(nu, rank, 2, 0)

    def train(env):
        set_env(monkeypatch, env)
        m = native.NativeALS(rank, nu, ni, lam=LAM, implicit=True, alpha=ALPHA)
        m.set_ratings(u, i, r)
        m.set_init(u0)
        m.run(2)
        out = m.get_factors()
        assert (m.phase_ms()["item_kernel"], m.phase_ms()["user_kernel"]) == ("pair", "pair")
        m.close()
        return out

    base = train({})
    for w, p in itertools.product((1, 2, 4, 6, 12), (1, 3, 8)):
        got = train({"PIO_ALS_PAIR_WARPS": str(w), "PIO_ALS_PIECES": str(p)})
        assert np.array_equal(got[0], base[0]) and np.array_equal(got[1], base[1]), (w, p)
