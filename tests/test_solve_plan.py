"""CPU: the ALS solve planner (csrc/solve_plan.h) against the path rules tests/test_gpu_halfstep.py restates.

A small driver is compiled against solve_plan.h alone, with g++, and asked for the parsed switches, the side plan and
the half-step plan of each request.  The kernel label and heavy-row threshold of every rank and switch setting must be
those path_of predicts (the GPU test asserts the same labels against phase_ms()); each switch must parse as documented
at its edges; and over ladders of row counts, long rows, pieces and world sizes every row, part and long row must be
launched exactly once, with today's grid formulas and caps."""
import shutil
import subprocess
from collections import namedtuple

import numpy as np
import pytest

import test_gpu_halfstep as G

CSRC = G.CSRC

# constants the GPU tests and the kernels are built around, restated so that a change to the planner shows here
PART, PAIR_PART, LS128_TILE, TC_TILE = 2016, 512, 32768, 1 << 20
NG = {16: 25, 32: 25, 64: 7, 128: 2}              # SolveCfg::NG: rows per CTA of the FP32 kernel
MMA_ROWS, TC_ROWS, TC_SOLVE_ROWS, FIN128_ROWS, FINISH_ROWS, PAIR_WARPS_PER_SM = 4, 8, 4, 6, 4, 12
LABEL = {0: "fp32", 1: "wgmma", 2: "mma", 3: "pair"}
PARTS, FINISH, LS128_TILE_ST, LS128_FINISH, ROWS, TC_SOLVE = range(6)

DRIVER = r"""
#include <cstdio>
#include <iostream>
#include <map>
#include <string>
#include "solve_plan.h"
using namespace pio;
static std::map<std::string, std::string> g_env;
static const char* env(const char* k) {
  auto it = g_env.find(k);
  return it == g_env.end() ? nullptr : it->second.c_str();
}
int main() {
  int kp, world, n_env;
  while (std::cin >> kp >> world >> n_env) {
    g_env.clear();
    for (int i = 0; i < n_env; ++i) {
      std::string kv;
      std::cin >> kv;
      const size_t eq = kv.find('=');
      g_env[kv.substr(0, eq)] = kv.substr(eq + 1);
    }
    int n_rows, sm, R, n_active, n_heavy, n_parts;
    long long nnz;
    std::cin >> n_rows >> nnz >> sm >> R >> n_active >> n_heavy >> n_parts;
    std::vector<int> rpp(n_heavy + 1);
    for (int& x : rpp) std::cin >> x;
    const SolveSwitches s = read_solve_switches(env, kp, world);
    printf("%d %.17g %d %d %d %d %d %d %d %d %d |", s.tc, s.tc_min_deg, s.tc_split, s.tc_timing, s.tc_debug, s.mma,
           s.pair, s.pair_seg_t, s.pair_part, s.pair_warps, s.n_pieces);
    const SidePlan sp = plan_side(s, kp, n_rows, nnz);
    printf(" %d %d %d %d |", (int)sp.kernel, phase_code(sp.kernel), sp.heavy_t, sp.part_len);
    const SolvePlan p = plan_half_step(s, sp, kp, sm, R, n_active, n_heavy, n_parts, rpp);
    printf(" %d %lld |", p.n_aux, p.partial_parts);
    for (const SolveLaunch& l : p.launches)
      printf(" %d %d %d %d %d %d %d", (int)l.stage, (int)l.aux, l.row_begin, l.row_end, l.wl_off, l.wl_count, l.grid);
    printf(" |");
    for (int c : p.piece_after) printf(" %d", c);
    printf("\n");
  }
}
"""

Switches = namedtuple("Switches", "tc tc_min_deg tc_split tc_timing tc_debug mma pair seg_t part warps pieces")
Side = namedtuple("Side", "kernel phase heavy_t part_len")
Launch = namedtuple("Launch", "stage aux r0 r1 w0 wc grid")
Result = namedtuple("Result", "sw side n_aux partial_parts launches piece_after")


class Planner:
    def __init__(self, exe):
        self.exe = exe

    def run(self, requests):
        """requests: dicts with kp, env and optionally world, n_rows, nnz, sm, R, n_active, n_heavy, rpp"""
        lines = []
        for q in requests:
            env = q.get("env", {})
            rpp = list(q.get("rpp", [0]))
            n_heavy = len(rpp) - 1
            lines.append(" ".join(str(x) for x in (
                q["kp"], q.get("world", 1), len(env), *(f"{k}={v}" for k, v in env.items()), q.get("n_rows", 1),
                q.get("nnz", 1), q.get("sm", 132), q.get("R", 0), q.get("n_active", n_heavy), n_heavy, rpp[-1], *rpp)))
        out = subprocess.run([str(self.exe)], input="\n".join(lines) + "\n", capture_output=True, text=True,
                             check=True).stdout.splitlines()
        assert len(out) == len(requests)
        res = []
        for line in out:
            sw, side, head, launches, pieces = line.split("|")
            sw = sw.split()
            l = [int(x) for x in launches.split()]
            n_aux, partial = (int(x) for x in head.split())
            res.append(Result(Switches(*(float(x) if i == 1 else int(x) for i, x in enumerate(sw))),
                              Side(*(int(x) for x in side.split())), n_aux, partial,
                              [Launch(*l[j:j + 7]) for j in range(0, len(l), 7)], [int(x) for x in pieces.split()]))
        return res

    def one(self, **q):
        return self.run([q])[0]


@pytest.fixture(scope="module")
def planner(tmp_path_factory):
    if shutil.which("g++") is None:
        pytest.skip("needs g++")
    d = tmp_path_factory.mktemp("solve_plan")
    (d / "driver.cpp").write_text(DRIVER)
    exe = d / "driver"
    subprocess.run(["g++", "-std=c++17", "-Wall", "-Wextra", "-Werror", "-O1", "-I", str(CSRC), "-o", str(exe),
                    str(d / "driver.cpp")], check=True)
    return Planner(exe)


def kp_of(rank):
    return 16 if rank <= 16 else 32 if rank <= 32 else 64 if rank <= 64 else 128


# ---- kernel choice ----------------------------------------------------------------------------------------------------
PATH_ENVS = [{}, {"PIO_ALS_TC": "1"}, {"PIO_ALS_MMA": "1"}, {"PIO_ALS_MMA": "0"}, {"PIO_ALS_TC": "1", "PIO_ALS_MMA": "1"},
             {"PIO_ALS_TC": "1", "PIO_ALS_MMA": "0"}, {"PIO_ALS_SEG_T": "64", "PIO_ALS_PART": "40"},
             {"PIO_ALS_SEG_T": "2000"}, {"PIO_ALS_PAIR_WARPS": "12", "PIO_ALS_PIECES": "3"}]


def test_kernel_and_threshold_match_path_of(planner):
    cases = [(rank, env) for rank in range(1, 129) for env in PATH_ENVS]
    reqs = [dict(kp=kp_of(rank), env=env, n_rows=300, nnz=30000) for rank, env in cases]
    for (rank, _), q, r in zip(cases, reqs, planner.run(reqs)):
        label, heavy_t, _ = G.path_of(rank, q["env"])
        assert (LABEL[r.side.phase], r.side.heavy_t) == (label, heavy_t), (q, r.side)
        pair_part = -(-int(q["env"].get("PIO_ALS_PART", PAIR_PART)) // 8) * 8
        assert r.side.part_len == (pair_part if label == "pair" else PART), (q, r.side)
        assert (r.side.kernel == 4) == (q["kp"] == 128)      # LS128: its own route, labelled fp32


def side(planner, env, n_rows, nnz, kp=64):
    r = planner.one(kp=kp, env=env, n_rows=n_rows, nnz=nnz).side
    return LABEL[r.phase], r.heavy_t


def test_rank64_selection_combinations(planner):
    # test_rank64_kernel_selection: 20000 users, 300 items, 400000 ratings (a few fewer after dedup)
    nu, ni, nnz = 20000, 300, 399000
    for env, item, user in (({}, "pair", "pair"), ({"PIO_ALS_TC": "1", "PIO_ALS_TC_MIN_DEG": "256"}, "wgmma", "pair"),
                            ({"PIO_ALS_MMA": "1"}, "mma", "mma"), ({"PIO_ALS_MMA": "0"}, "fp32", "fp32")):
        assert side(planner, env, ni, nnz)[0] == item and side(planner, env, nu, nnz)[0] == user, env
    # TC_MIN_DEG: a side averaging below, at and above the bound; the sides below it fall back to the MMA switch
    for mma, below in ((None, ("pair", 1024)), ("1", ("mma", 8192)), ("0", ("fp32", 4096))):
        env = {"PIO_ALS_TC": "1", "PIO_ALS_TC_MIN_DEG": "256", **({"PIO_ALS_MMA": mma} if mma else {})}
        assert side(planner, env, 100, 25599) == below, env
        assert side(planner, env, 100, 25600) == ("wgmma", 8192), env
        assert side(planner, env, 100, 25601) == ("wgmma", 8192), env
    # no rows, and ranks other than 33..64, never take the wgmma kernel
    assert side(planner, {"PIO_ALS_TC": "1"}, 0, 0) == ("pair", 1024)
    assert side(planner, {"PIO_ALS_TC": "1"}, 10, 100, kp=32) == ("fp32", 4096)
    assert side(planner, {"PIO_ALS_TC": "1"}, 10, 100, kp=128) == ("fp32", 0)


# ---- switch parsing ---------------------------------------------------------------------------------------------------
def switches(planner, env, kp=64, world=1):
    return planner.one(kp=kp, env=env, world=world).sw


def test_switch_parsing_edges(planner):
    d = switches(planner, {})
    assert d == Switches(0, 0.0, 0, 0, 0, 1, 1, 1024, 512, 4, 1)
    for v, on in (("1", 1), ("1x", 1), ("0", 0), ("", 0), ("2", 0), ("01", 0)):
        assert switches(planner, {"PIO_ALS_TC": v}).tc == on, v
    assert switches(planner, {"PIO_ALS_TC": "1"}, kp=32).tc == 0 and switches(planner, {"PIO_ALS_TC": "1"}, kp=128).tc == 0
    for v, mma, pair in (("0", 0, 1), ("1", 1, 0), ("", 1, 1), ("2", 1, 1), ("01", 0, 1), ("10", 1, 0)):
        s = switches(planner, {"PIO_ALS_MMA": v})
        assert (s.mma, s.pair) == (mma, pair), v
    for v, t in (("-5", 1024), ("0", 1024), ("x", 1024), ("1", 1), ("64", 64), ("2000", 2000)):
        assert switches(planner, {"PIO_ALS_SEG_T": v}).seg_t == t, v
    for v, p in (("0", 512), ("7", 512), ("8", 8), ("9", 16), ("40", 40), ("41", 48), ("x", 512)):
        assert switches(planner, {"PIO_ALS_PART": v}).part == p, v
    for v in range(-1, 14):
        assert switches(planner, {"PIO_ALS_PAIR_WARPS": str(v)}).warps == (v if v in (1, 2, 6, 12) else 4), v
    for world, default in ((1, 1), (2, 4), (8, 4)):
        assert switches(planner, {}, world=world).pieces == default
        for v in (-1, 0, 1, 2, 7, 8, 9, 100):
            assert switches(planner, {"PIO_ALS_PIECES": str(v)}, world=world).pieces == (v if 1 <= v <= 8 else default)
    for v, m in (("256", 256.0), ("2.5", 2.5), ("x", 0.0), ("-3", -3.0)):
        assert switches(planner, {"PIO_ALS_TC_MIN_DEG": v}).tc_min_deg == m, v
    for v, on in (("1", 1), ("10", 1), ("0", 0), ("", 0)):
        assert switches(planner, {"PIO_ALS_TC_SPLIT": v}).tc_split == on, v
    for name in ("PIO_ALS_TC_TIMING", "PIO_ALS_TC_DEBUG"):     # any value turns a dump on
        s = switches(planner, {name: "0"})
        assert (s.tc_timing, s.tc_debug) == ((1, 0) if name == "PIO_ALS_TC_TIMING" else (0, 1))


# ---- half-step plans --------------------------------------------------------------------------------------------------
ROUTES = {   # name: (kp, env)
    "fp32-16": (16, {}), "fp32-32": (32, {}), "fp32-64": (64, {"PIO_ALS_MMA": "0"}), "mma": (64, {"PIO_ALS_MMA": "1"}),
    "wgmma": (64, {"PIO_ALS_TC": "1"}), "wgmma-split": (64, {"PIO_ALS_TC": "1", "PIO_ALS_TC_SPLIT": "1"}),
    "pair": (64, {}), "ls128": (128, {}),
}


def row_part_ptr(n_heavy, seed):
    parts = np.random.default_rng(seed).integers(1, 7, n_heavy)
    return np.concatenate([[0], np.cumsum(parts)]).astype(int).tolist()


def expected_grid(route, l, sm, warps):
    n = l.r1 - l.r0
    cdiv = lambda a, b: -(-a // b)
    if route == "pair":
        if l.stage == FINISH:
            return min((n + 1) // 2, PAIR_WARPS_PER_SM * sm)
        items = l.wc if l.stage == PARTS else n
        return min(cdiv(cdiv(items, 2), warps), (PAIR_WARPS_PER_SM // warps) * sm)
    kp = ROUTES[route][0]
    if l.stage in (PARTS, LS128_TILE_ST):
        return cdiv(l.wc, NG[kp])
    if l.stage == FINISH:
        return cdiv(n, FINISH_ROWS)
    if l.stage == LS128_FINISH:
        return min(cdiv(n, FIN128_ROWS), sm)
    if l.stage == TC_SOLVE:
        return min(cdiv(n, TC_SOLVE_ROWS), 4 * sm)
    if route.startswith("wgmma"):
        return min(cdiv(n, TC_ROWS), sm)
    return cdiv(n, MMA_ROWS if route == "mma" else NG[kp])


def check_plan(route, q, r):
    """coverage, grids, streams, events and launch count of one half-step plan"""
    R, n_active, rpp = q["R"], q["n_active"], q["rpp"]
    n_heavy, n_parts = len(rpp) - 1, rpp[-1]
    warps, pieces = r.sw.warps, r.sw.pieces
    rows, parts, fin = np.zeros(R, int), np.zeros(n_parts, int), np.zeros(max(n_heavy, 1), int)
    tile_parts = 0
    for j, l in enumerate(r.launches):
        assert l.grid == expected_grid(route, l, q["sm"], warps) and l.grid >= 1, (route, q["sm"], l)
        assert l.aux == (route == "pair" and l.stage in (PARTS, FINISH)), l
        if l.stage in (PARTS, LS128_TILE_ST):
            parts[l.w0:l.w0 + l.wc] += 1
        if l.stage in (FINISH, LS128_FINISH):
            fin[l.r0:l.r1] += 1
        if l.stage == ROWS:
            rows[l.r0:l.r1] += 1
        if l.stage in (PARTS, FINISH):
            assert (l.r0, l.r1, l.w0, l.wc) == (0, n_heavy, 0, n_parts), l
        if l.stage in (LS128_TILE_ST, LS128_FINISH):   # a tile's parts are exactly those of its rows
            assert l.r1 - l.r0 <= LS128_TILE and (l.w0, l.wc) == (rpp[l.r0], rpp[l.r1] - rpp[l.r0]), l
            tile_parts = max(tile_parts, l.wc)
        if l.stage == LS128_FINISH:
            assert r.launches[j - 1].stage == LS128_TILE_ST and r.launches[j - 1][2:6] == l[2:6]
        if l.stage == TC_SOLVE:
            assert r.launches[j - 1].stage == ROWS and r.launches[j - 1][2:4] == l[2:4]
    assert (parts == 1).all(), route
    assert (fin[:n_heavy] == 1).all(), route
    lo = n_active if route == "ls128" else n_heavy    # LS128: every active row is finished from parts
    assert (rows[lo:n_active] == 1).all() and (rows[:lo] == 0).all() and (rows[n_active:] == 0).all(), route
    assert r.partial_parts == (tile_parts if route == "ls128" else n_parts if n_heavy else 0)
    # the aux launches come first; ev_piece once per piece on the pair path, including empty pieces
    assert r.n_aux == sum(l.aux for l in r.launches) and all(l.aux for l in r.launches[:r.n_aux])
    if route == "pair":
        assert len(r.piece_after) == pieces and r.piece_after == sorted(r.piece_after)
        assert r.piece_after[0] >= r.n_aux and r.piece_after[-1] == len(r.launches)
        for c in range(pieces):     # piece c's rows, and nothing after them, are launched before ev_piece[c]
            plo, phi = R * c // pieces, R * (c + 1) // pieces
            done = r.launches[:r.piece_after[c]]
            assert all(l.r1 <= phi for l in done if l.stage == ROWS)
            if min(phi, n_active) > max(plo, n_heavy):
                assert done[-1].stage == ROWS and (done[-1].r0, done[-1].r1) == (max(plo, n_heavy), min(phi, n_active))
    else:
        assert r.piece_after == []
    # solve launches of the half-step (pio_als_stats.solve_launches counts one per entry)
    nlight, cdiv = n_active - n_heavy, lambda a, b: -(-a // b)
    heavy = 2 if n_heavy else 0
    if route == "pair":
        want = heavy + sum(min(R * (c + 1) // pieces, n_active) > max(R * c // pieces, n_heavy) for c in range(pieces))
    elif route == "ls128":
        want = 2 * cdiv(n_heavy, LS128_TILE)
    elif route.startswith("wgmma"):
        want = heavy + (cdiv(nlight, TC_TILE) * 2 if route == "wgmma-split" else int(nlight > 0))
    else:
        want = heavy + int(nlight > 0)
    assert len(r.launches) == want, (route, len(r.launches), want)


def test_every_row_and_part_launched_once(planner):
    reqs = []
    for route, (kp, env) in ROUTES.items():
        for world in (1, 2, 8):
            for pieces in (None,) + tuple(range(1, 9)):
                if pieces and route != "pair":
                    continue
                e = {**env, **({"PIO_ALS_PIECES": str(pieces)} if pieces else {})}
                for R in (1, 2, 7, 100, 1001):
                    for n_active in sorted({0, 1, R // 2, R - 1, R}):
                        heavies = [n_active] if route == "ls128" else sorted({0, 1, n_active // 3, n_active})
                        for n_heavy in (h for h in heavies if h <= n_active):
                            for sm in (1, 3, 132):
                                reqs.append((route, dict(kp=kp, env=e, world=world, R=R, n_active=n_active, sm=sm,
                                                         rpp=row_part_ptr(n_heavy, R + n_heavy))))
    for w in (1, 2, 6, 12, 5):
        reqs.append(("pair", dict(kp=64, env={"PIO_ALS_PAIR_WARPS": str(w)}, R=5000, n_active=4000, sm=2,
                                  rpp=row_part_ptr(300, w))))
    # the wgmma split mode over more rows than one tile, and the rank 65..128 route over more than one tile
    reqs.append(("wgmma-split", dict(kp=64, env=ROUTES["wgmma-split"][1], R=TC_TILE + 10, n_active=TC_TILE + 7, sm=132,
                                     rpp=row_part_ptr(2, 1))))
    reqs.append(("wgmma", dict(kp=64, env=ROUTES["wgmma"][1], R=TC_TILE + 10, n_active=TC_TILE + 7, sm=132,
                               rpp=row_part_ptr(2, 1))))
    for n in (LS128_TILE - 1, LS128_TILE, LS128_TILE + 1, 2 * LS128_TILE + 5):
        reqs.append(("ls128", dict(kp=128, env={}, R=n + 3, n_active=n, sm=132, rpp=row_part_ptr(n, n))))
    results = planner.run([q for _, q in reqs])
    for (route, q), r in zip(reqs, results):
        check_plan(route, q, r)


def test_ls128_tiles(planner):
    # 34000 active rows: one tile of 32768 rows and one of 1232; the partial buffer holds the larger tile's parts
    n = G.SCALE_ROWS
    parts = np.ones(n, int)
    parts[:3] = (2, 3, 3)                      # the GPU test's users of 2017, 4033 and 6000 ratings
    parts[LS128_TILE:LS128_TILE + 500] = 4
    rpp = np.concatenate([[0], np.cumsum(parts)]).tolist()
    r = planner.one(kp=128, env={}, R=n, n_active=n, sm=132, rpp=rpp)
    tiles = [(l.r0, l.r1) for l in r.launches if l.stage == LS128_TILE_ST]
    assert tiles == [(0, 32768), (32768, 34000)]
    assert [l.stage for l in r.launches] == [LS128_TILE_ST, LS128_FINISH] * 2
    assert r.partial_parts == 32768 + 2 + 3 == max(rpp[32768] - rpp[0], rpp[34000] - rpp[32768])

