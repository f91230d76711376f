"""CPU: the scoring planner (csrc/score_plan.h) against the dispatch rules tests/test_gpu_scoring.py restates.

A small driver is compiled against score_plan.h alone, with g++, and asked for the plan of every call on ladders of
padded rank, query count, topk, query length and valid-vector pattern around each threshold.  The kernels and path bits
must be those rec_path / sim_path predict (the GPU test asserts the same bits against pio_als_stats.last_score_path), the
S5 shared memory must be s5_smem, and every plan must fit the device.  The constants of topk_geometry.h must still be
those of the GPU test, and its ladders must still straddle every threshold."""
import re
import shutil
import subprocess
from collections import namedtuple
from pathlib import Path

import numpy as np
import pytest

import test_gpu_scoring as G

ROOT = Path(__file__).resolve().parent.parent
CSRC = ROOT / "incubator-predictionio_b200" / "csrc"
SMEM_OPTIN = 227 * 1024       # largest dynamic shared memory a block may opt into (H100)
KPS = (16, 32, 64, 128)
TOPKS = (1, 32, 33, 128, 129, 256, 257)
ROUTE = {"none": 0, "one": 1, "arena": 2, "batch": 3, "per_query": 4}

DRIVER = r"""
#include <cstdio>
#include <iostream>
#include "score_plan.h"
using namespace pio;
static void print(const ScorePlan& p, const std::vector<int>& q0) {
  printf("%d %u %u %d %d %d %d %d %d %d %d %zu %d", (int)p.route, p.kernel, p.path(), p.threads, p.gx, p.ngroups, p.qpg,
         p.chunk, p.lists, p.pass_k, p.passes, p.smem, p.nvp);
  for (int x : q0) printf(" %d", x);
  printf("\n");
}
int main() {
  char op;
  int fused, blocked;
  ScoreEnv e;
  while (std::cin >> op >> e.kp >> e.sm_count >> e.n_internal >> fused >> blocked) {
    e.serve_fused = fused != 0;
    e.score_blocked = blocked != 0;
    std::vector<int> q0;
    if (op == 'R') {
      int n, topk;
      std::cin >> n >> topk;
      print(plan_recommend(e, n, topk), q0);
    } else if (op == 'S') {
      int nq, topk;
      long long len0, total;
      std::cin >> nq >> len0 >> total >> topk;
      print(plan_similar(e, nq, len0, total, topk), q0);
    } else if (op == 'B') {
      int topk, n;
      std::cin >> topk >> n;
      std::vector<int> nv(n);
      for (int& v : nv) std::cin >> v;
      print(plan_similar_batch(e, nv, topk, &q0), q0);
    } else if (op == 'Q') {
      int nqv, nq, topk;
      std::cin >> nqv >> nq >> topk;
      print(plan_similar_query(e, nqv, nq, topk), q0);
    }
  }
}
"""

Plan = namedtuple("Plan", "route kernel path threads gx ngroups qpg chunk lists pass_k passes smem nvp q0")


def _geometry():
    env = {}
    for f in ("topk_geometry.h", "score_plan.h"):
        for name, expr in re.findall(r"^constexpr int (\w+) = ([^;]+);", (CSRC / f).read_text(), re.M):
            env[name] = int(eval(expr, {}, dict(env)))   # integer literals and earlier constants only
    return env


def _path_bits():
    text = (ROOT / "include" / "pio_als.h").read_text()
    return {name.lower(): int(v, 16) for name, v in re.findall(r"#define PIO_ALS_PATH_(\w+) (0x[0-9a-fA-F]+)", text)}


BITS = _path_bits()


def names(path):
    return {n for n, b in BITS.items() if path & b}


class Planner:
    def __init__(self, exe):
        self.exe = exe

    def run(self, requests):
        text = "\n".join(" ".join(str(int(x)) if not isinstance(x, str) else x for x in r) for r in requests) + "\n"
        out = subprocess.run([str(self.exe)], input=text, capture_output=True, text=True, check=True).stdout.splitlines()
        assert len(out) == len(requests)
        plans = []
        for line in out:
            v = [int(x) for x in line.split()]
            plans.append(Plan(*v[:13], v[13:]))
        return plans

    def one(self, *request):
        return self.run([request])[0]


def env(kp, sm=132, n_items=100_000, fused=1, blocked=1):
    return (kp, sm, n_items, fused, blocked)


@pytest.fixture(scope="module")
def planner(tmp_path_factory):
    if shutil.which("g++") is None:
        pytest.skip("needs g++")
    d = tmp_path_factory.mktemp("score_plan")
    (d / "driver.cpp").write_text(DRIVER)
    exe = d / "driver"
    subprocess.run(["g++", "-std=c++17", "-Wall", "-Wextra", "-Werror", "-O1", "-I", str(CSRC), "-o", str(exe),
                    str(d / "driver.cpp")], check=True)
    return Planner(exe)


# the item-validity array of the similar ladders: ids below HALF own a factor, the rest do not
N_IH, HALF = 1000, 500
IH = (np.arange(N_IH) < HALF).astype(np.uint8)


def query(n_valid, n_invalid=0, n_unknown=0, start=0):
    """n_valid ids with a factor, n_invalid without, n_unknown out of range"""
    return ([start + t for t in range(n_valid)] + [HALF + start + t for t in range(n_invalid)] +
            [N_IH + t if t % 2 else -1 - t for t in range(n_unknown)])


def similar_plans(P, e, queries, topk):
    """the plans one pio_als_similar_batch call runs through, in the order pio_als.cu asks for them"""
    lens = [len(q) for q in queries]
    first = P.one("S", *e, len(queries), lens[0], sum(lens), topk)
    if first.route in (ROUTE["one"], ROUTE["arena"], ROUTE["none"]):
        return [first]
    if first.route == ROUTE["batch"]:
        nv = [G._n_valid(q, IH) for q in queries]
        b = P.one("B", *e, topk, len(nv), *nv)
        if b.route == ROUTE["batch"]:
            return [first, b]
    return [P.one("Q", *e, G._n_valid(q, IH), len(q), topk) for q in queries]


def similar_path(P, e, queries, topk):
    out = set()
    for p in similar_plans(P, e, queries, topk):
        out |= names(p.path)
    return out


def test_constants_match_sources():
    c = _geometry()
    for name in ("TK_MAXK", "DB_MAXK", "SB_QB", "S1_MAXNV", "SM_NV", "SM_QG", "SM_QIDS", "DB_QW", "CB_QPW", "DB_WPR",
                 "SB_THREADS", "SC_G", "GROUP_CHUNK"):
        assert getattr(G, name) == c[name], (name, getattr(G, name), c[name])
    assert set(BITS) == {"score_one", "dot_blocked", "cos_blocked", "dot_batched", "cos_multi", "cos_batched",
                         "cos_fallback", "multi_pass"}


def test_recommend_plans_match_the_gpu_test(planner):
    reqs, want = [], []
    for kp in KPS:
        for n in (1, 2, 16, 17, 1000, G.SPLIT_USERS):
            for topk in TOPKS:
                reqs.append(("R", *env(kp), n, topk))
                want.append((kp, n, topk))
    for (kp, n, topk), p in zip(want, planner.run(reqs)):
        assert names(p.path) == G.rec_path(kp, n, topk), (kp, n, topk, p)
        if p.route == ROUTE["batch"]:    # groups of SB_QB users, at most GROUP_CHUNK of them per launch
            assert p.qpg == G.SB_QB and p.ngroups == -(-n // G.SB_QB) and p.chunk == G.GROUP_CHUNK
            assert p.passes == -(-topk // G.TK_MAXK) and p.pass_k == min(topk, G.TK_MAXK)
        if n == G.SPLIT_USERS:
            assert p.ngroups > p.chunk    # the grid.y split runs


def test_similar_single_query_plans_match_the_gpu_test(planner):
    shapes = [(v, i, u) for v in (0, 1, 2, 3, 4, 5, 8, 9, 37, 40, 41, 56, 57, 70) for i in (0, 3) for u in (0, 2)]
    for kp in KPS:
        for topk in TOPKS:
            for v, i, u in shapes:
                q = query(v, i, u)
                if not q:
                    continue
                got = similar_path(planner, env(kp), [q], topk)
                assert got == G.sim_path(kp, [q], IH, topk), (kp, topk, v, i, u, got)


def test_similar_batch_plans_match_the_gpu_test(planner):
    batches = {
        "empty": [[], []],
        "two": [query(1), query(2, 1)],
        "db_qw": [query(8), query(8, 3), query(1)] * 6,
        "db_qw+1": [query(8), query(9), query(2)] * 6,
        "no_valid": [query(0, 2), query(0, 1, 1)] * 9,
        "group_40": [query(5)] * 8 + [query(3, 1)] * 9,
        "group_41": [query(5)] * 7 + [query(6)] + [query(3)] * 9,
        "bins": [query(v % 9, v % 3) for v in range(40)],
        "one_empty": [query(3), []] * 8 + [query(1)],
        "long_ids": [query(4, G.LONG_QUERY_IDS - 4), query(2)] * 3,
    }
    for kp in KPS:
        for topk in TOPKS:
            for what, qs in batches.items():
                got = similar_path(planner, env(kp), qs, topk)
                assert got == G.sim_path(kp, qs, IH, topk), (kp, topk, what, got)


def test_similar_batch_groups(planner):
    # S3 bins: consecutive queries, <= CB_QPW queries and <= DB_QW vectors each, a new bin only when the next query does
    # not fit; S4: groups of SM_QG queries
    for nv in ([(7 * j) % 9 for j in range(101)], [j % 2 for j in range(37)] + [1] * 21 + [0, 8, 0, 0, 0, 0, 2]):
        p = planner.one("B", *env(64), 10, len(nv), *nv)
        assert p.kernel == BITS["cos_blocked"] and p.qpg == 0 and p.chunk == G.GROUP_CHUNK
        q0 = p.q0
        assert q0[0] == 0 and q0[-1] == len(nv) and q0 == sorted(set(q0))
        for a, b in zip(q0, q0[1:]):
            assert b - a <= G.CB_QPW and sum(nv[a:b]) <= G.DB_QW
            if b < len(nv):
                assert b - a == G.CB_QPW or sum(nv[a:b + 1]) > G.DB_QW
        assert p.ngroups == -(-(len(q0) - 1) // G.DB_WPR)
    p = planner.one("B", *env(128), 10, len(nv), *nv)
    assert p.kernel == BITS["cos_multi"] and p.qpg == G.SM_QG and p.chunk == G.GROUP_CHUNK
    assert p.q0 == list(range(0, len(nv), G.SM_QG)) + [len(nv)] and p.ngroups == -(-len(nv) // G.SM_QG)
    # more query groups than one grid holds
    p = planner.one("B", *env(128), 10, G.SPLIT_QUERIES, *([1] * G.SPLIT_QUERIES))
    assert p.kernel == BITS["cos_multi"] and p.ngroups > p.chunk


def test_s5_shared_memory_matches_the_gpu_test(planner):
    reqs, want = [], []
    for kp in KPS:
        for topk in (1, 20, 128, 129, 300):
            for nqv in range(0, 200):
                for extra in (0, 3):
                    reqs.append(("Q", *env(kp), nqv, nqv + extra, topk))
                    want.append((kp, nqv, nqv + extra, topk))
    for (kp, nqv, nq, topk), p in zip(want, planner.run(reqs)):
        if nqv == 0:    # no valid vector: nothing to score
            assert p.route == ROUTE["none"] and p.path == 0
            continue
        smem = G.s5_smem(kp, nqv, nq, topk)
        if smem <= G.S5_SMEM_LIMIT:
            assert p.kernel == BITS["cos_batched"] and p.smem == smem, (kp, nqv, nq, topk, p)
        else:
            assert p.kernel == BITS["cos_fallback"] and p.smem == 0, (kp, nqv, nq, topk, p)
        assert names(p.path) == G._s5_path(kp, query(nqv, nq - nqv), IH, topk)


def test_switches_off_give_the_older_kernels(planner):
    for kp in (16, 32, 64):
        on, off_fused, off_blocked = env(kp), env(kp, fused=0), env(kp, blocked=0)
        assert planner.one("R", *on, 1, 10).kernel == BITS["score_one"]
        p = planner.one("R", *off_fused, 1, 10)
        assert p.kernel == BITS["dot_batched"] and p.route == ROUTE["arena"]
        assert planner.one("R", *on, 100, 10).kernel == BITS["dot_blocked"]
        p = planner.one("R", *off_blocked, 100, 10)
        assert p.kernel == BITS["dot_batched"] and p.route == ROUTE["batch"]
        assert similar_path(planner, on, [query(3)], 10) == {"score_one"}
        assert similar_path(planner, off_fused, [query(3)], 10) == {"cos_multi"}
        qs = [query(2), query(3)] * 5
        assert similar_path(planner, on, qs, 10) == {"cos_blocked"}
        assert similar_path(planner, off_blocked, qs, 10) == {"cos_multi"}


def test_plans_fit_the_device(planner):
    reqs = []
    for kp in KPS:
        for sm in (1, 2, 132, 300):
            for n_items in (1, 2, 255, 257, 100_000, 30_000_000):
                e = env(kp, sm, n_items)
                for topk in TOPKS + (1000,):
                    reqs += [("R", *e, n, topk) for n in (1, 2, 16, 17, 100_000)]
                    reqs += [("S", *e, 1, n, n, topk) for n in (1, 2, 3, 5, 8, 40)]
                    reqs += [("B", *e, topk, 3, 1, 8, 0), ("B", *e, topk, 9, *([5] * 9))]
                    reqs += [("Q", *e, nqv, nqv + 3, topk) for nqv in (1, 8, 57, 500)]
    plans = planner.run(reqs)
    for r, p in zip(reqs, plans):
        assert p.smem <= SMEM_OPTIN, (r, p)
        if p.kernel:
            assert p.gx >= 1 and p.lists >= p.gx and p.threads in (256, 512), (r, p)
        if p.kernel == BITS["score_one"]:
            assert p.gx <= _geometry()["S1_THREADS"] and p.nvp in (1, 2, 4, 8), (r, p)


def test_ladders_straddle_every_threshold():
    c = _geometry()
    topks = set(G.MULTI_TOPK) | {1, 10, 32, 33, 128}
    assert {c["DB_MAXK"], c["DB_MAXK"] + 1, c["TK_MAXK"], c["TK_MAXK"] + 1, 2 * c["TK_MAXK"], 2 * c["TK_MAXK"] + 1} <= topks
    assert max(G.MULTI_TOPK) > 3 * c["TK_MAXK"]
    # equal-score blocks covering ranks t - 1 and t for every topk boundary t
    for t in (1, 10, c["DB_MAXK"], c["TK_MAXK"], 2 * c["TK_MAXK"]):
        assert any(s <= t - 1 and s + n > t for s, n in G.TIE_BLOCKS), t
    assert max(n for _, n in G.TIE_BLOCKS) >= 300
    # item counts around one warp, one tile of SB_THREADS items, one blocked step of DB_RINGS * DB_ROWS rows and TK_TILE
    items = set(G.ITEM_LADDER)
    for t in (32, c["SB_THREADS"], c["DB_RINGS"] * c["DB_ROWS"], c["TK_TILE"]):
        assert {t - 1, t + 1} <= items, t
    assert {1, 2} <= items
    # the smallest and largest rank, and the first rank of every padded width (KP 16, 32, 64, 128) beside the last of the
    # width below it
    assert {1, 16, 17, 33, 64, 65, 128} <= set(G.RANKS)
    # one similar query: S2 takes up to SM_NV query ids, valid or not; one id more goes to S5.  A batch: S4 takes 8-query
    # groups of up to SM_NV valid vectors; one vector more sends it to S5.
    assert set(G.S2_QUERY_IDS) == {c["SM_NV"], c["SM_NV"] + 1}
    assert set(G.GROUP_VECTORS) == {c["SM_NV"], c["SM_NV"] + 1}
    assert G.SM_QG == c["SM_QG"] and max(G.GROUP_VECTORS) // 4 > c["DB_QW"]   # the 4-query groups stay off the blocked kernel
    # the S5 shared-memory / fallback boundary at KP 64, topk 20 (the GPU test's S5 queries carry three invalid ids
    # besides nv valid ones); test_s5_shared_memory_matches_the_gpu_test ties s5_smem to the planner
    batched = [nv for nv in range(1, 200) if G.s5_smem(64, nv, nv + 3, 20) <= G.S5_SMEM_LIMIT]
    last = max(batched)
    assert batched == list(range(1, last + 1))
    assert {last, last + 1} <= set(G.S5_QUERY_VALID), (last, G.S5_QUERY_VALID)
    assert min(G.S5_QUERY_VALID) + 3 > c["SM_NV"]                        # every such query has more than SM_NV ids
    assert G.s5_smem(128, 1, 1, 1) > G.S5_SMEM_LIMIT          # KP 128 always takes the fallback kernel
    assert G.LONG_QUERY_IDS > c["SM_QIDS"]
    # more query groups than one grid holds, on both batch paths
    assert G.SPLIT_USERS > G.GROUP_CHUNK * c["SB_QB"]
    assert G.SPLIT_QUERIES > G.GROUP_CHUNK * c["SM_QG"]
