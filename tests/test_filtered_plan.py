"""CPU: the planner's rules for filtered batch calls (csrc/score_plan.h), compiled alone with g++ like
tests/test_scoring_plan.py does for the plain calls.

A filtered call splits into white-listed queries (the listed route: one CTA per query, one candidate list per warp) and
scanned queries (the batch kernels in their filtered instantiation, never the single-query or arena routes).  Checked at
the boundaries: 16 / 17 users, topk 32 / 33 and 128 / 129, padded rank 64 / 128, 8 / 9 valid vectors per query, and the
listed / scanned split itself."""
import re
import shutil
import subprocess
from collections import namedtuple
from pathlib import Path

import pytest

ROOT = Path(__file__).resolve().parent.parent
CSRC = ROOT / "incubator-predictionio_b200" / "csrc"
SMEM_OPTIN = 227 * 1024
ROUTE_BATCH, ROUTE_PER_QUERY = 3, 4

DRIVER = r"""
#include <cstdio>
#include <iostream>
#include "score_plan.h"
using namespace pio;
static void print(const ScorePlan& p) {
  printf("%d %u %u %u %d %d %d %d %d %d %d %zu %d\n", (int)p.route, p.kernel, p.launch_bits(), p.path(), p.threads, p.gx,
         p.ngroups, p.qpg, p.lists, p.pass_k, p.passes, p.smem, (int)p.filtered);
}
int main() {
  char op;
  int blocked;
  ScoreEnv e;
  e.serve_fused = true;
  while (std::cin >> op >> e.kp >> e.sm_count >> e.n_internal >> blocked) {
    e.score_blocked = blocked != 0;
    if (op == 'R') {
      int n, topk;
      std::cin >> n >> topk;
      print(plan_recommend_filtered(e, n, topk));
    } else if (op == 'L') {
      int n, topk;
      std::cin >> n >> topk;
      print(plan_listed(n, topk));
    } else if (op == 'S') {
      int n, topk;
      long long total;
      std::cin >> n >> total >> topk;
      print(plan_similar_filtered(n, total, topk));
    } else if (op == 'B') {   // the scanned queries once gathered: plan_similar_batch, marked filtered by the caller
      int topk, n;
      std::cin >> topk >> n;
      std::vector<int> nv(n), q0;
      for (int& v : nv) std::cin >> v;
      ScorePlan p = plan_similar_batch(e, nv, topk, &q0);
      if (p.route == ROUTE_BATCH) p.filtered = true;
      print(p);
    } else if (op == 'P') {   // split: n flags follow
      int n;
      std::cin >> n;
      std::vector<unsigned char> wl(n);
      for (auto& w : wl) { int x; std::cin >> x; w = (unsigned char)x; }
      std::vector<int> listed, scanned;
      split_listed(n ? wl.data() : nullptr, n, &listed, &scanned);
      printf("%zu", listed.size());
      for (int x : listed) printf(" %d", x);
      printf(" |");
      for (int x : scanned) printf(" %d", x);
      printf("\n");
    }
  }
}
"""

Plan = namedtuple("Plan", "route kernel launch_bits path threads gx ngroups qpg lists pass_k passes smem filtered")


def _consts():
    env = {}
    for f in ("topk_geometry.h", "score_plan.h"):
        for name, expr in re.findall(r"^constexpr int (\w+) = ([^;]+);", (CSRC / f).read_text(), re.M):
            env[name] = int(eval(expr, {}, dict(env)))
    return env


def _bits():
    text = (ROOT / "include" / "pio_als.h").read_text()
    return {name.lower(): int(v, 16) for name, v in re.findall(r"#define PIO_ALS_F?PATH_(\w+) (0x[0-9a-fA-F]+)", text)}


C, BITS = _consts(), _bits()


@pytest.fixture(scope="module")
def run(tmp_path_factory):
    if shutil.which("g++") is None:
        pytest.skip("needs g++")
    d = tmp_path_factory.mktemp("filtered_plan")
    (d / "driver.cc").write_text(DRIVER)
    subprocess.run(["g++", "-std=c++17", "-O1", "-I", str(CSRC), "-o", str(d / "driver"), str(d / "driver.cc")], check=True)

    def call(*request):
        text = " ".join(str(int(x)) if not isinstance(x, str) else x for x in request) + "\n"
        return subprocess.run([str(d / "driver")], input=text, capture_output=True, text=True, check=True).stdout.strip()

    return call


def plan(run, *request):
    return Plan(*[int(x) for x in run(*request).split()])


def names(bits):
    return {n for n, b in BITS.items() if bits & b}


def test_the_new_path_bits_are_free_bits():
    assert BITS["filtered"] == 0x100 and BITS["listed"] == 0x200
    assert len(set(BITS.values())) == len(BITS)


@pytest.mark.parametrize("kp", [16, 32, 64, 128])
@pytest.mark.parametrize("blocked", [1, 0])
def test_scanned_users_take_the_batch_kernels_whatever_their_number(run, kp, blocked):
    for n in (1, 2, 16, 17, 4100):
        for topk in (1, 32, 33, 128, 129, 300):
            p = plan(run, "R", kp, 132, 100_000, blocked, n, topk)
            want = "dot_blocked" if blocked and kp <= 64 and topk <= C["DB_MAXK"] else "dot_batched"
            assert p.route == ROUTE_BATCH and p.filtered == 1
            assert names(p.launch_bits) == {want, "filtered"}
            assert names(p.path) == {want, "filtered"} | ({"multi_pass"} if topk > C["TK_MAXK"] else set())
            assert p.ngroups == -(-n // C["SB_QB"]) and p.qpg == C["SB_QB"]
            assert p.pass_k == min(topk, C["TK_MAXK"]) and p.passes == -(-topk // C["TK_MAXK"])
            assert 0 < p.smem <= SMEM_OPTIN and p.gx >= 1
            assert p.lists == p.gx * (C["DB_RINGS"] if want == "dot_blocked" else 1)


def test_listed_queries_get_one_cta_each(run):
    for n in (1, 17, 40_000):
        for topk in (1, 32, 33, 128, 129, 300):
            p = plan(run, "L", 64, 132, 100_000, 1, n, topk)
            assert p.route == ROUTE_BATCH and names(p.kernel) == {"listed"} and p.filtered == 0
            assert names(p.path) == {"listed"} | ({"multi_pass"} if topk > C["TK_MAXK"] else set())
            assert (p.threads, p.gx, p.ngroups, p.qpg, p.lists) == (C["LS_THREADS"], 1, n, 1, C["LS_WARPS"])
            assert p.smem == 12 * C["LS_WARPS"] * min(topk, C["TK_MAXK"])
    assert plan(run, "L", 64, 132, 100_000, 1, 0, 10).route == 0


def test_scanned_similar_queries_never_take_the_single_query_routes(run):
    assert plan(run, "S", 64, 132, 100_000, 1, 1, 3, 10).route == ROUTE_BATCH          # one query of three ids
    assert plan(run, "S", 64, 132, 100_000, 1, 5, 0, 10).route == ROUTE_PER_QUERY      # nothing to gather
    assert plan(run, "S", 64, 132, 100_000, 1, 5, 1 << 31, 10).route == ROUTE_PER_QUERY
    assert plan(run, "S", 64, 132, 100_000, 1, 0, 0, 10).route == 0


def test_gathered_scanned_queries_keep_the_similar_batch_rules(run):
    for kp in (64, 128):
        for topk in (32, 33):
            for nv in (8, 9):
                p = plan(run, "B", kp, 132, 100_000, 1, topk, 3, 1, nv, 2)
                s3 = kp <= 64 and topk <= C["DB_MAXK"] and nv <= C["DB_QW"]
                assert p.route == ROUTE_BATCH and p.filtered == 1
                assert names(p.launch_bits) == {"cos_blocked" if s3 else "cos_multi", "filtered"}
                assert 0 < p.smem <= SMEM_OPTIN
    # more than SM_NV vectors in a group of SM_QG queries: one query at a time, no filtered kernel
    p = plan(run, "B", 64, 132, 100_000, 1, 10, 2, C["SM_NV"] + 1, 1)
    assert p.route == ROUTE_PER_QUERY and p.filtered == 0 and p.kernel == 0


def test_split_keeps_the_call_order(run):
    assert run("P", 64, 132, 1000, 1, 6, 0, 1, 1, 0, 0, 1) == "3 1 2 5 | 0 3 4"
    assert run("P", 64, 132, 1000, 1, 3, 0, 0, 0) == "0 | 0 1 2"
    assert run("P", 64, 132, 1000, 1, 2, 1, 1) == "2 0 1 |"
