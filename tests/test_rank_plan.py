"""CPU: the product ranking planner (csrc/rank_plan.h) against the plan model in tests/productranking_ref.py.

A small driver is compiled against rank_plan.h alone, with g++, and asked for the parts, radix-path queries and tiles of
list-length ladders around the tile size and of budgets that give parts of 1, 2 and 3 queries."""
import re
import shutil
import subprocess
from pathlib import Path

import numpy as np
import pytest

from tests import productranking_ref as ref

ROOT = Path(__file__).resolve().parent.parent
CSRC = ROOT / "incubator-predictionio_b200" / "csrc"
T = ref.TILE

DRIVER = r"""
#include <cstdio>
#include <iostream>
#include "rank_plan.h"
using namespace pio;
static void list(const std::vector<int>& v) {
  printf(" %zu", v.size());
  for (int x : v) printf(" %d", x);
}
int main() {
  int n;
  long long budget;
  while (std::cin >> budget >> n) {
    std::vector<int64_t> ptr(n + 1);
    for (auto& x : ptr) std::cin >> x;
    const std::vector<RankPart> parts = plan_rank_lists(ptr.data(), n, budget);
    printf("%zu", parts.size());
    for (const RankPart& p : parts) {
      printf(" %d %d %lld %lld", p.q0, p.q1, p.e0, p.e1);
      list(p.radix), list(p.tile_q), list(p.tile_ptr), list(p.tile_off), list(p.tile_n);
    }
    printf("\n");
  }
}
"""
KEYS = ("radix", "tile_q", "tile_ptr", "tile_off", "tile_n")


@pytest.fixture(scope="module")
def planner(tmp_path_factory):
    if shutil.which("g++") is None:
        pytest.skip("needs g++")
    d = tmp_path_factory.mktemp("rank_plan")
    (d / "driver.cpp").write_text(DRIVER)
    exe = d / "driver"
    subprocess.run(["g++", "-std=c++17", "-Wall", "-Wextra", "-Werror", "-O1", "-I", str(CSRC), "-o", str(exe),
                    str(d / "driver.cpp")], check=True)

    def run(cases):
        text = "".join(f"{b} {len(lens)} " + " ".join(map(str, _ptr(lens))) + "\n" for lens, b in cases)
        out = subprocess.run([str(exe)], input=text, capture_output=True, text=True, check=True).stdout.splitlines()
        assert len(out) == len(cases)
        plans = []
        for line in out:
            v = [int(x) for x in line.split()]
            at, parts = 1, []
            for _ in range(v[0]):
                p = dict(zip(("q0", "q1", "e0", "e1"), v[at:at + 4]))
                at += 4
                for k in KEYS:
                    p[k] = v[at + 1:at + 1 + v[at]]
                    at += 1 + v[at]
                parts.append(p)
            assert at == len(v)
            plans.append(parts)
        return plans
    return run


def _ptr(lens):
    return np.concatenate([[0], np.cumsum(lens, dtype=np.int64)]).tolist()


CASES = {
    "around_the_tile": ([T - 1, T, T + 1, 1, T - 1, 2, T + 1, 0, 7], ref.BUDGET),
    "exact_fill": ([1000, 1048, 5, 2043, 3, 0, 2048], ref.BUDGET),
    "one_entry_queries": ([1] * (T + 5), ref.BUDGET),
    "parts_of_1": ([10, 20, 25], 25),
    "parts_of_2": ([10, 20, 30, 5, 7, 9], 40),
    "parts_of_3": ([10, 20, 30, 20, 20, 20, 1, 1, 1], 60),
    "over_the_budget": ([5, 100, 5, 0, 5], 50),
    "empty": ([], 10),
    "empty_lists": ([0, 0, 0], 1),
    "seeded": (np.random.default_rng(3).integers(0, 3 * T, 200).tolist(), 20000),
}


def test_plans_equal_the_model(planner):
    names = list(CASES)
    for name, got in zip(names, planner([CASES[n] for n in names])):
        lens, budget = CASES[name]
        assert got == ref.plan(_ptr(lens), budget), name


def test_plan_invariants(planner):
    names = list(CASES)
    for name, parts in zip(names, planner([CASES[n] for n in names])):
        lens, budget = CASES[name]
        ptr = _ptr(lens)
        assert [p["q0"] for p in parts] == sorted({p["q0"] for p in parts})
        assert (parts[0]["q0"] if parts else 0) == 0 and (parts[-1]["q1"] if parts else 0) == len(lens)
        for p, nxt in zip(parts, parts[1:] + [None]):
            ent = p["e1"] - p["e0"]
            assert ent <= budget or p["q1"] - p["q0"] == 1 or all(lens[q] == 0 for q in range(p["q0"] + 1, p["q1"]))
            if nxt is not None:
                assert nxt["q0"] == p["q1"] and ent + lens[nxt["q0"]] > budget
            qs = range(p["q0"], p["q1"])
            assert p["radix"] == [q for q in qs if lens[q] > T]
            assert p["tile_q"] == [q for q in qs if 0 < lens[q] <= T]
            for t in range(len(p["tile_n"])):
                a, b = p["tile_ptr"][t], p["tile_ptr"][t + 1]
                members = p["tile_q"][a:b]
                assert b > a and p["tile_n"][t] == sum(lens[q] for q in members) <= T
                assert p["tile_off"][a:b] == np.concatenate([[0], np.cumsum([lens[q] for q in members])[:-1]]).tolist()
                if t + 1 < len(p["tile_n"]):   # closed before a query that would overflow it
                    assert p["tile_n"][t] + lens[p["tile_q"][b]] > T
            assert p["e0"] == ptr[p["q0"]] and p["e1"] == ptr[p["q1"]]
    exact = planner([CASES["exact_fill"]])[0][0]
    assert exact["tile_n"] == [2048, 2048, 3, 2048]
    parts = {n: len(p) for n, p in zip(("parts_of_1", "parts_of_2", "parts_of_3"),
                                       planner([CASES[n] for n in ("parts_of_1", "parts_of_2", "parts_of_3")]))}
    assert parts == {"parts_of_1": 3, "parts_of_2": 3, "parts_of_3": 3}   # of 1, 2 and 3 queries each
    over = planner([CASES["over_the_budget"]])[0]
    assert [(p["q0"], p["q1"]) for p in over] == [(0, 1), (1, 2), (2, 5)]


def test_tile_matches_the_source():
    text = (CSRC / "rank_plan.h").read_text()
    assert int(re.search(r"constexpr int RL_TILE = (\d+);", text).group(1)) == T
    budget = re.search(r"#define PIO_RANK_LISTS_BUDGET \(1ll << (\d+)\)", (ROOT / "include" / "pio_als.h").read_text())
    assert 1 << int(budget.group(1)) == ref.BUDGET
