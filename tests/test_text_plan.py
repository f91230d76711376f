"""CPU: the text featurizer's planner (csrc/text_plan.h) against the plan model in tests/textclassification_ref.py.

A small driver is compiled against text_plan.h alone, with g++, and asked for the parts of budgets that give parts of
1, 2 and 3 documents, and of a document larger than the budget."""
import re
import shutil
import subprocess
from pathlib import Path

import numpy as np
import pytest

from tests import textclassification_ref as ref

ROOT = Path(__file__).resolve().parent.parent
CSRC = ROOT / "incubator-predictionio_b200" / "csrc"

DRIVER = r"""
#include <cstdio>
#include <iostream>
#include "text_plan.h"
using namespace pio;
int main() {
  int n;
  long long budget;
  while (std::cin >> budget >> n) {
    std::vector<int64_t> off(n + 1);
    for (auto& x : off) std::cin >> x;
    const std::vector<TextPart> parts = plan_text(off.data(), n, budget);
    printf("%zu", parts.size());
    for (const TextPart& p : parts) printf(" %d %d %lld %lld", p.d0, p.d1, p.b0, p.b1);
    printf("\n");
  }
}
"""

CASES = {
    "parts_of_1": ([10, 20, 25], 25),
    "parts_of_2": ([10, 20, 30, 5, 7, 9], 40),
    "parts_of_3": ([10, 20, 30, 20, 20, 20, 2, 2, 2], 60),
    "over_the_budget": ([5, 100, 5, 2, 5], 50),
    "empty": ([], 10),
    "seeded": (np.random.default_rng(3).integers(2, 3000, 300).tolist(), 20000),
}


def _off(lens):
    return np.concatenate([[0], np.cumsum(lens, dtype=np.int64)]).tolist()


@pytest.fixture(scope="module")
def planner(tmp_path_factory):
    if shutil.which("g++") is None:
        pytest.skip("needs g++")
    d = tmp_path_factory.mktemp("text_plan")
    (d / "driver.cpp").write_text(DRIVER)
    exe = d / "driver"
    subprocess.run(["g++", "-std=c++17", "-Wall", "-Wextra", "-Werror", "-O1", "-I", str(CSRC), "-o", str(exe),
                    str(d / "driver.cpp")], check=True)

    def run(cases):
        text = "".join(f"{b} {len(lens)} " + " ".join(map(str, _off(lens))) + "\n" for lens, b in cases)
        out = subprocess.run([str(exe)], input=text, capture_output=True, text=True, check=True).stdout.splitlines()
        plans = []
        for line in out:
            v = [int(x) for x in line.split()]
            plans.append([tuple(v[1 + 4 * k:5 + 4 * k]) for k in range(v[0])])
        return plans
    return run


def test_plans_equal_the_model(planner):
    names = list(CASES)
    for name, got in zip(names, planner([CASES[n] for n in names])):
        lens, budget = CASES[name]
        off = _off(lens)
        assert [(a, b) for a, b, _, _ in got] == ref.plan(off, budget), name
        assert all(b0 == off[a] and b1 == off[b] for a, b, b0, b1 in got), name


def test_part_counts(planner):
    names = ("parts_of_1", "parts_of_2", "parts_of_3", "over_the_budget")
    got = dict(zip(names, planner([CASES[n] for n in names])))
    assert {n: len(got[n]) for n in names[:3]} == {"parts_of_1": 3, "parts_of_2": 3, "parts_of_3": 3}
    assert [(a, b) for a, b, _, _ in got["over_the_budget"]] == [(0, 1), (1, 2), (2, 5)]


def test_budget_matches_the_header():
    budget = re.search(r"#define PIO_TEXT_BUDGET \(1ll << (\d+)\)", (ROOT / "include" / "pio_als.h").read_text())
    assert 1 << int(budget.group(1)) == ref.BUDGET
