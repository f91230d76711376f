"""CPU: the paths pio_rf_train takes (csrc/pio_als.cu rf_bin_and_grow, csrc/forest.cuh) for each case of
tests/test_gpu_forest_bounds.py, from the case's parameters, forest_ref.find_thresholds and the constants read from the
CUDA sources: bin code width, staged thresholds, slots per shared-memory pass, slots per histogram chunk, subset
features against select warps.  expected_record() turns that and the restatement's per-level slot counts into the
record native.rf_train_paths() must return (the GPU test asserts it).  The tests here fail when the cases stop
straddling a boundary, so that a change of a constant cannot quietly leave a path untested."""
import math
import re
from pathlib import Path

import numpy as np
import pytest

from tests import forest_ref as fr
from tests import test_gpu_forest_bounds as B

CSRC = Path(__file__).resolve().parents[1] / "incubator-predictionio_b200" / "csrc"


def _const(src, pattern):
    m = re.search(pattern, src)
    assert m, pattern
    return m.group(1)


def constants():
    cu = (CSRC / "pio_als.cu").read_text()
    cuh = (CSRC / "forest.cuh").read_text()
    h = (CSRC / "forest_splits.h").read_text()
    ev = lambda s: int(eval(s.replace("ll", ""), {}))          # noqa: E731  (1ll << 30, 96 * 1024)
    return dict(
        smem=ev(_const(cu, r"constexpr int RF_SMEM = ([^;]+);")),
        hist_budget=ev(_const(cu, r"constexpr int64_t RF_HIST_BUDGET = ([^;]+);")),
        node_budget=ev(_const(cu, r"constexpr int64_t RF_NODE_BUDGET = ([^;]+);")),
        stage_bytes=ev(_const(cu, r"const int staged = thr_bytes <= ([^?]+) \?")),
        width_cut=ev(_const(cu, r"NB <= (\d+) \? rf_bin_and_grow<uint8_t>")),
        sel_warps=ev(_const(cuh, r"constexpr int SEL_WARPS = (\d+);")),
        max_classes=ev(_const(h, r"constexpr int RF_MAX_CLASSES = (\d+);")),
        max_bins=ev(_const(h, r"constexpr int RF_MAX_BINS = (\d+);")),
        max_depth=ev(_const(h, r"constexpr int RF_MAX_DEPTH = (\d+);")),
    )


def plan_groups(num_trees, n, node_budget, per_pass=0):
    """rf_plan_groups of forest_splits.h."""
    g = per_pass if per_pass > 0 else node_budget // max(1, 4 * n)
    g = max(1, min(g, num_trees))
    return [(t, min(num_trees, t + g)) for t in range(0, num_trees, g)]


def static_paths(case, x):
    """What a case's shapes select before any tree grows."""
    c = constants()
    n, n_feat = x.shape
    thr = fr.find_thresholds(x, case.bins, case.seed)
    n_thr = [len(t) for t in thr]
    nb = max(n_thr) + 1
    k = fr.subset_size(case.strategy, n_feat, case.T)
    slot = k * nb * case.C
    budget = case.budget if case.budget is not None else c["hist_budget"]
    return dict(nb=nb, k=k, n=n, bin_bytes=1 if nb <= c["width_cut"] else 2,
                staged=int(8 * sum(n_thr) <= c["stage_bytes"]), thresholds=sum(n_thr), slot_entries=slot,
                pass_slots=c["smem"] // (4 * slot), chunk_max=max(1, budget // (8 * slot)),
                groups=plan_groups(case.T, n, c["node_budget"]), sample=fr.sample_fraction(n, case.bins) < 1.0)


def expected_record(case, x, level_slots):
    """native.rf_train_paths() of a case, from its static paths and the restatement's active slots per tree and level
    (info["level_slots"] of forest_ref.train): the device counts the slots of a level over every tree of a group."""
    s = static_paths(case, x)
    rec = dict(bin_bytes=s["bin_bytes"], staged=s["staged"], smem_launches=0, global_launches=0, max_chunks=0,
               max_passes=0, levels=0, groups=len(s["groups"]))
    for t0, t1 in s["groups"]:
        depth = max(len(level_slots[t]) for t in range(t0, t1))
        rec["levels"] = max(rec["levels"], depth)
        for level in range(depth):
            S = sum(level_slots[t][level] for t in range(t0, t1) if level < len(level_slots[t]))
            cap = min(S, s["chunk_max"])
            rec["max_chunks"] = max(rec["max_chunks"], -(-S // cap))
            for c0 in range(0, S, cap):
                size = min(S, c0 + cap) - c0
                if s["pass_slots"] >= 1:
                    passes = -(-size // s["pass_slots"])
                    rec["smem_launches"] += passes
                    rec["max_passes"] = max(rec["max_passes"], passes)
                else:
                    rec["global_launches"] += 1
    return rec


@pytest.fixture(scope="module")
def paths():
    out = {}
    for case in B.CASES + B.CHUNK_CASES:
        y, x, _ = case.make()
        out[case.name] = static_paths(case, x)
    return out


def test_constants_are_the_ones_the_cases_were_sized_for():
    c = constants()
    assert c == dict(smem=96 * 1024, hist_budget=1 << 29, node_budget=1 << 30, stage_bytes=48 * 1024, width_cut=256,
                     sel_warps=8, max_classes=64, max_bins=65536, max_depth=30)


def test_bin_width_cut(paths):
    c = constants()
    assert paths["nb256_uint8"]["nb"] == c["width_cut"] and paths["nb256_uint8"]["bin_bytes"] == 1
    assert paths["nb257_uint16"]["nb"] == c["width_cut"] + 1 and paths["nb257_uint16"]["bin_bytes"] == 2
    assert paths["nb65536"]["nb"] == c["max_bins"] and paths["nb65536"]["bin_bytes"] == 2


def test_threshold_staging_cut(paths):
    c = constants()
    assert paths["thr6144_staged"]["thresholds"] * 8 == c["stage_bytes"] and paths["thr6144_staged"]["staged"] == 1
    assert paths["thr6145_global"]["thresholds"] * 8 == c["stage_bytes"] + 8 and paths["thr6145_global"]["staged"] == 0


def test_shared_and_global_histograms(paths):
    c = constants()
    one, glob = paths["smem_one_slot_c32"], paths["global_c33"]
    assert one["slot_entries"] * 4 == c["smem"] and one["pass_slots"] == 1
    assert glob["slot_entries"] * 4 > c["smem"] and glob["pass_slots"] == 0
    assert paths["passes_shallow"]["pass_slots"] == paths["passes_deep"]["pass_slots"] > 1


def test_chunk_budgets(paths):
    want = {"None": None, "1": 1, "2": 2, "3": 3, "0.3": 1}
    for kind in ("smem", "global"):
        for b, chunk in want.items():
            p = paths[f"chunk_{kind}_{b}"]
            assert (p["pass_slots"] >= 1) == (kind == "smem")
            if chunk is None:
                assert p["chunk_max"] > 100
            else:
                assert p["chunk_max"] == chunk, (kind, b)
    d = paths["chunked_default"]
    assert 1 < d["chunk_max"] < 10 and d["pass_slots"] == 0     # the case's level 1 holds 10 slots


def test_subset_features_against_select_warps(paths):
    w = constants()["sel_warps"]
    ks = sorted(paths[n]["k"] for n in ("k8", "k9", "k16", "k17", "k10_sqrt100"))
    assert ks == [w, w + 1, w + 2, 2 * w, 2 * w + 1]
    assert paths["k10_sqrt100"]["k"] == math.ceil(math.sqrt(100))


def test_class_counts_against_warp_width():
    c = constants()
    by = {case.name: case.C for case in B.CASES}
    assert {by["c2"], by["smem_one_slot_c32"], by["global_c33"], by["c64_all"], by["c64_five"]} == \
        {2, 32, 33, c["max_classes"]}


def test_depth_and_degenerate_cases(paths):
    c = constants()
    by = {case.name: case for case in B.CASES}
    assert by["depth30_comb"].depth == c["max_depth"]
    assert paths["constant"]["nb"] == 1
    assert paths["n1"]["n"] == 1 and paths["n2"]["n"] == 2 and by["n2"].bins > 2


def test_split_sample_and_groups(paths):
    a, b = paths["sample_all_90000"], paths["sample_some_90001"]
    assert a["n"] == max(300 ** 2, 10000) and not a["sample"]
    assert b["n"] == a["n"] + 1 and b["sample"]
    assert len(paths["two_groups"]["groups"]) >= 2


def test_expected_record_counts_slots_over_a_group():
    case = B.Case("t", None, 4, 3, "all", 3, 32, 3 * 32 * 4 * 8 * 2, 0)      # two slots a chunk
    x = np.tile(np.arange(32.0)[:, None], (1, 3))
    rec = expected_record(case, x, [[1, 2, 3], [1, 2], [1]])
    assert rec["levels"] == 3 and rec["groups"] == 1
    # levels of 3, 4 and 3 slots in chunks of two: 2, 2 and 2 chunks, one pass each
    assert rec["max_chunks"] == 2 and rec["smem_launches"] == 6 and rec["max_passes"] == 1
