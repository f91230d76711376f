"""CPU: the paths pio_rf_train_regressor takes (csrc/pio_als.cu rf_bin_and_grow<BinT, true>, rf_select_var,
csrc/forest.cuh) for each case of tests/test_gpu_forest_reg_bounds.py, from the case's parameters, the restatement's
thresholds and the constants read from the CUDA sources: bin code width, staged thresholds, 40-byte variance entries
per shared-memory pass, slots per histogram chunk (histogram, split order and centroids), block-scan tiles, the
in-block / multi-block category ranking and its tiles, label sums against 2^64, depth.  expected_record() turns that
and the restatement's per-level slot counts into the record native.rf_train_paths() must return (the GPU test asserts
it).  The tests here fail when the cases stop straddling a boundary, so that a change of a constant or a fixture cannot
quietly leave a path untested."""
import re
from pathlib import Path

import numpy as np
import pytest

from tests import forest_ref as fr
from tests import forest_reg_ref as rr
from tests import test_gpu_forest_reg_bounds as B
from tests.test_forest_paths import plan_groups

CSRC = Path(__file__).resolve().parents[1] / "incubator-predictionio_b200" / "csrc"
GRID_Y_MAX = 65535             # CUDA's limit on gridDim.y


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
        width_cut=ev(_const(cu, r"NB <= (\d+) \? rf_bin_and_grow<uint8_t, true>")),
        cat_smem_arity=ev(_const(cuh, r"constexpr int CAT_SMEM_ARITY = (\d+);")),
        rank_tile=ev(_const(cuh, r"constexpr int RANK_TILE = (\d+);")),
        sel_warps=ev(_const(cuh, r"constexpr int SEL_WARPS = (\d+);")),
        var_words=ev(_const(cuh, r"constexpr int VAR_WORDS = (\d+);")),
        max_depth=ev(_const(h, r"constexpr int RF_MAX_DEPTH = (\d+);")),
        label_bits=ev(_const(h, r"constexpr int RF_LABEL_BITS = (\d+);")),
        # bytes per bin and subset feature of a regressor chunk: variance entry, split order, centroids
        entry_bytes=ev(_const(cu, r"REG \? \(int64_t\)K \* NB \* rf::VAR_WORDS \* (\d+)")) * ev(
            _const(cuh, r"constexpr int VAR_WORDS = (\d+);")),
        order_bytes=ev(_const(cu, r"any_cat \? \(int64_t\)K \* NB \* (\d+)")),
        centroid_bytes=ev(_const(cu, r"wide_cat \? \(int64_t\)K \* NB \* (\d+)")),
    )


def static_paths(case, x, cat):
    """What a regressor case's shapes select before any tree grows."""
    c = constants()
    n, n_feat = x.shape
    cont = [f for f in range(n_feat) if f not in cat]
    n_thr = [len(t) for t in fr.find_thresholds(x[:, cont], case.bins, case.seed)] if cont else [0]
    nb = max([max(n_thr) + 1] + list(cat.values()))
    k = rr.subset_size(case.strategy, n_feat, case.T)
    any_cat = bool(cat)
    wide = any(a > c["cat_smem_arity"] for a in cat.values())
    entry = k * nb * c["entry_bytes"]
    chunk_slot = entry + (k * nb * c["order_bytes"] if any_cat else 0) + (k * nb * c["centroid_bytes"] if wide else 0)
    budget = case.budget if case.budget is not None else c["hist_budget"]
    return dict(nb=nb, k=k, n=n, n_thr=max(n_thr), bin_bytes=1 if nb <= c["width_cut"] else 2,
                staged=int(8 * sum(n_thr) <= c["stage_bytes"]), thresholds=sum(n_thr), slot_bytes=entry,
                chunk_slot=chunk_slot, pass_slots=c["smem"] // entry, chunk_max=max(1, budget // chunk_slot),
                wide=wide, scan_tiles=-(-nb // (c["sel_warps"] * 32)))


def expected_record(case, x, cat, level_slots, per_pass=None):
    """native.rf_train_paths() of a regressor case, from its static paths and the restatement's active slots per tree
    and level (info["level_slots"] of forest_reg_ref.train): the device counts the slots of a level over every tree of a
    group."""
    s = static_paths(case, x, cat)
    groups = plan_groups(case.T, s["n"], constants()["node_budget"], per_pass or 0)
    rec = dict(bin_bytes=s["bin_bytes"], staged=s["staged"], smem_launches=0, global_launches=0, max_chunks=0,
               max_passes=0, levels=0, groups=len(groups))
    for t0, t1 in groups:
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


ALL = {c.name: c for c in B.CASES + B.WIDE_CASES}
LIGHT = [c for c in B.CASES if not c.name.startswith("sums_")] + B.WIDE_CASES


@pytest.fixture(scope="module")
def paths():
    out = {}
    for case in LIGHT:
        y, x, cat, _ = case.make()
        out[case.name] = static_paths(case, x, cat)
    return out


def test_constants_are_the_ones_the_cases_were_sized_for():
    assert constants() == dict(smem=96 * 1024, hist_budget=1 << 29, node_budget=1 << 30, stage_bytes=48 * 1024,
                               width_cut=256, cat_smem_arity=2048, rank_tile=2048, sel_warps=8, var_words=5,
                               max_depth=30, label_bits=44, entry_bytes=40, order_bytes=4, centroid_bytes=8)


def test_continuous_bins_cross_the_block_scan_and_the_shared_histogram(paths):
    c = constants()
    tile = c["sel_warps"] * 32
    nb = {name: paths[name]["nb"] for name in ("nb255", "nb256_uint8", "nb257_uint16", "nb512_tie", "nb513",
                                               "nb2457_smem", "nb2458_global")}
    assert nb == dict(nb255=tile - 1, nb256_uint8=tile, nb257_uint16=tile + 1, nb512_tie=2 * tile, nb513=2 * tile + 1,
                      nb2457_smem=c["smem"] // c["entry_bytes"], nb2458_global=c["smem"] // c["entry_bytes"] + 1)
    for name in nb:
        p = paths[name]
        assert p["k"] == 1 and p["n_thr"] + 1 == p["nb"]               # every bin from thresholds: no categories
    assert paths["nb256_uint8"]["bin_bytes"] == 1 and paths["nb257_uint16"]["bin_bytes"] == 2
    assert paths["nb2457_smem"]["slot_bytes"] <= c["smem"] and paths["nb2457_smem"]["pass_slots"] == 1
    assert paths["nb2458_global"]["slot_bytes"] > c["smem"] and paths["nb2458_global"]["pass_slots"] == 0
    # levels deeper than one pass holds: 2^(depth - 1) possible slots against the slots of a pass
    for name in ("nb255", "nb256_uint8", "nb257_uint16", "nb512_tie", "nb513"):
        assert 2 ** (ALL[name].depth - 1) > 4 * paths[name]["pass_slots"] >= 4
    # the tie cases: 256 positions between the two equal gains (one thread of the scan), past the first tile
    for name in ("nb512_tie", "nb2457_smem", "nb2458_global"):
        m = paths[name]["nb"]
        a1 = (m - 256) // 2
        assert (m - 1 - (m - 256 - a1)) - (a1 - 1) == tile and m - 1 - (m - 256 - a1) >= tile


def test_label_sums_pass_2_64():
    """Root sums of the big cases: |S| of 65 bits ending in the sticky-bit tie (signed both ways, bagged), and a
    cancelling S beside a Q above 2^100."""
    c = constants()
    assert (1 << 20) * 2 ** c["label_bits"] <= 2 ** 64 < B.N_BIG * 2 ** c["label_bits"]   # 2^20 rows cannot pass
    signs = set()
    for name in ("sums_negative", "sums_positive", "sums_bagged", "sums_cancel"):
        case = ALL[name]
        y, x, cat, _ = case.make()
        assert x.shape[0] == B.N_BIG and cat == {0: 8}
        w = np.ones(len(y), np.int64) if case.T == 1 else fr.bag_weights(case.seed, 0, len(y))
        s, yq, S = B.label_sums(y, w)
        assert 2 ** 43 <= np.abs(yq).max() <= 2 ** 44
        if name == "sums_cancel":
            assert abs(S) < 2 ** 64
            q = yq.astype(np.float64)
            assert float(np.sum(q * q)) > 2.0 ** 100
        else:
            assert abs(S).bit_length() == 65 and abs(S) & B.STICKY_MASK == B.STICKY_LOW
            signs.add(S > 0)
        if case.T > 1:
            assert case.strategy == "all" and w.max() >= 8
    assert signs == {True, False}


def test_depth_30():
    c = constants()
    assert ALL["depth30"].depth == c["max_depth"]
    y, x, _, _ = ALL["depth30"].make()
    assert x.shape[0] > c["max_depth"] and np.unique(x).size == x.shape[0]


def test_quantisation_edges():
    want = {"label_min": 2.0 ** -rr.LABEL_EXP_MAX, "label_max": np.nextafter(2.0 ** rr.LABEL_EXP_MAX, 0),
            "label_round_to_2_44": np.nextafter(2.0, 0.0), "labels_zero": 0.0, "label_ties": 2.0 ** 43 + 0.5}
    for name, top in want.items():
        y, _, _, _ = ALL[name].make()
        assert np.abs(y).max() == top, name
    yq, s = rr.quantize(ALL["label_round_to_2_44"].make()[0])
    assert max(abs(v) for v in yq) == 2 ** constants()["label_bits"]
    y = ALL["label_ties"].make()[0]
    assert (np.ldexp(y, rr.quantize(y)[1]) % 1 == 0.5).sum() > 500


def test_category_ranking_switch_and_tiles(paths):
    c = constants()
    ar = {name: max(B.CASES[[k.name for k in B.CASES].index(name)].make()[2].values())
          for name in ("ties_arity4097", "ties_arity6000", "one_category_nodes")}
    assert ar["ties_arity4097"] == 2 * c["rank_tile"] + 1 and ar["ties_arity6000"] > 2 * c["rank_tile"] + 1
    assert ar["one_category_nodes"] > c["cat_smem_arity"]
    assert paths["one_category_nodes"]["wide"] and paths["ties_arity4097"]["wide"]
    # the metamorphic pair: arity 2048 ranks in the select block, 2049 through cat_rank_kernel
    assert c["cat_smem_arity"] == 2048


def test_wide_categories_chunk_and_group(paths):
    c = constants()
    for b, case in zip((1, 2), B.WIDE_CASES):
        p = paths[case.name]
        assert p["wide"] and p["chunk_slot"] == B.WIDE_SLOT and p["chunk_max"] == b
        assert p["pass_slots"] == 0                         # 5000-bin entries: the global histogram
        assert case.T >= 3 and len(plan_groups(case.T, p["n"], c["node_budget"], 2)) == 2


def test_many_subset_features(paths):
    assert paths["k300_copies"]["k"] == 300 > constants()["sel_warps"] * 32


def test_wide_category_segments_fit_a_grid_y():
    """cat_centroid_kernel and cat_rank_kernel put one (slot, wide feature) segment per gridDim.y.  A chunk holds at
    most RF_HIST_BUDGET / (K NB 52) slots of K subset features, so its segments are at most RF_HIST_BUDGET / (NB 52)
    with NB > CAT_SMEM_ARITY; a chunk of one slot (the budget below one slot) has at most K segments, one per feature,
    and such a slot alone needs K NB 52 bytes, more than any device holds for K >= 65536."""
    c = constants()
    per_bin = c["entry_bytes"] + c["order_bytes"] + c["centroid_bytes"]
    assert per_bin == 52
    assert c["hist_budget"] // ((c["cat_smem_arity"] + 1) * per_bin) <= GRID_Y_MAX


def test_expected_record_counts_slots_over_a_group():
    case = B.Case("t", None, 3, "all", 3, 32, 2 * 3 * 32 * 40, 0)          # two slots a chunk, no categories
    x = np.tile(np.arange(32.0)[:, None], (1, 3))
    rec = expected_record(case, x, {}, [[1, 2, 3], [1, 2], [1]])
    assert rec["levels"] == 3 and rec["groups"] == 1
    assert rec["max_chunks"] == 2 and rec["smem_launches"] == 6 and rec["max_passes"] == 1
    rec = expected_record(case, x, {}, [[1, 2, 3], [1, 2], [1]], per_pass=1)
    # one tree a group: levels of 1, 2, 3 | 1, 2 | 1 slots in chunks of two
    assert rec["groups"] == 3 and rec["max_chunks"] == 2 and rec["smem_launches"] == 7
