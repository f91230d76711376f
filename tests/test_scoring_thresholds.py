"""CPU: the scoring dispatch constants of the CUDA sources still match tests/test_gpu_scoring.py, and its ladders still
straddle every threshold.  Moving a threshold in topk.cuh or pio_als.cu without moving the GPU test's cases fails here."""
import re
from pathlib import Path

import test_gpu_scoring as G

CSRC = Path(__file__).resolve().parent.parent / "incubator-predictionio_b200" / "csrc"


def _constants():
    src = (CSRC / "topk.cuh").read_text()
    env = {}
    for name, expr in re.findall(r"^constexpr int (\w+) = ([^;]+);", src, re.M):
        env[name] = int(eval(expr, {}, dict(env)))   # integer literals and earlier constants only
    return env


def _host():
    return " ".join((CSRC / "pio_als.cu").read_text().split())


def test_constants_match_sources():
    c = _constants()
    for name in ("TK_MAXK", "DB_MAXK", "SB_QB", "S1_MAXNV", "SM_NV", "SM_QG", "SM_QIDS", "DB_QW", "CB_QPW", "DB_WPR",
                 "SB_THREADS", "SC_G"):
        assert getattr(G, name) == c[name], (name, getattr(G, name), c[name])
    host = _host()
    # the S5 choice between the shared-memory and the fallback kernel, as tests/test_gpu_scoring.py s5_smem restates it
    assert ("sc_smem = sizeof(double) * ((size_t)KP * nqp + nqp) + sizeof(float) * (size_t)SB_THREADS * (KP + 4) + "
            "(sizeof(double) + sizeof(int)) * (size_t)SC_WARPS * pass_max + sizeof(int) * (size_t)nq + 16;") in host
    assert "constexpr int SC_WARPS = SB_THREADS / 32;" in host
    assert "const int nqp = (nqv + SC_G - 1) / SC_G * SC_G;" in host
    limit = re.search(r"const bool batched = sc_smem <= (\d+) \* 1024;", host)
    assert limit and int(limit.group(1)) * 1024 == G.S5_SMEM_LIMIT
    # both batch paths launch at most GROUP_CHUNK query groups per grid (grid.y)
    chunks = re.findall(r"for \(int g0 = 0; g0 < ngroups; g0 \+= (\d+)\)", host)
    assert len(chunks) == 3 and {int(x) for x in chunks} == {G.GROUP_CHUNK}, chunks
    # the dispatch conditions the path predictions of the GPU test restate
    assert "h->serve_fused && h->KP <= 64 && topk <= TK_MAXK && nq >= 1 && nq <= S1_MAXNV" in host
    assert "if (n <= SB_QB && topk <= TK_MAXK)" in host
    assert "q_ptr[1] - q_ptr[0] <= SM_NV && topk <= TK_MAXK" in host
    assert host.count("KP <= 64 && topk <= DB_MAXK") == 2


def test_ladders_straddle_every_threshold():
    c = _constants()
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
    # one similar query: S2 takes up to SM_NV query ids, valid or not (the host tests q_ptr[1] - q_ptr[0]); one id more
    # goes to S5.  A batch: S4 takes 8-query groups of up to SM_NV valid vectors; one vector more sends it to S5.
    assert set(G.S2_QUERY_IDS) == {c["SM_NV"], c["SM_NV"] + 1}
    assert set(G.GROUP_VECTORS) == {c["SM_NV"], c["SM_NV"] + 1}
    assert G.SM_QG == c["SM_QG"] and max(G.GROUP_VECTORS) // 4 > c["DB_QW"]   # the 4-query groups stay off the blocked kernel
    # the S5 shared-memory / fallback boundary at KP 64, topk 20, recomputed from the sc_smem formula (the GPU test's
    # S5 queries carry three invalid ids besides nv valid ones)
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
