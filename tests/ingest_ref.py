"""numpy restatement of the ALS rating ingest (pio_als.cu: ingest_device, rank_rows, build_side): what one set_ratings
builds on each side of each rank, written from these rules.

  dedup  none       every event is kept; duplicates stay separate and keep event order inside a row
         sum        one entry per (user, item): the sequential fp32 reduce of its ratings in event order
                    (reduceByKey(_ + _): a run of one keeps its rating, -0.0 included), in (user, item) order
         keep_last  the rating of the largest ts wins; on a tie, and with no ts, the later event wins
  counts            deg = entries of the row after dedup; npos = entries > 0 (0, -0.0, NaN and sums that cancel are not);
                    nreg = npos when implicit, deg when explicit (0 on padding rows)
  renumbering       a stable sort by descending degree (ties by row id); position p goes to rank snake(p // W, p % W)
                    and internal id rank * R + p // W; inv = -1 on padding
  CSR               rows in internal order; inside a row, entries by the column's degree-rank position (rpos); idx = the
                    column's internal id
  heavy rows        of a rank's local rows (degree-descending), those with more than heavy_t ratings, each cut into parts
                    of part_len ratings; heavy_t and part_len are the side's plan (solve_plan.h: plan_side)
"""
import re
from pathlib import Path

import numpy as np

CSRC = Path(__file__).resolve().parent.parent / "incubator-predictionio_b200" / "csrc"
MODES = {"none": 0, "sum": 1, "keep_last": 2}


def ceil_log2(n: int) -> int:
    """Bits of an index below n, at least 1 (pio_als.cu ceil_log2)."""
    return max(1, (int(n) - 1).bit_length())


def plan_constants() -> dict:
    """`constexpr int NAME = value;` of solve_plan.h."""
    text = (CSRC / "solve_plan.h").read_text()
    return {k: int(v) for k, v in re.findall(r"constexpr\s+int\s+(\w+)\s*=\s*(\d+)\s*;", text)}


def pad_rank(rank: int) -> int:
    return 16 if rank <= 16 else 32 if rank <= 32 else 64 if rank <= 64 else 128


def side_plan(rank: int, n_rows: int, nnz: int, env=None) -> tuple:
    """(heavy_t, part_len) of a side (plan_side) under the switches in env (PIO_ALS_TC, PIO_ALS_TC_MIN_DEG, PIO_ALS_MMA,
    PIO_ALS_SEG_T, PIO_ALS_PART)."""
    env = env or {}
    c = plan_constants()
    kp = pad_rank(rank)
    seg_t, part = c["PAIR_SEG_T"], c["PAIR_PART"]
    if "PIO_ALS_SEG_T" in env and int(env["PIO_ALS_SEG_T"]) > 0:
        seg_t = int(env["PIO_ALS_SEG_T"])
    if "PIO_ALS_PART" in env and int(env["PIO_ALS_PART"]) >= 8:
        part = (int(env["PIO_ALS_PART"]) + 7) // 8 * 8
    mma_env = env.get("PIO_ALS_MMA")
    mma, pair = mma_env is None or mma_env[0] != "0", mma_env is None or mma_env[0] != "1"
    tc = (kp == 64 and env.get("PIO_ALS_TC", "")[:1] == "1" and n_rows > 0
          and nnz / n_rows >= float(env.get("PIO_ALS_TC_MIN_DEG", 0.0)))
    use_pair = not tc and kp == 64 and mma and pair
    heavy_t = 0 if kp == 128 else seg_t if use_pair else c["HEAVY_T_TC"] if (tc or (kp == 64 and mma)) else c["HEAVY_T"]
    return heavy_t, part if use_pair else c["PART"]


def dedup(user, item, rating, mode: str, ts=None):
    """(user int64, item int64, rating float32) after dedup: `none` in event order, the others in (user, item) order."""
    u = np.asarray(user, np.int64)
    i = np.asarray(item, np.int64)
    r = np.asarray(rating, np.float32)
    if mode == "none":
        return u, i, r
    n = u.shape[0]
    ev = np.arange(n, dtype=np.int64)
    if mode == "keep_last":
        t = np.zeros(n, np.int64) if ts is None else np.asarray(ts, np.int64)
        o = np.lexsort((ev, t, i, u))           # by (user, item), then ts, then event: the winner ends its run
        us, is_ = u[o], i[o]
        last = np.ones(n, bool)
        last[:-1] = (us[1:] != us[:-1]) | (is_[1:] != is_[:-1])
        return us[last], is_[last], r[o][last]
    if mode != "sum":
        raise ValueError(mode)
    o = np.lexsort((ev, i, u))                  # stable: event order inside each (user, item) run
    us, is_, rs = u[o], i[o], r[o]
    head = np.ones(n, bool)
    head[1:] = (us[1:] != us[:-1]) | (is_[1:] != is_[:-1])
    starts = np.flatnonzero(head)
    lens = np.diff(np.append(starts, n))
    acc = rs[starts].copy()
    # position p of every run at once, runs longest first so the runs still going are a prefix; runs longer than
    # SHORT finish one by one on np.cumsum, itself a sequential fp32 left fold
    SHORT = 64
    by_len = np.argsort(-lens, kind="stable")
    sl = lens[by_len]
    for p in range(1, min(int(sl[0]) if n else 0, SHORT)):
        live = by_len[:int(np.searchsorted(-sl, -p, side="left"))]   # runs with lens > p
        acc[live] = acc[live] + rs[starts[live] + p]
    for q in by_len[:int(np.searchsorted(-sl, -SHORT, side="left"))]:
        tail = np.concatenate([acc[q:q + 1], rs[starts[q] + SHORT:starts[q] + lens[q]]])
        acc[q] = np.cumsum(tail, dtype=np.float32)[-1]
    return us[starts], is_[starts], acc


def renumber(deg: np.ndarray, W: int):
    """(perm, inv, rpos, R, n_internal, bits) of one side's rows dealt to W ranks."""
    n = deg.shape[0]
    R = (n + W - 1) // W
    order = np.argsort(-deg.astype(np.int64), kind="stable")
    p = np.arange(n, dtype=np.int64)
    blk, pos = p // W, p % W
    rk = np.where(blk & 1, W - 1 - pos, pos)
    internal = rk * R + blk
    perm = np.empty(n, np.int64)
    perm[order] = internal
    rpos = np.empty(n, np.int64)
    rpos[order] = p
    inv = np.full(R * W, -1, np.int64)
    inv[internal] = order
    return perm, inv, rpos, R, R * W, ceil_log2(R * W)


def ingest(user, item, rating, n_users: int, n_items: int, mode: str = "none", ts=None, implicit: bool = False,
           W: int = 1, rank: int = 10, env=None):
    """Per side ("user", "item") a list of W dicts, one per rank, with the fields debug_side reports."""
    u, i, r = dedup(user, item, rating, mode, ts)
    nnz = u.shape[0]
    pos = r > 0
    sides = {}
    for name, rows, n in (("user", u, n_users), ("item", i, n_items)):
        deg = np.bincount(rows, minlength=n).astype(np.uint32)
        npos = np.bincount(rows[pos], minlength=n).astype(np.uint32)
        sides[name] = (rows, n, deg, npos, *renumber(deg, W))
    out = {}
    for name, other in (("user", "item"), ("item", "user")):
        rows, n, deg, npos, perm, inv, rpos, R, n_int, bits = sides[name]
        cols, _, _, _, cperm, _, crpos, _, _, _ = sides[other]
        heavy_t, part_len = side_plan(rank, n, nnz, env)
        o = np.lexsort((crpos[cols], perm[rows]))   # stable: duplicates (dedup none) keep event order
        ptr_full = np.zeros(n_int + 1, np.int64)
        ptr_full[1:] = np.cumsum(np.bincount(perm[rows], minlength=n_int))
        idx_all, val_all = cperm[cols[o]].astype(np.int32), r[o]
        ranks = []
        for rk in range(W):
            b, e = ptr_full[rk * R], ptr_full[(rk + 1) * R]
            ext = inv[rk * R:(rk + 1) * R]
            d = np.where(ext >= 0, deg[np.maximum(ext, 0)], 0)
            nreg = np.where(ext >= 0, (npos if implicit else deg)[np.maximum(ext, 0)], 0).astype(np.float32)
            ptr = ptr_full[rk * R:(rk + 1) * R + 1] - b
            n_heavy = int((d > heavy_t).sum())
            part_beg, part_end, rpp = [], [], [0]
            for row in range(n_heavy):
                starts = np.arange(ptr[row], ptr[row + 1], part_len, dtype=np.int64)
                part_beg.append(starts)
                part_end.append(np.minimum(starts + part_len, ptr[row + 1]))
                rpp.append(rpp[-1] + starts.shape[0])
            pb = np.concatenate(part_beg) if part_beg else np.zeros(0, np.int64)
            ranks.append(dict(
                n=n, R=R, n_internal=n_int, bits=bits, nnz_local=int(e - b), n_active=int((d > 0).sum()),
                n_heavy=n_heavy, n_parts=int(pb.shape[0]), nnz=nnz, heavy_t=heavy_t, part_len=part_len,
                deg=deg, npos=npos, perm=perm.astype(np.int32), inv=inv.astype(np.int32), rpos=rpos.astype(np.int32),
                ptr=ptr, idx=idx_all[b:e], val=val_all[b:e], nreg=nreg, part_beg=pb,
                part_end=np.concatenate(part_end) if part_end else np.zeros(0, np.int64),
                row_part_ptr=np.asarray(rpp, np.int32)))
        out[name] = ranks
    return out


SCALARS = ("n", "R", "n_internal", "bits", "nnz_local", "n_active", "n_heavy", "n_parts", "nnz", "heavy_t", "part_len")
ARRAYS = ("deg", "npos", "perm", "inv", "rpos", "ptr", "idx", "val", "nreg", "part_beg", "part_end", "row_part_ptr")


def differences(got: dict, want: dict) -> list:
    """Names of the fields where got != want: integers equal, floats equal as bits."""
    bad = [k for k in SCALARS if int(got[k]) != int(want[k])]
    for k in ARRAYS:
        g, w = np.asarray(got[k]), np.asarray(want[k])
        if g.dtype.kind == "f" or w.dtype.kind == "f":
            same = g.shape == w.shape and np.array_equal(g.astype(np.float32).view(np.uint32),
                                                         w.astype(np.float32).view(np.uint32))
        else:
            same = g.shape == w.shape and np.array_equal(g.astype(np.int64), w.astype(np.int64))
        if not same:
            bad.append(k)
    return bad
