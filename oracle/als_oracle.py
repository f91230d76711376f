"""CPU ORACLE -- test infrastructure, not product code.

ctypes front-end for ``oracle/als_oracle.c`` (the C/OpenMP restatement of the
Spark-MLlib arithmetic PredictionIO's templates call; see that file's header
for the reference call sites) plus an independent dense NumPy/SciPy
restatement used to cross-check the C code on tiny problems.

PARITY UNPINNED: the reference holds no golden vectors for ALS and MLlib
cannot run here; see als_oracle.c.

Only ``tests/``, ``__graft_entry__.smoke()`` and ``bench.py``'s
``cpu_baseline`` / ``--impl reference`` leg may import this module.
"""
from __future__ import annotations

import ctypes as C
import os
import subprocess
from pathlib import Path

import numpy as np

_HERE = Path(__file__).resolve().parent
_SRC = _HERE / "als_oracle.c"
_SO = _HERE / "_build" / "libals_oracle.so"
_lib = None


def build(force: bool = False) -> Path:
    """Compile als_oracle.c -> oracle/_build/libals_oracle.so (gcc -O3 -fopenmp)."""
    if _SO.exists() and not force and _SO.stat().st_mtime >= _SRC.stat().st_mtime:
        return _SO
    _SO.parent.mkdir(parents=True, exist_ok=True)
    cmd = ["gcc", "-O3", "-march=x86-64-v2", "-fopenmp", "-fPIC", "-shared", "-fvisibility=hidden", "-ffp-contract=off",
           "-o", str(_SO), str(_SRC), "-lm"]
    subprocess.run(cmd, check=True)
    return _SO


def _p(a, t):
    if a is None:
        return None
    return a.ctypes.data_as(C.POINTER(t))


def lib():
    global _lib
    if _lib is None:
        if not _SO.exists():
            build()
        _lib = C.CDLL(str(_SO))
        _lib.oracle_num_threads.restype = C.c_int
    return _lib


def num_threads() -> int:
    return int(lib().oracle_num_threads())


def set_num_threads(n: int) -> None:
    lib().oracle_set_num_threads(C.c_int(n))


def csr_build(n_rows, row, col, val):
    row = np.ascontiguousarray(row, np.int32)
    col = np.ascontiguousarray(col, np.int32)
    val = np.ascontiguousarray(val, np.float32)
    nnz = row.shape[0]
    ptr = np.zeros(n_rows + 1, np.int64)
    oc = np.empty(max(nnz, 1), np.int32)
    ov = np.empty(max(nnz, 1), np.float32)
    rc = lib().oracle_csr_build(C.c_int32(n_rows), C.c_int64(nnz), _p(row, C.c_int32), _p(col, C.c_int32),
                                _p(val, C.c_float), _p(ptr, C.c_int64), _p(oc, C.c_int32), _p(ov, C.c_float))
    if rc != 0:
        raise ValueError(f"oracle_csr_build failed rc={rc}")
    return ptr, oc[:nnz], ov[:nnz]


def gram(f, has=None):
    f = np.ascontiguousarray(f, np.float32)
    n, k = f.shape
    out = np.zeros(k * (k + 1) // 2, np.float64)
    hp = None if has is None else _p(np.ascontiguousarray(has, np.uint8), C.c_uint8)
    lib().oracle_gram(C.c_int32(n), C.c_int(k), _p(f, C.c_float), hp, _p(out, C.c_double))
    return out


def unpack_upper(ap, k):
    a = np.zeros((k, k), np.float64)
    for j in range(k):
        for i in range(j + 1):
            a[i, j] = a[j, i] = ap[j * (j + 1) // 2 + i]
    return a


def half_step(ptr, idx, val, src, dst, lam, implicit, alpha, yty=None, row_begin=0, row_end=None, row_stride=1):
    """dst rows (in place) from src factors. Returns #failed rows."""
    n_dst, k = dst.shape
    assert src.dtype == np.float32 and dst.dtype == np.float32 and dst.flags.c_contiguous
    if row_end is None:
        row_end = n_dst
    yp = None if yty is None else _p(np.ascontiguousarray(yty, np.float64), C.c_double)
    return int(lib().oracle_als_half_step(
        C.c_int32(n_dst), C.c_int(k), _p(ptr, C.c_int64), _p(idx, C.c_int32), _p(val, C.c_float),
        _p(src, C.c_float), _p(dst, C.c_float), C.c_double(lam), C.c_int(int(implicit)), C.c_double(alpha),
        yp, C.c_int32(row_begin), C.c_int32(row_end), C.c_int32(row_stride)))


def half_step_rows(ptr, idx, val, src, rows, lam, implicit, alpha, yty=None):
    """Solutions of the listed destination rows (len(rows) x k) from src factors; rows without ratings stay zero."""
    k = src.shape[1]
    rows = np.ascontiguousarray(rows, np.int32)
    out = np.zeros((rows.shape[0], k), np.float32)
    assert src.dtype == np.float32 and src.flags.c_contiguous
    yp = None if yty is None else _p(np.ascontiguousarray(yty, np.float64), C.c_double)
    fails = int(lib().oracle_als_half_step_rows(
        C.c_int(k), _p(ptr, C.c_int64), _p(idx, C.c_int32), _p(val, C.c_float), _p(src, C.c_float), C.c_double(lam),
        C.c_int(int(implicit)), C.c_double(alpha), yp, _p(rows, C.c_int32), C.c_int32(rows.shape[0]),
        _p(out, C.c_float)))
    return out, fails


def csr_dedup_sum(ptr, col, val):
    """reduceByKey(_ + _) inside every CSR row (same result as dedup_coo(mode="sum")); returns new (ptr, col, val)."""
    ptr = np.array(ptr, np.int64, copy=True)
    col = np.array(col, np.int32, copy=True)
    val = np.array(val, np.float32, copy=True)
    lib().oracle_csr_dedup_sum.restype = C.c_int64
    n = int(lib().oracle_csr_dedup_sum(C.c_int32(ptr.shape[0] - 1), _p(ptr, C.c_int64), _p(col, C.c_int32),
                                       _p(val, C.c_float)))
    if n < 0:
        raise MemoryError("oracle_csr_dedup_sum")
    return ptr, col[:n], val[:n]


def csr_rows(ptr):
    """Row index of every CSR entry (int32)."""
    n = ptr.shape[0] - 1
    return np.repeat(np.arange(n, dtype=np.int32), np.diff(ptr))


def als_train(n_users, n_items, user, item, rating, rank, iters, lam, implicit, alpha, user_init, item_init):
    """Full MLlib-style training. Returns (user_f, item_f, user_has, item_has)."""
    user = np.ascontiguousarray(user, np.int32)
    item = np.ascontiguousarray(item, np.int32)
    rating = np.ascontiguousarray(rating, np.float32)
    uf = np.array(user_init, np.float32, order="C", copy=True)
    itf = np.array(item_init, np.float32, order="C", copy=True)
    assert uf.shape == (n_users, rank) and itf.shape == (n_items, rank)
    uh = np.zeros(max(n_users, 1), np.uint8)
    ih = np.zeros(max(n_items, 1), np.uint8)
    rc = lib().oracle_als_train(
        C.c_int32(n_users), C.c_int32(n_items), C.c_int64(user.shape[0]), _p(user, C.c_int32),
        _p(item, C.c_int32), _p(rating, C.c_float), C.c_int(rank), C.c_int(iters), C.c_double(lam),
        C.c_int(int(implicit)), C.c_double(alpha), _p(uf, C.c_float), _p(itf, C.c_float),
        _p(uh, C.c_uint8), _p(ih, C.c_uint8))
    if rc != 0:
        raise RuntimeError(f"oracle_als_train rc={rc}")
    return uf, itf, uh[:n_users], ih[:n_items]


def recommend(user_f, user_has, item_f, item_has, users, topk, mask=None, weight=None):
    user_f = np.ascontiguousarray(user_f, np.float32)
    item_f = np.ascontiguousarray(item_f, np.float32)
    users = np.ascontiguousarray(users, np.int32)
    n_items, k = item_f.shape
    nq = users.shape[0]
    oi = np.full((nq, topk), -1, np.int32)
    os_ = np.zeros((nq, topk), np.float32)
    oc = np.zeros(nq, np.int32)
    uh = None if user_has is None else np.ascontiguousarray(user_has, np.uint8)
    ih = None if item_has is None else np.ascontiguousarray(item_has, np.uint8)
    mk = None if mask is None else np.ascontiguousarray(mask, np.uint8)
    wt = None if weight is None else np.ascontiguousarray(weight, np.float64)
    lib().oracle_recommend(C.c_int32(n_items), C.c_int(k), _p(user_f, C.c_float), _p(uh, C.c_uint8),
                           _p(item_f, C.c_float), _p(ih, C.c_uint8), _p(users, C.c_int32), C.c_int(nq),
                           C.c_int(topk), _p(mk, C.c_uint8), _p(wt, C.c_double), _p(oi, C.c_int32), _p(os_, C.c_float),
                           _p(oc, C.c_int32))
    return oi, os_, oc


def similar(item_f, item_has, query, topk, mask=None, weight=None, keep_query=False):
    item_f = np.ascontiguousarray(item_f, np.float32)
    query = np.ascontiguousarray(query, np.int32)
    n_items, k = item_f.shape
    oi = np.full(topk, -1, np.int32)
    os_ = np.zeros(topk, np.float32)
    oc = C.c_int32(0)
    ih = None if item_has is None else np.ascontiguousarray(item_has, np.uint8)
    mk = None if mask is None else np.ascontiguousarray(mask, np.uint8)
    wt = None if weight is None else np.ascontiguousarray(weight, np.float64)
    lib().oracle_similar(C.c_int32(n_items), C.c_int(k), _p(item_f, C.c_float), _p(ih, C.c_uint8),
                         _p(query, C.c_int32), C.c_int(query.shape[0]), C.c_int(topk), _p(mk, C.c_uint8),
                         _p(wt, C.c_double), C.c_int(int(keep_query)), _p(oi, C.c_int32), _p(os_, C.c_float), C.byref(oc))
    return oi, os_, int(oc.value)


def nb_train(label, x, n_class, lam):
    label = np.ascontiguousarray(label, np.int32)
    x = np.ascontiguousarray(x, np.float32)
    n, f = x.shape
    pi = np.zeros(n_class, np.float64)
    theta = np.zeros((n_class, f), np.float64)
    lib().oracle_nb_train(C.c_int64(n), C.c_int(f), C.c_int(n_class), _p(label, C.c_int32), _p(x, C.c_float),
                          C.c_double(lam), _p(pi, C.c_double), _p(theta, C.c_double))
    return pi, theta


def nb_predict(x, pi, theta):
    x = np.ascontiguousarray(x, np.float32)
    n, f = x.shape
    out = np.zeros(n, np.int32)
    pi = np.ascontiguousarray(pi, np.float64)
    theta = np.ascontiguousarray(theta, np.float64)
    lib().oracle_nb_predict(C.c_int64(n), C.c_int(f), C.c_int(pi.shape[0]), _p(x, C.c_float), _p(pi, C.c_double),
                            _p(theta, C.c_double), _p(out, C.c_int32))
    return out


# ----------------------------------------------------------------------------
# Template-side data preparation (host logic the reference does in Spark):
#   none      -> recommendation template: duplicates kept (ALSAlgorithm.scala:62-65)
#   sum       -> similarproduct: reduceByKey(_ + _) (multi-events ALSAlgorithm.scala:106)
#   keep_last -> ecommerce: latest timestamp wins (ECommAlgorithm.scala:189-197)
# Output order: sorted by (user, item); ties keep input order.
# ----------------------------------------------------------------------------
def dedup_coo(user, item, rating, mode="none", ts=None):
    user = np.asarray(user, np.int64)
    item = np.asarray(item, np.int64)
    rating = np.asarray(rating, np.float32)
    key = (user << 32) | item
    order = np.argsort(key, kind="stable")
    if mode == "none":
        return user[order].astype(np.int32), item[order].astype(np.int32), rating[order]
    ks = key[order]
    head = np.ones(ks.shape[0], bool)
    head[1:] = ks[1:] != ks[:-1]
    starts = np.flatnonzero(head)
    if mode == "sum":
        # sequential fp32 sums in input order (reduceByKey(_ + _): a run of one keeps its rating, -0.0 included)
        seg = np.cumsum(head) - 1
        out = np.zeros(starts.shape[0], np.float32)
        rs = rating[order]
        for s in range(starts.shape[0]):
            e = starts[s + 1] if s + 1 < starts.shape[0] else ks.shape[0]
            acc = rs[starts[s]]
            for v in rs[starts[s] + 1:e]:
                acc = np.float32(acc + v)
            out[s] = acc
        del seg
    elif mode == "keep_last":
        if ts is None:
            ts = np.arange(user.shape[0], dtype=np.int64)
        ts = np.asarray(ts, np.int64)[order]
        rs = rating[order]
        out = np.zeros(starts.shape[0], np.float32)
        for s in range(starts.shape[0]):
            e = starts[s + 1] if s + 1 < starts.shape[0] else ks.shape[0]
            seg_ts = ts[starts[s]:e]
            # latest timestamp wins; among equal timestamps the later input wins
            j = len(seg_ts) - 1 - int(np.argmax(seg_ts[::-1]))
            out[s] = rs[starts[s] + j]
    else:
        raise ValueError(mode)
    return (ks[starts] >> 32).astype(np.int32), (ks[starts] & 0xFFFFFFFF).astype(np.int32), out


# ----------------------------------------------------------------------------
# Independent dense restatement (NumPy/SciPy), for cross-checking the C oracle
# on tiny problems only (O(rows * k^2) Python loops).
# ----------------------------------------------------------------------------
def numpy_half_step(n_dst, rows, cols, vals, src, dst, lam, implicit, alpha, src_has=None):
    from scipy.linalg import cho_factor, cho_solve
    k = src.shape[1]
    s64 = src.astype(np.float64)
    if implicit:
        m = s64 if src_has is None else s64[np.asarray(src_has, bool)]
        yty = m.T @ m
    out = dst.copy()
    for r in range(n_dst):
        sel = np.flatnonzero(rows == r)
        if sel.size == 0:
            continue
        Y = s64[cols[sel]]
        rr = vals[sel].astype(np.float64)
        if implicit:
            c1 = alpha * np.abs(rr)
            A = yty + (Y * c1[:, None]).T @ Y
            pos = rr > 0
            b = ((1.0 + c1[pos])[:, None] * Y[pos]).sum(0) if pos.any() else np.zeros(k)
            n = int(pos.sum())
        else:
            A = Y.T @ Y
            b = (rr[:, None] * Y).sum(0)
            n = sel.size
        A = A + lam * n * np.eye(k)
        x = cho_solve(cho_factor(A), b)
        out[r] = x.astype(np.float32)
    return out


def numpy_als_train(n_users, n_items, user, item, rating, rank, iters, lam, implicit, alpha, user_init, item_init):
    user = np.asarray(user)
    item = np.asarray(item)
    rating = np.asarray(rating, np.float32)
    uh = np.bincount(user, minlength=n_users) > 0
    ih = np.bincount(item, minlength=n_items) > 0
    uf = np.array(user_init, np.float32, copy=True)
    itf = np.array(item_init, np.float32, copy=True)
    uf[~uh] = 0
    itf[~ih] = 0
    for _ in range(iters):
        itf = numpy_half_step(n_items, item, user, rating, uf, itf, lam, implicit, alpha, uh)
        uf = numpy_half_step(n_users, user, item, rating, itf, uf, lam, implicit, alpha, ih)
    return uf, itf, uh.astype(np.uint8), ih.astype(np.uint8)


def als_objective(user, item, rating, uf, itf, lam, implicit, alpha):
    """ALS-WR (explicit) / Hu-Koren-Volinsky with n-weighted ridge (implicit) objective, fp64."""
    U = uf.astype(np.float64)
    V = itf.astype(np.float64)
    r = np.asarray(rating, np.float64)
    pred = np.einsum("ij,ij->i", U[user], V[item])
    if not implicit:
        nu = np.bincount(user, minlength=U.shape[0])
        ni = np.bincount(item, minlength=V.shape[0])
        return float(((r - pred) ** 2).sum() + lam * ((nu * (U ** 2).sum(1)).sum() + (ni * (V ** 2).sum(1)).sum()))
    # implicit: sum over ALL (u,i) of c_ui (p_ui - x.y)^2, c = 1 + alpha|r| on observed, 1 elsewhere
    full = U @ V.T
    has_u = np.bincount(user, minlength=U.shape[0]) > 0
    has_i = np.bincount(item, minlength=V.shape[0]) > 0
    base = (full[np.ix_(has_u, has_i)] ** 2).sum()
    c1 = alpha * np.abs(r)
    p = (r > 0).astype(np.float64)
    # duplicates are separate terms, as in MLlib
    corr = (c1 * pred ** 2 + (1 + c1) * p * (1 - 2 * pred)).sum() - 0.0
    # (1+c1)(p - pred)^2 - pred^2 = c1 pred^2 + (1+c1) p^2 - 2(1+c1) p pred ; p^2 = p
    nu = np.bincount(user, weights=p, minlength=U.shape[0])
    ni = np.bincount(item, weights=p, minlength=V.shape[0])
    return float(base + corr + lam * ((nu * (U ** 2).sum(1)).sum() + (ni * (V ** 2).sum(1)).sum()))


# ----------------------------------------------------------------------------
# similarproduct CooccurrenceAlgorithm.trainCooccurrence (CooccurrenceAlgorithm.scala:72-105), restated with Python
# sets / dicts: distinct (user, item), all item pairs per user, count per pair, per item the topn by
# (count descending, item index ascending) -- the reference leaves ties unspecified.
# ----------------------------------------------------------------------------
def cooc_train(user, item, n_items, topn):
    from collections import defaultdict
    per_user = defaultdict(set)
    for u, i in zip(np.asarray(user).tolist(), np.asarray(item).tolist()):
        per_user[u].add(i)
    cnt = defaultdict(int)
    for items in per_user.values():
        li = sorted(items)
        for a in range(len(li)):
            for b in range(a + 1, len(li)):
                cnt[(li[a], li[b])] += 1
    per_item = defaultdict(list)
    for (a, b), c in cnt.items():
        per_item[a].append((b, c))
        per_item[b].append((a, c))
    oi = np.full((n_items, topn), -1, np.int32)
    oc = np.zeros((n_items, topn), np.int32)
    on = np.zeros(n_items, np.int32)
    for it, lst in per_item.items():
        lst.sort(key=lambda t: (-t[1], t[0]))
        for r, (o, c) in enumerate(lst[:topn]):
            oi[it, r], oc[it, r] = o, c
        on[it] = min(len(lst), topn)
    return oi, oc, on
