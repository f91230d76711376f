"""Plain fp64 restatement of one ALS half-step, and the error measures the row-by-row GPU tests apply to it.

For every destination row with ratings it forms MLlib's normal equations from the source factors (the same formula as
``oracle.numpy_half_step``, written independently of ``oracle/``):

  explicit: A = sum y y^T + lambda * n * I,                 b = sum r * y                 (n: ratings of the row)
  implicit: A = YtY + sum alpha|r| * y y^T + lambda * n+ * I, b = sum_{r > 0} (1 + alpha|r|) * y  (n+: positive ratings)

YtY is taken over every source row, so the caller passes source factors whose rows without ratings are zero (what the
library holds for them).  Duplicated (row, column) pairs are separate terms, as in MLlib.

Rows are processed in buckets of similar degree: each bucket gathers its ratings into a zero-padded
[rows, max degree, k] block, and the Gramians, solves and eigenvalues are batched NumPy calls at fp64.
"""
from __future__ import annotations

import os
from concurrent.futures import ThreadPoolExecutor
from dataclasses import dataclass

import numpy as np

_BLOCK = 1 << 21     # fp64 elements gathered per bucket (16 MB): the largest test cases take seconds, not minutes


@dataclass
class HalfStepRef:
    deg: np.ndarray        # int64 [n_dst]: ratings per destination row
    npos: np.ndarray       # int64 [n_dst]: positive ratings per row (implicit ridge count)
    b: np.ndarray          # fp64 [n_dst, k]
    x: np.ndarray          # fp64 [n_dst, k]: the exact-arithmetic solution x* (rows without ratings: 0)
    eta: np.ndarray | None = None     # backward error of the candidate, per row (inactive rows: 0)
    fwd: np.ndarray | None = None     # ||x^ - x*|| / ||x*|| (inactive rows: 0)
    kappa: np.ndarray | None = None   # 2-norm condition number of A (inactive rows: 1)
    fwd_bound: np.ndarray | None = None   # ||A^-1|| ||A x^ - b|| / ||x*||: what the residual allows fwd to be


def half_step(dst, col, val, n_dst, src, lam, implicit, alpha, cand=None) -> HalfStepRef:
    """Normal equations of every destination row from the COO ratings (dst[j], col[j], val[j]) and the source factors
    ``src`` [n_src, k]; with ``cand`` [n_dst, k] (a computed half-step) also its per-row backward and forward errors.

    Backward error (the primary measure, independent of the row's conditioning):
        eta = ||A x^ - b||_2 / (||A||_2 ||x^||_2 + || sum |w| |y| ||_2)
    where b = sum w y.  The right-hand side enters with the magnitude it is summed from rather than ||b||: a row's b can
    cancel to a small fraction of its terms (at rank 1 a single number, often 1e-3 of them), while the rounding error
    of any fp32 summation scales with the terms.  A plain sequential fp32 accumulation of such a rank-1 row has
    ||A x^ - b|| / (||A|| ||x^|| + ||b||) of 3e-4; measured with the terms' magnitude, 1.3e-7.
    """
    dst = np.asarray(dst, np.int64)
    col = np.asarray(col, np.int64)
    val = np.asarray(val, np.float64)
    s64 = np.asarray(src, np.float64)
    k = s64.shape[1]
    order = np.argsort(dst, kind="stable")
    scol, sval = col[order], val[order]
    deg = np.bincount(dst, minlength=n_dst).astype(np.int64)
    npos = np.bincount(dst, weights=(val > 0), minlength=n_dst).astype(np.int64)
    start = np.zeros(n_dst + 1, np.int64)
    start[1:] = np.cumsum(deg)
    yty = s64.T @ s64 if implicit else None
    out = HalfStepRef(deg, npos, np.zeros((n_dst, k)), np.zeros((n_dst, k)))
    if cand is not None:
        xh_all = np.asarray(cand, np.float64)
        out.eta, out.fwd, out.kappa, out.fwd_bound = np.zeros(n_dst), np.zeros(n_dst), np.ones(n_dst), np.zeros(n_dst)
    rows = np.flatnonzero(deg)
    rows = rows[np.argsort(deg[rows], kind="stable")]
    buckets, i = [], 0
    while i < rows.size:
        # grow the bucket while its padded gather and its matrices fit the block
        j = i + 1
        while j < rows.size and (j + 1 - i) * (deg[rows[j]] * k + k * k) <= _BLOCK:
            j += 1
        buckets.append(rows[i:j])
        i = j

    def solve_bucket(rb):
        d = int(deg[rb[-1]])
        pos = np.arange(d)
        mask = pos[None, :] < deg[rb][:, None]
        at = np.where(mask, start[rb][:, None] + pos[None, :], 0)
        Y = s64[scol[at]]                                  # [n, d, k]
        r = np.where(mask, sval[at], 0.0)                  # [n, d], padded ratings are 0
        if implicit:
            c1 = alpha * np.abs(r)
            A = yty[None] + np.matmul(np.swapaxes(Y * c1[..., None], 1, 2), Y)
            w = np.where(r > 0, 1.0 + c1, 0.0)
            reg = lam * npos[rb]
        else:
            A = np.matmul(np.swapaxes(Y * mask[..., None], 1, 2), Y)
            w = r
            reg = lam * deg[rb]
        A[:, np.arange(k), np.arange(k)] += reg[:, None]
        b = np.einsum("nd,ndk->nk", w, Y)
        babs = np.einsum("nd,ndk->nk", np.abs(w), np.abs(Y))
        x = np.linalg.solve(A, b[..., None])[..., 0]
        out.b[rb], out.x[rb] = b, x
        if cand is not None:
            xh = xh_all[rb]
            ev = np.linalg.eigvalsh(A)
            na = ev[:, -1]
            out.kappa[rb] = na / ev[:, 0]
            res = np.linalg.norm(np.matmul(A, xh[..., None])[..., 0] - b, axis=1)
            den = na * np.linalg.norm(xh, axis=1) + np.linalg.norm(babs, axis=1)
            out.eta[rb] = np.where(den > 0, res / np.where(den > 0, den, 1.0), np.where(res > 0, np.inf, 0.0))
            nx = np.linalg.norm(x, axis=1)
            dx = np.linalg.norm(xh - x, axis=1)
            out.fwd[rb] = np.where(nx > 0, dx / np.where(nx > 0, nx, 1.0), np.where(dx > 0, np.inf, 0.0))
            out.fwd_bound[rb] = np.where(nx > 0, res / ev[:, 0] / np.where(nx > 0, nx, 1.0), np.where(res > 0, np.inf, 0.0))

    # the batched LAPACK calls release the GIL: buckets (disjoint rows) run on a thread pool
    with ThreadPoolExecutor(max_workers=min(16, os.cpu_count() or 1)) as ex:
        list(ex.map(solve_bucket, buckets))
    return out

