"""ctypes binding of the C ABI in ``include/pio_als.h`` (library: ``libpio_als.so``).

This is the Python stand-in for the JNI shim a ``native-als`` Scala module would carry
(INTEGRATION.md): it only marshals host buffers and status codes; no arithmetic happens here
and there is no CPU fallback -- if the CUDA library is missing or no H100 is visible every
call raises ``NativeError``.
"""
from __future__ import annotations

import ctypes as C
import os
import subprocess
from dataclasses import dataclass, field
from pathlib import Path
from typing import Any, Dict, List, Optional, Sequence

import numpy as np

PKG_DIR = Path(__file__).resolve().parent
REPO_ROOT = PKG_DIR.parent
LIB_PATH = PKG_DIR / "libpio_als.so"
CSRC = PKG_DIR / "csrc"

ABI_VERSION = 2
DEDUP_NONE, DEDUP_SUM, DEDUP_KEEP_LAST = 0, 1, 2
INIT_CALLER, INIT_HASH = 0, 1
SIM_KEEP_QUERY_ITEMS = 1
ERR_ARG, ERR_CUDA, ERR_STATE, ERR_NUMERIC, ERR_IO, ERR_COMM, ERR_NOMEM = -1, -2, -3, -4, -5, -6, -7

EXPORTED_SYMBOLS = [
    "pio_als_abi_version", "pio_als_device_count", "pio_als_nccl_unique_id", "pio_als_create",
    "pio_als_destroy", "pio_als_last_error", "pio_als_set_ratings_coo", "pio_als_set_ratings_coo_device", "pio_als_set_ratings_coo_sharded",
    "pio_als_set_ratings_coo_sharded_device",
    "pio_als_set_init", "pio_als_run", "pio_als_get_factors", "pio_als_train", "pio_als_recommend",
    "pio_als_similar", "pio_als_similar_batch", "pio_als_recommend_filtered", "pio_als_similar_batch_filtered",
    "pio_als_model_import", "pio_als_save", "pio_als_load", "pio_als_get_stats", "pio_als_get_phase_ms",
    "pio_als_synth_ratings_device", "pio_nb_train", "pio_nb_predict", "pio_ids_encode", "pio_cooc_train",
    "pio_events_scan", "pio_events_scan_keys", "pio_events_fold", "pio_events_scan_props", "pio_events_fold_props",
    "pio_events_index_create",
    "pio_events_index_append", "pio_events_index_add_host", "pio_events_index_lookup", "pio_events_index_get_stats",
    "pio_events_index_destroy", "pio_rf_train", "pio_rf_forest_size", "pio_rf_forest_get", "pio_rf_forest_destroy",
    "pio_rf_predict", "pio_eval_folds_create", "pio_eval_folds_sizes", "pio_eval_folds_maps",
    "pio_eval_folds_set_ratings", "pio_eval_folds_result_add", "pio_eval_folds_result_free",
    "pio_eval_folds_rank_counts", "pio_eval_folds_destroy", "pio_cls_folds_create", "pio_cls_folds_sizes",
    "pio_cls_folds_classes", "pio_cls_folds_nb_train", "pio_cls_folds_rf_train", "pio_cls_folds_nb_predict",
    "pio_cls_folds_rf_predict", "pio_cls_folds_result_labels", "pio_cls_folds_result_counts",
    "pio_cls_folds_result_free", "pio_cls_folds_destroy", "pio_cooc_model_create", "pio_cooc_model_destroy",
    "pio_cooc_predict_filtered", "pio_cooc_model_get_stats", "pio_serve_zscore_merge", "pio_popular_model_create",
    "pio_popular_predict_filtered", "pio_popular_model_get_stats", "pio_popular_model_destroy", "pio_assoc_train",
    "pio_assoc_model_size", "pio_assoc_model_get", "pio_assoc_model_destroy",
]


_KERNEL_NAMES = {0: "fp32", 1: "wgmma", 2: "mma", 3: "pair"}


class NativeError(RuntimeError):
    def __init__(self, code: int, msg: str):
        super().__init__(f"pio_als error {code}: {msg}")
        self.code = code


class Config(C.Structure):
    _fields_ = [
        ("abi_version", C.c_int32), ("rank", C.c_int32), ("implicit_prefs", C.c_int32),
        ("n_users", C.c_int32), ("n_items", C.c_int32), ("device", C.c_int32),
        ("world_size", C.c_int32), ("world_rank", C.c_int32), ("init_mode", C.c_int32),
        ("reserved0", C.c_int32), ("lambda_", C.c_double), ("alpha", C.c_double),
        ("seed", C.c_int64), ("nccl_id", C.c_uint8 * 128),
    ]


class Stats(C.Structure):
    _fields_ = [
        ("nnz", C.c_int64), ("kernel_launches", C.c_int64), ("solve_launches", C.c_int64),
        ("last_run_ms", C.c_double), ("last_solve_ms", C.c_double), ("last_gram_ms", C.c_double),
        ("last_comm_ms", C.c_double), ("last_ingest_ms", C.c_double),
        ("n_users_active", C.c_int32), ("n_items_active", C.c_int32), ("sm_count", C.c_int32),
        ("last_score_path", C.c_int32),
    ]


# pio_als_stats.last_score_path bits (PIO_ALS_PATH_* in pio_als.h)
SCORE_PATH_BITS = {"score_one": 0x01, "dot_blocked": 0x02, "cos_blocked": 0x04, "dot_batched": 0x08, "cos_multi": 0x10,
                   "cos_batched": 0x20, "cos_fallback": 0x40, "multi_pass": 0x80, "filtered": 0x100, "listed": 0x200}


class _QueryFilterStruct(C.Structure):
    """pio_als_query_filter"""
    _fields_ = [
        ("ex_ptr", C.c_void_p), ("ex_items", C.c_void_p), ("has_wl", C.c_void_p), ("wl_ptr", C.c_void_p),
        ("wl_items", C.c_void_p), ("set_ix", C.c_void_p), ("item_sets", C.c_void_p), ("n_sets", C.c_int32),
    ]


def _csr(lists, n):
    """(ptr int64 [n + 1], flat int32) of n id lists; None entries are empty lists."""
    ptr = np.zeros(n + 1, np.int64)
    arrs = [np.zeros(0, np.int32) if l is None else np.asarray(l, np.int32).reshape(-1) for l in lists]
    if len(arrs) != n:
        raise ValueError(f"expected {n} lists, got {len(arrs)}")
    if n:
        ptr[1:] = np.cumsum([a.shape[0] for a in arrs])
    flat = np.ascontiguousarray(np.concatenate(arrs) if n and ptr[-1] else np.zeros(0, np.int32), np.int32)
    return ptr, flat


class QueryFilter:
    """The per-query filters of a batch scoring call (pio_als_query_filter), built from per-query Python lists or arrays.

    exclude    : n id lists (None = empty), the items query j may not return (black lists, seen items)
    white      : n entries, None = no white list, else the only items query j may return (an empty list: none)
    set_ix     : n rows of item_sets, -1 = none; item_sets: [n_sets, n_items] uint8, 1 = not a candidate
    Ids outside the item range and duplicates are ignored by the library."""

    def __init__(self, n_queries: int, exclude=None, white=None, set_ix=None, item_sets=None):
        self.n = int(n_queries)
        self.ex_ptr = self.ex_items = self.has_wl = self.wl_ptr = self.wl_items = self.set_ix = self.item_sets = None
        self.n_sets = 0
        if exclude is not None:
            self.ex_ptr, self.ex_items = _csr(exclude, self.n)
        if white is not None:
            if len(white) != self.n:
                raise ValueError(f"expected {self.n} white lists, got {len(white)}")
            self.has_wl = np.array([w is not None for w in white], np.uint8)
            self.wl_ptr, self.wl_items = _csr(white, self.n)
        if set_ix is not None:
            self.set_ix = np.ascontiguousarray(set_ix, np.int32)
            if self.set_ix.shape != (self.n,):
                raise ValueError("set_ix must have one entry per query")
            if item_sets is not None:
                self.item_sets = np.ascontiguousarray(item_sets, np.uint8)
                if self.item_sets.ndim != 2:
                    raise ValueError("item_sets must be [n_sets, n_items]")
                self.n_sets = int(self.item_sets.shape[0])

    def struct(self, n_queries: int, n_items: int) -> _QueryFilterStruct:
        """The C struct over this object's arrays (which must outlive the call)."""
        if n_queries != self.n:
            raise ValueError(f"query filter built for {self.n} queries, call has {n_queries}")
        if self.item_sets is not None and self.item_sets.shape[1] != n_items:
            raise ValueError("item_sets rows must have n_items entries")
        return _QueryFilterStruct(_addr(self.ex_ptr), _addr(self.ex_items), _addr(self.has_wl), _addr(self.wl_ptr),
                                  _addr(self.wl_items), _addr(self.set_ix), _addr(self.item_sets), self.n_sets)


NVCC_FLAGS = ["-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-lineinfo", "-std=c++17",
              "-Xcompiler", "-fPIC,-fvisibility=hidden", "-shared"]


def build(force: bool = False, verbose: bool = False) -> Path:
    """nvcc cross-compile of csrc/pio_als.cu for sm_90a (H100) into the in-tree libpio_als.so."""
    srcs = (sorted(CSRC.glob("*.cu")) + sorted(CSRC.glob("*.cuh")) + sorted(CSRC.glob("*.h")) +
            [REPO_ROOT / "include" / "pio_als.h"])
    if LIB_PATH.exists() and not force and all(LIB_PATH.stat().st_mtime >= s.stat().st_mtime for s in srcs):
        return LIB_PATH
    cmd = ["nvcc", *NVCC_FLAGS, "-o", str(LIB_PATH), str(CSRC / "pio_als.cu")]
    if verbose:
        cmd.insert(1, "-Xptxas=-v")
    subprocess.run(cmd, check=True)
    return LIB_PATH


_lib = None


def lib():
    """Load libpio_als.so; raises (no fallback) if it has not been built."""
    global _lib
    if _lib is None:
        if not LIB_PATH.exists():
            raise NativeError(ERR_CUDA, f"{LIB_PATH} is missing: run `python -c 'import __graft_entry__ as g; g.build()'`; "
                                        "there is no CPU fallback")
        L = C.CDLL(str(LIB_PATH), mode=C.RTLD_GLOBAL)
        L.pio_als_last_error.restype = C.c_char_p
        L.pio_als_last_error.argtypes = [C.c_void_p]
        L.pio_als_destroy.restype = None
        L.pio_als_destroy.argtypes = [C.c_void_p]
        # the serving calls take raw addresses (ndarray.ctypes.data): building typed ctypes pointers costs ~2 us each,
        # which is visible next to a 50 us query
        vp, ci = C.c_void_p, C.c_int
        L.pio_als_recommend.restype = ci
        L.pio_als_recommend.argtypes = [vp, vp, ci, ci, vp, vp, vp, vp, vp]
        L.pio_als_similar.restype = ci
        L.pio_als_similar.argtypes = [vp, vp, ci, ci, vp, vp, ci, vp, vp, vp]
        L.pio_als_similar_batch.restype = ci
        L.pio_als_similar_batch.argtypes = [vp, vp, vp, ci, ci, vp, vp, ci, vp, vp, vp]
        L.pio_als_recommend_filtered.restype = ci
        L.pio_als_recommend_filtered.argtypes = [vp, vp, ci, ci, vp, vp, vp, vp, vp, vp]
        L.pio_als_similar_batch_filtered.restype = ci
        L.pio_als_similar_batch_filtered.argtypes = [vp, vp, vp, ci, ci, vp, vp, ci, vp, vp, vp, vp]
        i64 = C.c_int64
        L.pio_events_index_lookup.restype = ci
        L.pio_events_index_lookup.argtypes = [vp, vp, vp, C.c_int32, i64, i64, vp, vp, vp, vp]
        L.pio_events_index_destroy.argtypes = [vp]
        L.pio_cooc_model_create.restype = ci
        L.pio_cooc_model_create.argtypes = [ci, C.c_int32, C.c_int32, vp, vp, vp, vp]
        L.pio_cooc_model_destroy.argtypes = [vp]
        L.pio_cooc_predict_filtered.restype = ci
        L.pio_cooc_predict_filtered.argtypes = [vp, vp, vp, C.c_int32, C.c_int32, vp, vp, vp, vp]
        L.pio_cooc_model_get_stats.argtypes = [vp, vp]
        L.pio_serve_zscore_merge.restype = ci
        L.pio_serve_zscore_merge.argtypes = [ci, C.c_int32, C.c_int32, C.c_int32, vp, vp, vp, vp, vp, C.c_int32, vp, vp,
                                             vp]
        L.pio_popular_model_create.restype = ci
        L.pio_popular_model_create.argtypes = [ci, C.c_int32, vp, vp]
        L.pio_popular_model_destroy.argtypes = [vp]
        L.pio_popular_predict_filtered.restype = ci
        L.pio_popular_predict_filtered.argtypes = [vp, C.c_int32, C.c_int32, vp, vp, vp, vp]
        L.pio_popular_model_get_stats.argtypes = [vp, vp]
        for name in EXPORTED_SYMBOLS:
            getattr(L, name)  # AttributeError if the ABI is incomplete
        _lib = L
    return _lib


def _ptr(a, t):
    if a is None:
        return None
    return a.ctypes.data_as(C.POINTER(t))


def _addr(a):
    """Raw address of a contiguous ndarray (None stays None) for entry points declared with c_void_p parameters."""
    return None if a is None else a.ctypes.data


def _check(rc, h=None):
    """Raises NativeError for a nonzero status, with the library's last error message (of handle h, if given)."""
    if rc != 0:
        raise NativeError(rc, lib().pio_als_last_error(h).decode())


def _str_column(enc):
    """A string column (bytes uint8[], offsets int64[n + 1]) from a list of already-encoded bytes."""
    off = np.zeros(len(enc) + 1, np.int64)
    off[1:] = np.cumsum([len(b) for b in enc], dtype=np.int64)
    return np.frombuffer(b"".join(enc), np.uint8), off


def device_count() -> int:
    return int(lib().pio_als_device_count())


def nccl_unique_id() -> bytes:
    buf = (C.c_uint8 * 128)()
    _check(lib().pio_als_nccl_unique_id(buf))
    return bytes(buf)


class NativeALS:
    """One training job / trained model behind an opaque ``pio_als_handle``."""

    def __init__(self, rank, n_users, n_items, lam=0.01, implicit=False, alpha=1.0, seed=0, device=0,
                 world_size=1, world_rank=0, nccl_id: bytes | None = None, init_mode=INIT_CALLER, _handle=None):
        self._h = C.c_void_p()
        self.rank, self.n_users, self.n_items = int(rank), int(n_users), int(n_items)
        if _handle is not None:
            self._h = _handle
            return
        cfg = Config()
        cfg.abi_version = ABI_VERSION
        cfg.rank, cfg.implicit_prefs = int(rank), int(bool(implicit))
        cfg.n_users, cfg.n_items, cfg.device = int(n_users), int(n_items), int(device)
        cfg.world_size, cfg.world_rank, cfg.init_mode = int(world_size), int(world_rank), int(init_mode)
        cfg.lambda_, cfg.alpha, cfg.seed = float(lam), float(alpha), int(seed)
        if nccl_id is not None:
            cfg.nccl_id[:] = list(nccl_id)
        _check(lib().pio_als_create(C.byref(cfg), C.byref(self._h)))

    # -- lifecycle --------------------------------------------------------------------------
    def close(self):
        if self._h:
            lib().pio_als_destroy(self._h)
            self._h = C.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def _check(self, rc):
        _check(rc, self._h)

    # -- training ---------------------------------------------------------------------------
    def set_ratings(self, user, item, rating, dedup=DEDUP_NONE, ts=None):
        user = np.ascontiguousarray(user, np.int32)
        item = np.ascontiguousarray(item, np.int32)
        rating = np.ascontiguousarray(rating, np.float32)
        if not (user.shape == item.shape == rating.shape) or user.ndim != 1:
            raise ValueError("user/item/rating must be 1-D arrays of equal length")
        tsa = None if ts is None else np.ascontiguousarray(ts, np.int64)
        self._check(lib().pio_als_set_ratings_coo(self._h, _ptr(user, C.c_int32), _ptr(item, C.c_int32),
                                                  _ptr(rating, C.c_float), C.c_int64(user.shape[0]),
                                                  C.c_int(dedup), _ptr(tsa, C.c_int64)))

    def set_ratings_device(self, d_user: int, d_item: int, d_rating: int, nnz: int, dedup=DEDUP_NONE, d_ts: int = 0,
                           sharded=False):
        """Raw device pointers (ints), e.g. ``tensor.data_ptr()``.  sharded: this rank's slice of the events."""
        f = lib().pio_als_set_ratings_coo_sharded_device if sharded else lib().pio_als_set_ratings_coo_device
        self._check(f(self._h, C.c_void_p(d_user), C.c_void_p(d_item), C.c_void_p(d_rating), C.c_int64(nnz), C.c_int(dedup),
                      C.c_void_p(d_ts) if d_ts else None))

    def set_ratings_sharded(self, user, item, rating, dedup=DEDUP_NONE, ts=None):
        """This rank's slice of the events (HOST arrays); collective over the ranks of the job."""
        user = np.ascontiguousarray(user, np.int32)
        item = np.ascontiguousarray(item, np.int32)
        rating = np.ascontiguousarray(rating, np.float32)
        tsa = None if ts is None else np.ascontiguousarray(ts, np.int64)
        self._check(lib().pio_als_set_ratings_coo_sharded(self._h, _ptr(user, C.c_int32), _ptr(item, C.c_int32),
                                                          _ptr(rating, C.c_float), C.c_int64(user.shape[0]),
                                                          C.c_int(dedup), _ptr(tsa, C.c_int64)))

    def set_init(self, user_factors, item_factors=None):
        uf = np.ascontiguousarray(user_factors, np.float32)
        if uf.shape != (self.n_users, self.rank):
            raise ValueError("user_factors must be n_users x rank")
        itf = None
        if item_factors is not None:
            itf = np.ascontiguousarray(item_factors, np.float32)
            if itf.shape != (self.n_items, self.rank):
                raise ValueError("item_factors must be n_items x rank")
        self._check(lib().pio_als_set_init(self._h, _ptr(uf, C.c_float), _ptr(itf, C.c_float)))

    def run(self, n_iters: int):
        self._check(lib().pio_als_run(self._h, C.c_int(n_iters)))

    def get_factors(self, out_user=None, out_item=None):
        uf = out_user if out_user is not None else np.empty((self.n_users, self.rank), np.float32)
        itf = out_item if out_item is not None else np.empty((self.n_items, self.rank), np.float32)
        uh = np.empty(self.n_users, np.uint8)
        ih = np.empty(self.n_items, np.uint8)
        self._check(lib().pio_als_get_factors(self._h, _ptr(uf, C.c_float), _ptr(itf, C.c_float),
                                              _ptr(uh, C.c_uint8), _ptr(ih, C.c_uint8)))
        return uf, itf, uh, ih

    def train(self, user, item, rating, n_iters, dedup=DEDUP_NONE, ts=None, user_init=None, item_init=None,
              out_user=None, out_item=None):
        """One-shot host COO -> host factors (the call a JNI ALS.train binding makes)."""
        user = np.ascontiguousarray(user, np.int32)
        item = np.ascontiguousarray(item, np.int32)
        rating = np.ascontiguousarray(rating, np.float32)
        tsa = None if ts is None else np.ascontiguousarray(ts, np.int64)
        ui = None if user_init is None else np.ascontiguousarray(user_init, np.float32)
        ii = None if item_init is None else np.ascontiguousarray(item_init, np.float32)
        uf = out_user if out_user is not None else np.empty((self.n_users, self.rank), np.float32)
        itf = out_item if out_item is not None else np.empty((self.n_items, self.rank), np.float32)
        uh = np.empty(self.n_users, np.uint8)
        ih = np.empty(self.n_items, np.uint8)
        self._check(lib().pio_als_train(self._h, _ptr(user, C.c_int32), _ptr(item, C.c_int32), _ptr(rating, C.c_float),
                                        C.c_int64(user.shape[0]), C.c_int(dedup), _ptr(tsa, C.c_int64),
                                        _ptr(ui, C.c_float), _ptr(ii, C.c_float), C.c_int(n_iters),
                                        _ptr(uf, C.c_float), _ptr(itf, C.c_float), _ptr(uh, C.c_uint8),
                                        _ptr(ih, C.c_uint8)))
        return uf, itf, uh, ih

    # -- scoring ----------------------------------------------------------------------------
    def _mask_weight(self, item_mask, item_weight):
        mk = None if item_mask is None else np.ascontiguousarray(item_mask, np.uint8)
        if mk is not None and mk.shape != (self.n_items,):
            raise ValueError("item_mask must have n_items entries")
        wt = None if item_weight is None else np.ascontiguousarray(item_weight, np.float64)
        if wt is not None and wt.shape != (self.n_items,):
            raise ValueError("item_weight must have n_items entries")
        return mk, wt

    def recommend(self, users, topk, item_mask=None, item_weight=None, query_filter=None):
        """query_filter (QueryFilter, one entry per user): pio_als_recommend_filtered."""
        users = np.ascontiguousarray(users, np.int32)
        n = users.shape[0]
        oi = np.full((n, topk), -1, np.int32)
        os_ = np.zeros((n, topk), np.float32)
        oc = np.zeros(n, np.int32)
        mk, wt = self._mask_weight(item_mask, item_weight)
        if query_filter is not None:
            qf = query_filter.struct(n, self.n_items)
            self._check(lib().pio_als_recommend_filtered(self._h, users.ctypes.data, n, topk, _addr(mk), _addr(wt),
                                                         C.addressof(qf), oi.ctypes.data, os_.ctypes.data, oc.ctypes.data))
            return oi, os_, oc
        self._check(lib().pio_als_recommend(self._h, users.ctypes.data, n, topk, _addr(mk), _addr(wt), oi.ctypes.data,
                                            os_.ctypes.data, oc.ctypes.data))
        return oi, os_, oc

    def similar(self, query_items, topk, item_mask=None, item_weight=None, keep_query_items=False):
        q = np.ascontiguousarray(query_items, np.int32)
        oi = np.full(topk, -1, np.int32)
        os_ = np.zeros(topk, np.float32)
        oc = np.zeros(1, np.int32)
        mk, wt = self._mask_weight(item_mask, item_weight)
        self._check(lib().pio_als_similar(self._h, q.ctypes.data, q.shape[0], topk, _addr(mk), _addr(wt),
                                          SIM_KEEP_QUERY_ITEMS if keep_query_items else 0, oi.ctypes.data,
                                          os_.ctypes.data, oc.ctypes.data))
        return oi, os_, int(oc[0])

    def similar_batch(self, queries, topk, item_mask=None, item_weight=None, keep_query_items=False, query_filter=None):
        """queries: sequence of item-index sequences; returns (items [n, topk], scores [n, topk], count [n]).
        query_filter (QueryFilter, one entry per query): pio_als_similar_batch_filtered."""
        n = len(queries)
        ptr = np.zeros(n + 1, np.int64)
        ptr[1:] = np.cumsum([len(q) for q in queries])
        flat = np.ascontiguousarray(np.concatenate([np.asarray(q, np.int32) for q in queries]) if n and ptr[-1] else
                                    np.zeros(0, np.int32), np.int32)
        oi = np.full((n, topk), -1, np.int32)
        os_ = np.zeros((n, topk), np.float32)
        oc = np.zeros(n, np.int32)
        mk, wt = self._mask_weight(item_mask, item_weight)
        if query_filter is not None:
            qf = query_filter.struct(n, self.n_items)
            self._check(lib().pio_als_similar_batch_filtered(
                self._h, ptr.ctypes.data, flat.ctypes.data, n, topk, _addr(mk), _addr(wt),
                SIM_KEEP_QUERY_ITEMS if keep_query_items else 0, C.addressof(qf), oi.ctypes.data, os_.ctypes.data,
                oc.ctypes.data))
            return oi, os_, oc
        self._check(lib().pio_als_similar_batch(self._h, ptr.ctypes.data, flat.ctypes.data, n, topk, _addr(mk), _addr(wt),
                                                SIM_KEEP_QUERY_ITEMS if keep_query_items else 0, oi.ctypes.data,
                                                os_.ctypes.data, oc.ctypes.data))
        return oi, os_, oc

    # -- persistence / introspection -----------------------------------------------------------
    def save(self, path: str):
        self._check(lib().pio_als_save(self._h, str(path).encode()))

    @classmethod
    def load(cls, path: str, device: int = 0) -> "NativeALS":
        h = C.c_void_p()
        _check(lib().pio_als_load(str(path).encode(), C.c_int(device), C.byref(h)))
        # read the header for the shape
        hdr = np.fromfile(path, dtype=np.int32, count=8)
        return cls(rank=int(hdr[3]), n_users=int(hdr[5]), n_items=int(hdr[6]), _handle=h)

    @classmethod
    def from_factors(cls, user_factors, item_factors, user_has=None, item_has=None, device: int = 0, lam=0.0,
                     implicit=False, alpha=1.0) -> "NativeALS":
        """pio_als_model_import: a scoring handle from host factors (user_factors may be None: item-only model)."""
        itf = np.ascontiguousarray(item_factors, np.float32)
        ni, k = itf.shape
        uf = None if user_factors is None else np.ascontiguousarray(user_factors, np.float32)
        nu = 0 if uf is None else uf.shape[0]
        cfg = Config()
        cfg.abi_version, cfg.rank, cfg.implicit_prefs = ABI_VERSION, int(k), int(bool(implicit))
        cfg.n_users, cfg.n_items, cfg.device, cfg.world_size = int(nu), int(ni), int(device), 1
        cfg.lambda_, cfg.alpha = float(lam), float(alpha)
        uh = None if user_has is None else np.ascontiguousarray(user_has, np.uint8)
        ih = None if item_has is None else np.ascontiguousarray(item_has, np.uint8)
        h = C.c_void_p()
        _check(lib().pio_als_model_import(C.byref(cfg), _ptr(uf, C.c_float), _ptr(itf, C.c_float), _ptr(uh, C.c_uint8),
                                          _ptr(ih, C.c_uint8), C.byref(h)))
        return cls(rank=int(k), n_users=max(int(nu), 1), n_items=int(ni), _handle=h)

    def stats(self) -> dict:
        st = Stats()
        self._check(lib().pio_als_get_stats(self._h, C.byref(st)))
        out = {name: getattr(st, name) for name, _ in Stats._fields_}
        # the scoring kernels of the last recommend / similar call, as a set of SCORE_PATH_BITS names
        out["last_score_path"] = {name for name, bit in SCORE_PATH_BITS.items() if st.last_score_path & bit}
        return out

    _SIDE_SCALARS = ("n", "R", "n_internal", "bits", "nnz_local", "n_active", "n_heavy", "n_parts", "nnz", "heavy_t",
                     "part_len")

    def debug_side(self, side: str) -> dict:
        """What the last set_ratings built on one side ("user" or "item") of this rank (pio_als_debug_side, debug only):
        the scalars of _SIDE_SCALARS, then deg / npos / perm / rpos per external row, inv per internal row (-1: padding),
        the local CSR ptr / idx / val, nreg per local row, and the heavy rows' part bounds part_beg / part_end and
        row_part_ptr."""
        f = lib().pio_als_debug_side
        sc = np.zeros(len(self._SIDE_SCALARS), np.int64)
        which = {"user": 0, "item": 1}[side]
        nul = [None] * 12
        self._check(f(self._h, C.c_int(which), _ptr(sc, C.c_int64), *nul))
        out = dict(zip(self._SIDE_SCALARS, (int(x) for x in sc)))
        n, R, nl = out["n"], out["R"], out["nnz_local"]
        arrs = dict(deg=np.empty(n, np.uint32), npos=np.empty(n, np.uint32), perm=np.empty(n, np.int32),
                    inv=np.empty(out["n_internal"], np.int32), rpos=np.empty(n, np.int32), ptr=np.empty(R + 1, np.int64),
                    idx=np.empty(nl, np.int32), val=np.empty(nl, np.float32), nreg=np.empty(R, np.float32),
                    part_beg=np.empty(out["n_parts"], np.int64), part_end=np.empty(out["n_parts"], np.int64),
                    row_part_ptr=np.zeros(out["n_heavy"] + 1, np.int32))
        self._check(f(self._h, C.c_int(which), _ptr(sc, C.c_int64), *(C.c_void_p(a.ctypes.data) for a in arrs.values())))
        out.update(arrs)
        return out

    def phase_ms(self) -> dict:
        """Device-time breakdown of the last run (pio_als_get_phase_ms)."""
        out = (C.c_double * 8)()
        self._check(lib().pio_als_get_phase_ms(self._h, out))
        return {"item_solve_ms": out[0], "user_solve_ms": out[1], "gram_ms": out[2], "comm_ms": out[3],
                "item_kernel": _KERNEL_NAMES[int(out[4])], "user_kernel": _KERNEL_NAMES[int(out[5])],
                "iterations": int(out[6])}


def synth_ratings_device(device, n_users, n_items, nnz, seed, implicit, start, d_user, d_item, d_rating):
    _check(lib().pio_als_synth_ratings_device(C.c_int(device), C.c_int32(n_users), C.c_int32(n_items), C.c_int64(nnz),
                                              C.c_int64(seed), C.c_int(int(implicit)), C.c_int64(start),
                                              C.c_void_p(d_user), C.c_void_p(d_item), C.c_void_p(d_rating)))


def ids_encode(strings, device=0):
    """BiMap.stringInt on the GPU: (index per string int32[n], first-occurrence position per distinct id int64[n_unique]).
    `strings`: a sequence of str / bytes, or a (bytes_buffer uint8[], offsets int64[n+1]) pair."""
    if isinstance(strings, tuple):
        buf, off = strings
        buf = np.ascontiguousarray(buf, np.uint8)
        off = np.ascontiguousarray(off, np.int64)
    else:
        buf, off = _str_column([s if isinstance(s, (bytes, bytearray)) else str(s).encode("utf-8") for s in strings])
    n = off.shape[0] - 1
    idx = np.empty(n, np.int32)
    first = np.empty(max(n, 1), np.int64)
    nu = C.c_int32(0)
    _check(lib().pio_ids_encode(C.c_int(device), _ptr(buf, C.c_uint8) if buf.size else None, _ptr(off, C.c_int64),
                                C.c_int64(n), _ptr(idx, C.c_int32), _ptr(first, C.c_int64), C.byref(nu)))
    return idx, first[:nu.value]


class EvalFolds:
    """pio_eval_folds: the k-fold split of n ratings on the device (rating e tests in fold e % k_fold and trains in every
    other fold), from global user / item indices (ids_encode of the whole columns) and fp64 ratings.  Per fold: the
    fold-local BiMap.stringInt indices of its training ratings, its training COO, and its queries (distinct test users in
    order of first occurrence).  The device memory goes with this object; EvalResult objects keep it alive."""

    def __init__(self, user, item, rating, k_fold: int, device: int = 0):
        self._h = C.c_void_p()
        user = np.ascontiguousarray(user, np.int32)
        item = np.ascontiguousarray(item, np.int32)
        rating = np.ascontiguousarray(rating, np.float64)
        if not (user.shape == item.shape == rating.shape) or user.ndim != 1:
            raise ValueError("user/item/rating must be 1-D arrays of equal length")
        self.k_fold, self.device = int(k_fold), int(device)
        _check(lib().pio_eval_folds_create(C.c_int(device), _ptr(user, C.c_int32), _ptr(item, C.c_int32),
                                           _ptr(rating, C.c_double), C.c_int64(user.shape[0]), C.c_int32(k_fold),
                                           C.byref(self._h)))

    def close(self):
        if self._h:
            lib().pio_eval_folds_destroy(self._h)
            self._h = C.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def sizes(self, fold: int) -> tuple:
        """(users, items, training ratings, queries) of fold `fold`."""
        out = np.zeros(4, np.int64)
        _check(lib().pio_eval_folds_sizes(self._h, C.c_int32(fold), _ptr(out, C.c_int64)))
        return tuple(int(x) for x in out)

    def maps(self, fold: int) -> dict:
        """Global index of each fold-local user / item, and per query its global user and fold-local training user
        (-1: none)."""
        nu, ni, _, nq = self.sizes(fold)
        out = {"user": np.empty(nu, np.int32), "item": np.empty(ni, np.int32), "query_user": np.empty(nq, np.int32),
               "query_train_user": np.empty(nq, np.int32)}
        _check(lib().pio_eval_folds_maps(self._h, C.c_int32(fold), *_addrs(out, "user", "item", "query_user",
                                                                           "query_train_user")))
        return out

    def set_ratings(self, fold: int, als: "NativeALS"):
        """The fold's training COO into `als` (created with the fold's user and item counts)."""
        _check(lib().pio_eval_folds_set_ratings(self._h, C.c_int32(fold), als._h))

    def add_result(self, fold: int, items, count) -> "EvalResult":
        """Keeps a top-N result of the fold (items [n_queries, num] of fold-local indices, count [n_queries])."""
        items = np.ascontiguousarray(items, np.int32)
        count = np.ascontiguousarray(count, np.int32)
        if items.ndim != 2 or count.shape != (items.shape[0],):
            raise ValueError("items must be [n_queries, num] and count [n_queries]")
        rid = C.c_int32(-1)
        _check(lib().pio_eval_folds_result_add(self._h, C.c_int32(fold), _ptr(items, C.c_int32), _ptr(count, C.c_int32),
                                               C.c_int32(items.shape[0]), C.c_int32(items.shape[1]), C.byref(rid)))
        return EvalResult(self, fold, rid.value, items, count)


class EvalResult:
    """A fold's top-N result kept on the device by its EvalFolds (which it keeps alive); `items` / `count` are the host
    arrays it was made from."""

    def __init__(self, folds: EvalFolds, fold: int, rid: int, items: np.ndarray, count: np.ndarray):
        self.folds, self.fold, self._rid, self.items, self.count = folds, fold, rid, items, count
        self.n_queries = int(count.shape[0])

    def rank_counts(self, k: int, threshold: float):
        """Per query (int32 each): hits among the first min(k, count) items, distinct test items with a largest rating
        >= threshold, and test ratings >= threshold."""
        out = {name: np.zeros(self.n_queries, np.int32) for name in ("hits", "npos", "nraw")}
        _check(lib().pio_eval_folds_rank_counts(self.folds._h, C.c_int32(self._rid), C.c_int32(k), C.c_double(threshold),
                                                *_addrs(out, "hits", "npos", "nraw")))
        return out["hits"], out["npos"], out["nraw"]

    def close(self):
        if self._rid is not None and self.folds._h:
            lib().pio_eval_folds_result_free(self.folds._h, C.c_int32(self._rid))
        self._rid = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


class ClsFolds:
    """pio_cls_folds: the k-fold split of n labeled points on the device (row i tests in fold i % k_fold and trains in
    every other fold, in row order), from fp64 labels and n x n_feat fp64 features.  Folds train NaiveBayes / RandomForest
    and predict their test rows without their rows leaving the device.  The device memory goes with this object;
    ClsResult objects keep it alive."""

    def __init__(self, label, x, k_fold: int, device: int = 0):
        self._h = C.c_void_p()
        label = np.ascontiguousarray(label, np.float64)
        x = np.ascontiguousarray(x, np.float64)
        if x.ndim != 2 or label.shape != (x.shape[0],):
            raise ValueError("x must be n x n_feat and label must have n entries")
        self.k_fold, self.device, self.n_feat = int(k_fold), int(device), int(x.shape[1])
        _check(lib().pio_cls_folds_create(C.c_int(device), _ptr(label, C.c_double), _ptr(x, C.c_double),
                                          C.c_int64(x.shape[0]), C.c_int32(x.shape[1]), C.c_int32(k_fold),
                                          C.byref(self._h)))

    def close(self):
        if self._h:
            lib().pio_cls_folds_destroy(self._h)
            self._h = C.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def sizes(self, fold: int) -> tuple:
        """(training rows, test rows) of fold `fold`."""
        out = np.zeros(2, np.int64)
        _check(lib().pio_cls_folds_sizes(self._h, C.c_int32(fold), _ptr(out, C.c_int64)))
        return int(out[0]), int(out[1])

    def classes(self, fold: int) -> np.ndarray:
        """The distinct labels of the fold's training rows, ascending."""
        nc = C.c_int32(0)
        _check(lib().pio_cls_folds_classes(self._h, C.c_int32(fold), C.byref(nc), None))
        out = np.empty(nc.value, np.float64)
        _check(lib().pio_cls_folds_classes(self._h, C.c_int32(fold), C.byref(nc), _ptr(out, C.c_double)))
        return out

    def nb_train(self, fold: int, lam: float, n_class: int):
        """(pi, theta) of NaiveBayes on the fold's training rows; n_class = len(classes(fold))."""
        pi = np.zeros(n_class, np.float64)
        theta = np.zeros((n_class, self.n_feat), np.float64)
        _check(lib().pio_cls_folds_nb_train(self._h, C.c_int32(fold), C.c_double(lam), C.c_int32(n_class),
                                            _ptr(pi, C.c_double), _ptr(theta, C.c_double)))
        return pi, theta

    def rf_train(self, fold: int, num_classes, num_trees, strategy, impurity, max_depth, max_bins, seed=0) -> dict:
        """rf_train on the fold's training rows: the forest as rf_train's dict of flat per-node arrays."""
        p = _rf_params(num_classes, num_trees, strategy, impurity, max_depth, max_bins, seed)
        h = C.c_void_p()
        _check(lib().pio_cls_folds_rf_train(self._h, C.c_int32(fold), C.byref(p), C.byref(h)))
        return _rf_forest_take(h)

    def nb_predict(self, fold: int, pi, theta, class_label) -> "ClsResult":
        """The NaiveBayes model's predicted labels (class_label[class]) of the fold's test rows, kept on the device."""
        pi = np.ascontiguousarray(pi, np.float64)
        theta = np.ascontiguousarray(theta, np.float64)
        class_label = np.ascontiguousarray(class_label, np.float64)
        if theta.shape != (pi.shape[0], self.n_feat) or class_label.shape != pi.shape:
            raise ValueError("theta must be n_class x n_feat and class_label must have n_class entries")
        rid = C.c_int32(-1)
        _check(lib().pio_cls_folds_nb_predict(self._h, C.c_int32(fold), C.c_int32(pi.shape[0]), _ptr(pi, C.c_double),
                                              _ptr(theta, C.c_double), _ptr(class_label, C.c_double), C.byref(rid)))
        return ClsResult(self, fold, rid.value)

    def rf_predict(self, fold: int, forest: dict, num_classes: int) -> "ClsResult":
        """The forest's predicted labels (class index) of the fold's test rows, kept on the device."""
        args, _arrays = _rf_flat(forest, num_classes)
        rid = C.c_int32(-1)
        _check(lib().pio_cls_folds_rf_predict(self._h, C.c_int32(fold), *args, C.byref(rid)))
        return ClsResult(self, fold, rid.value)


class ClsResult:
    """The predicted labels of one fold's test rows, kept on the device by its ClsFolds (which it keeps alive)."""

    def __init__(self, folds: ClsFolds, fold: int, rid: int):
        self.folds, self.fold, self._rid = folds, fold, rid
        self.n_rows = folds.sizes(fold)[1]

    def labels(self) -> np.ndarray:
        out = np.empty(self.n_rows, np.float64)
        _check(lib().pio_cls_folds_result_labels(self.folds._h, C.c_int32(self._rid), _ptr(out, C.c_double)))
        return out

    def counts(self, label: float = 0.0) -> tuple:
        """(test rows, rows predicted correctly, rows predicted as `label`, those of them that are correct)."""
        out = np.zeros(4, np.int64)
        _check(lib().pio_cls_folds_result_counts(self.folds._h, C.c_int32(self._rid), C.c_double(label),
                                                 _ptr(out, C.c_int64)))
        return tuple(int(v) for v in out)

    def close(self):
        if self._rid is not None and self.folds._h:
            lib().pio_cls_folds_result_free(self.folds._h, C.c_int32(self._rid))
        self._rid = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


EVENTS_TARGET_ANY, EVENTS_TARGET_ABSENT, EVENTS_TARGET_EQUALS = 0, 1, 2
EVENTS_MIN_EVENT_BYTES = 64
EVENTS_HAS_VALUE, EVENTS_HAS_TARGET = 1, 2


class EventsFilter(C.Structure):
    _fields_ = [
        ("entity_type", C.c_char_p), ("event_names", C.POINTER(C.c_char_p)), ("n_event_names", C.c_int32),
        ("target_entity_type_mode", C.c_int32), ("target_entity_type", C.c_char_p), ("property", C.c_char_p),
        ("has_start", C.c_int32), ("has_until", C.c_int32), ("start_us", C.c_int64), ("until_us", C.c_int64),
    ]


EVENTS_MAX_KEYS = 8


def events_scan(text, entity_type=None, event_names=None, target_mode=EVENTS_TARGET_ANY, target_entity_type=None,
                prop=None, start_us=None, until_us=None, device=0):
    """pio_events_scan over one buffer of complete JSON lines (bytes / uint8 array).  Returns a dict of numpy columns:
    line, code, value, flags, time_us, eid_bytes/eid_off, tid_bytes/tid_off (matched events, line order), fb_line,
    fb_begin, fb_end (lines the caller parses) and n_lines."""
    return _events_scan(text, entity_type, event_names, target_mode, target_entity_type, prop, start_us, until_us,
                        device, None)


def events_scan_keys(text, keys, entity_type=None, event_names=None, target_mode=EVENTS_TARGET_ANY,
                     target_entity_type=None, start_us=None, until_us=None, device=0):
    """pio_events_scan_keys: events_scan's columns plus, per matched event, the top-level `properties` keys `keys`:
    present / number (uint8 bit masks, bit q = keys[q]), num (float64 [n, n_keys]) and the raw JSON tokens as a string
    column tok_bytes / tok_off with n_keys slots per event (slot e * n_keys + q)."""
    return _events_scan(text, entity_type, event_names, target_mode, target_entity_type, None, start_us, until_us,
                        device, list(keys))


def _events_scan(text, entity_type, event_names, target_mode, target_entity_type, prop, start_us, until_us, device,
                 keys):
    """pio_events_scan (keys None) or pio_events_scan_keys, with any filter (the ABI refuses a keyed scan with prop)."""
    filt = (entity_type, event_names, target_mode, target_entity_type, prop, start_us, until_us)
    if keys is None:
        return _scan(text, filt, device, lambda n, cap: {},
                     lambda head, base, out, tail: lib().pio_events_scan(*head, *base, *tail))[0]
    kb = [k.encode("utf-8") if isinstance(k, str) else k for k in keys]
    nk = len(kb)
    kp = (C.c_char_p * max(nk, 1))(*kb)
    res, out = _scan(
        text, filt, device,
        lambda n, cap: dict(present=np.empty(cap, np.uint8), number=np.empty(cap, np.uint8),
                            num=np.empty((cap, max(nk, 1))), tok_bytes=np.empty(max(n, 1), np.uint8),
                            tok_off=np.empty(cap * max(nk, 1) + 1, np.int64)),
        lambda head, base, out, tail: lib().pio_events_scan_keys(
            *head, kp, C.c_int(nk), *base, *_addrs(out, "present", "number", "num", "tok_bytes", "tok_off"), *tail))
    m = len(res["line"])
    res["present"], res["number"], res["num"] = out["present"][:m], out["number"][:m], out["num"][:m, :nk]
    _take_strings(res, out, "tok", m * nk)
    return res


EVENTS_MIN_RECORD_BYTES = 4


def events_scan_props(text, entity_type=None, event_names=None, target_mode=EVENTS_TARGET_ANY, target_entity_type=None,
                      start_us=None, until_us=None, device=0):
    """pio_events_scan_props: events_scan's columns plus, per matched event, utc_off (eventTime's UTC offset in minutes,
    int16) and prop_off (int64 [n + 1]: its records), and per record r, one per top-level key of `properties` in object
    order: the decoded key key_bytes[key_off[r]:key_off[r + 1]] and the raw JSON token of its value
    tok_bytes[tok_off[r]:tok_off[r + 1]]."""
    rcap, n_rec = C.c_int64(0), C.c_int64(0)

    def cols(n, cap):
        rcap.value = n // EVENTS_MIN_RECORD_BYTES + 1
        return dict(utc_off=np.empty(cap, np.int16), prop_off=np.empty(cap + 1, np.int64),
                    key_bytes=np.empty(max(n, 1), np.uint8), key_off=np.empty(rcap.value + 1, np.int64),
                    tok_bytes=np.empty(max(n, 1), np.uint8), tok_off=np.empty(rcap.value + 1, np.int64))

    res, out = _scan(
        text, (entity_type, event_names, target_mode, target_entity_type, None, start_us, until_us), device, cols,
        lambda head, base, out, tail: lib().pio_events_scan_props(
            *head, *base, *_addrs(out, "utc_off", "prop_off"), rcap,
            *_addrs(out, "key_bytes", "key_off", "tok_bytes", "tok_off"), tail[0], C.byref(n_rec), *tail[1:]))
    m = len(res["line"])
    res["utc_off"], res["prop_off"] = out["utc_off"][:m], out["prop_off"][:m + 1]
    for k in ("key", "tok"):
        _take_strings(res, out, k, n_rec.value)
    return res


_SCAN_COLS = (("line", np.int64), ("code", np.int32), ("value", np.float64), ("flags", np.uint8),
              ("time_us", np.int64))


def _scan(text, filt, device, extra_cols, call):
    """What every event scan marshals: the text buffer, the filter (filt: _events_filter's arguments), the base columns,
    the second call with room for every fallback line, and the slicing of the base results.  extra_cols(n_bytes, cap)
    gives the scan's own output arrays; call(head, base, out, tail) makes its ABI call, where head is (device, text,
    n_bytes, filter), base is (capacity, the base columns), out holds every output array and tail is (n_events,
    fallback capacity, the three fallback columns, n_fallback, n_lines).  Returns the dict of base results and `out`,
    from which the caller slices its own columns."""
    buf = np.frombuffer(text, np.uint8) if isinstance(text, (bytes, bytearray, memoryview)) else \
        np.ascontiguousarray(text, np.uint8)
    n = int(buf.shape[0])
    f, keep = _events_filter(*filt)
    cap = n // EVENTS_MIN_EVENT_BYTES + 1
    out = {k: np.empty(cap, t) for k, t in _SCAN_COLS}
    out.update(eid_bytes=np.empty(max(n, 1), np.uint8), eid_off=np.empty(cap + 1, np.int64),
               tid_bytes=np.empty(max(n, 1), np.uint8), tid_off=np.empty(cap + 1, np.int64), **extra_cols(n, cap))
    head = (C.c_int(device), _ptr(buf, C.c_uint8) if n else None, C.c_int64(n), C.byref(f))
    base = (C.c_int64(cap), *_addrs(out, *[k for k, _ in _SCAN_COLS], "eid_bytes", "eid_off", "tid_bytes", "tid_off"))
    fb_cap = max(1024, n // 4096)
    n_ev, n_fb, n_lines = C.c_int64(0), C.c_int64(0), C.c_int64(0)
    while True:
        fb = [np.empty(fb_cap, np.int64) for _ in range(3)]
        _check(call(head, base, out, (C.byref(n_ev), C.c_int64(fb_cap), *[_ptr(a, C.c_int64) for a in fb],
                                      C.byref(n_fb), C.byref(n_lines))))
        if n_fb.value <= fb_cap:
            break
        fb_cap = n_fb.value     # more fallback lines than room: once more with room for all of them
    m = n_ev.value
    res = {k: out[k][:m] for k, _ in _SCAN_COLS}
    for k in ("eid", "tid"):
        _take_strings(res, out, k, m)
    res["fb_line"], res["fb_begin"], res["fb_end"] = (a[:n_fb.value] for a in fb)
    res["n_lines"] = n_lines.value
    return res, out


def _addrs(out, *keys):
    return [C.c_void_p(_addr(out[k])) for k in keys]


def _take_strings(res, out, name, count):
    """res[name_off], res[name_bytes]: the first `count` strings of the string column out[name_bytes / name_off]."""
    res[name + "_off"] = out[name + "_off"][:count + 1]
    res[name + "_bytes"] = out[name + "_bytes"][:res[name + "_off"][-1]]


def events_fold_props(eid, code, time_us, prop_off, keys, device=0):
    """pio_events_fold_props: LEventAggregator's fold of every key, over $set (code 0) / $unset (1) / $delete (2)
    events in file order whose records (one per key of `properties`, object order) are prop_off[e]:prop_off[e + 1] of
    keys = (bytes uint8[], offsets int64[n_records + 1]).  eid: (bytes, offsets).  Returns, per entity in order of first
    occurrence: first_event, exists (bool), first_time_event / last_time_event (the events giving firstUpdated /
    lastUpdated), win_off (int64 [n_entities + 1]) over win_rec (the record holding each key's value, in the map's
    order) and win_key (its key code); and key_first (the first record of each key code)."""
    buf, off = np.ascontiguousarray(eid[0], np.uint8), np.ascontiguousarray(eid[1], np.int64)
    kbuf, koff = np.ascontiguousarray(keys[0], np.uint8), np.ascontiguousarray(keys[1], np.int64)
    code = np.ascontiguousarray(code, np.int32)
    time_us = np.ascontiguousarray(time_us, np.int64)
    prop_off = np.ascontiguousarray(prop_off, np.int64)
    n = int(code.shape[0])
    nr = int(prop_off[-1]) if prop_off.size else 0
    first, exists = np.empty(max(n, 1), np.int64), np.empty(max(n, 1), np.uint8)
    fev, lev, woff = np.empty(max(n, 1), np.int64), np.empty(max(n, 1), np.int64), np.empty(n + 1, np.int64)
    wrec, wkey, kfirst = np.empty(max(nr, 1), np.int64), np.empty(max(nr, 1), np.int32), np.empty(max(nr, 1), np.int64)
    ne, nk = C.c_int64(0), C.c_int64(0)
    _check(lib().pio_events_fold_props(
        C.c_int(device), _ptr(buf, C.c_uint8) if buf.size else None, _ptr(off, C.c_int64), _ptr(code, C.c_int32),
        _ptr(time_us, C.c_int64), _ptr(prop_off, C.c_int64), C.c_int64(n), _ptr(kbuf, C.c_uint8) if kbuf.size else None,
        _ptr(koff, C.c_int64), _ptr(first, C.c_int64), _ptr(exists, C.c_uint8), _ptr(fev, C.c_int64),
        _ptr(lev, C.c_int64), _ptr(woff, C.c_int64), _ptr(wrec, C.c_int64), _ptr(wkey, C.c_int32),
        _ptr(kfirst, C.c_int64), C.byref(ne), C.byref(nk)))
    g = ne.value
    w_off = woff[:g + 1] if g else np.zeros(1, np.int64)
    nw = int(w_off[-1])
    return dict(first_event=first[:g], exists=exists[:g].astype(bool), first_time_event=fev[:g],
                last_time_event=lev[:g], win_off=w_off, win_rec=wrec[:nw], win_key=wkey[:nw], key_first=kfirst[:nk.value])


def events_fold(eid, code, time_us, present=None, n_keys=0, device=0):
    """pio_events_fold: LEventAggregator's fold of $set (code 0) / $unset (1) / $delete (2) events in file order, per
    entity in order of first occurrence.  eid: (bytes uint8[], offsets int64[n + 1]).  Returns a dict: first_event,
    exists (bool), first_us, last_us, winner (int64 [n_entities, n_keys], -1 = key absent)."""
    buf = np.ascontiguousarray(eid[0], np.uint8)
    off = np.ascontiguousarray(eid[1], np.int64)
    code = np.ascontiguousarray(code, np.int32)
    time_us = np.ascontiguousarray(time_us, np.int64)
    n = int(code.shape[0])
    pm = None if present is None else np.ascontiguousarray(present, np.uint8)
    first, exists = np.empty(max(n, 1), np.int64), np.empty(max(n, 1), np.uint8)
    fus, lus = np.empty(max(n, 1), np.int64), np.empty(max(n, 1), np.int64)
    win = np.empty((max(n, 1), max(int(n_keys), 1)), np.int64)
    ne = C.c_int64(0)
    _check(lib().pio_events_fold(C.c_int(device), _ptr(buf, C.c_uint8) if buf.size else None, _ptr(off, C.c_int64),
                                 _ptr(code, C.c_int32), _ptr(time_us, C.c_int64), _ptr(pm, C.c_uint8), C.c_int64(n),
                                 C.c_int(int(n_keys)), _ptr(first, C.c_int64), _ptr(exists, C.c_uint8), _ptr(fus, C.c_int64),
                                 _ptr(lus, C.c_int64), _ptr(win, C.c_int64), C.byref(ne)))
    g = ne.value
    return dict(first_event=first[:g], exists=exists[:g].astype(bool), first_us=fus[:g], last_us=lus[:g],
                winner=win[:g, :int(n_keys)])


class EventsIndexStats(C.Structure):
    _fields_ = [("n_main", C.c_int64), ("n_delta", C.c_int64), ("n_merges", C.c_int64), ("scan_ms", C.c_double),
                ("sort_ms", C.c_double), ("merge_ms", C.c_double)]


def _events_filter(entity_type, event_names, target_mode, target_entity_type, prop, start_us, until_us):
    """A pio_events_filter, and the ctypes objects its pointers refer to (keep both alive together)."""
    names = [] if event_names is None else [x.encode("utf-8") for x in event_names]
    f = EventsFilter()
    keep = (C.c_char_p * max(len(names), 1))(*names)
    f.entity_type = None if entity_type is None else entity_type.encode("utf-8")
    f.event_names = None if event_names is None else keep   # None: any name; []: no event matches (as in find)
    f.n_event_names = len(names)
    f.target_entity_type_mode = int(target_mode)
    f.target_entity_type = None if target_entity_type is None else target_entity_type.encode("utf-8")
    f.property = None if prop is None else prop.encode("utf-8")
    f.has_start, f.start_us = (0, 0) if start_us is None else (1, int(start_us))
    f.has_until, f.until_us = (0, 0) if until_us is None else (1, int(until_us))
    return f, keep


class EventsIndex:
    """pio_events_index: the events of one view (entity type, event names, target entity type) of an append-only event
    file on the device, looked up by entityId in LEventStore.findByEntity's order (latest first, file order among equal
    times).  Lines are given by byte offset and length in the file."""

    def __init__(self, entity_type, event_names, target_mode=EVENTS_TARGET_ANY, target_entity_type=None, device=0):
        self._h = C.c_void_p()
        f, keep = _events_filter(entity_type, event_names, target_mode, target_entity_type, None, None, None)
        self._check(lib().pio_events_index_create(C.c_int(device), C.byref(f), C.byref(self._h)))

    def _check(self, rc):
        _check(rc)

    def close(self):
        if self._h:
            lib().pio_events_index_destroy(self._h)
            self._h = C.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def append(self, text, base_offset: int):
        """Indexes the complete lines `text` (bytes / memoryview), whose first byte is at `base_offset` in the file.
        Returns the fallback lines as (begin, end) file offsets, in line order: the caller parses them and adds the
        matching ones with add_host."""
        buf = np.frombuffer(text, np.uint8)
        n = int(buf.shape[0])
        fb_cap = max(1024, n // 4096)
        n_fb = C.c_int64(0)
        while True:
            fb = [np.empty(fb_cap, np.int64) for _ in range(2)]
            self._check(lib().pio_events_index_append(self._h, _ptr(buf, C.c_uint8) if n else None, C.c_int64(n),
                                                      C.c_int64(base_offset), C.c_int64(fb_cap),
                                                      *[_ptr(a, C.c_int64) for a in fb], C.byref(n_fb)))
            if n_fb.value <= fb_cap:
                break
            fb_cap = n_fb.value     # nothing was added: once more with room for every fallback line
        return fb[0][:n_fb.value] + base_offset, fb[1][:n_fb.value] + base_offset

    def add_host(self, ids, time_us, offset, length):
        """Events parsed on the host, in file order: entityId strings, eventTime (us), line offset and length."""
        enc = [x.encode("utf-8", "surrogatepass") for x in ids]
        buf, off = _str_column(enc)
        t, o, ln = (np.ascontiguousarray(a, d) for a, d in ((time_us, np.int64), (offset, np.int64), (length, np.int32)))
        self._check(lib().pio_events_index_add_host(self._h, _ptr(buf, C.c_uint8) if buf.size else None,
                                                    _ptr(off, C.c_int64), _ptr(t, C.c_int64), _ptr(o, C.c_int64),
                                                    _ptr(ln, C.c_int32), C.c_int64(len(enc))))

    def lookup(self, ids, limit=None):
        """For each entityId of `ids` (str): (offsets int64[], lengths int32[]) of its lines, latest first, at most
        `limit` (None or negative: all)."""
        buf, off = _str_column([x.encode("utf-8", "surrogatepass") for x in ids])
        n = off.shape[0] - 1
        lim = -1 if limit is None else int(limit)
        count = np.zeros(max(n, 1), np.int64)
        total = C.c_int64(0)
        cap = max(16, 16 * n if lim < 0 else lim * n)
        while True:
            ro, rl = np.empty(cap, np.int64), np.empty(cap, np.int32)
            self._check(lib().pio_events_index_lookup(self._h, buf.ctypes.data if buf.size else None, off.ctypes.data,
                                                      n, lim, cap, count.ctypes.data, C.addressof(total),
                                                      ro.ctypes.data, rl.ctypes.data))
            if total.value <= cap:
                break
            cap = total.value       # the result did not fit: ask again with room for all of it
        pos = np.zeros(n + 1, np.int64)
        np.cumsum(count[:n], out=pos[1:])
        return [(ro[pos[k]:pos[k + 1]], rl[pos[k]:pos[k + 1]]) for k in range(n)]

    def stats(self) -> dict:
        st = EventsIndexStats()
        self._check(lib().pio_events_index_get_stats(self._h, C.byref(st)))
        return {name: getattr(st, name) for name, _ in EventsIndexStats._fields_}


def events_scan_timing() -> dict:
    """Where the last events_scan on this thread spent its time (milliseconds, summed over its device chunks):
    host-to-device copy, kernels, device-to-host copy (CUDA events), and the host copy into pinned staging."""
    out = (C.c_double * 5)()
    rc = lib().pio_events_debug_timing(out)
    if rc != 0:
        raise NativeError(rc, "pio_events_debug_timing")
    return {"h2d_ms": out[0], "kernel_ms": out[1], "d2h_ms": out[2], "stage_ms": out[3], "chunks": int(out[4])}


def cooc_train(user, item, n_users, n_items, topn, device=0):
    """CooccurrenceAlgorithm.trainCooccurrence on the GPU: (items [n_items, topn], counts [n_items, topn], n [n_items])."""
    user = np.ascontiguousarray(user, np.int32)
    item = np.ascontiguousarray(item, np.int32)
    oi = np.full((n_items, topn), -1, np.int32)
    oc = np.zeros((n_items, topn), np.int32)
    on = np.zeros(n_items, np.int32)
    _check(lib().pio_cooc_train(C.c_int(device), _ptr(user, C.c_int32), _ptr(item, C.c_int32), C.c_int64(user.shape[0]),
                                C.c_int32(n_users), C.c_int32(n_items), C.c_int(topn), _ptr(oi, C.c_int32),
                                _ptr(oc, C.c_int32), _ptr(on, C.c_int32)))
    return oi, oc, on


class CoocStats(C.Structure):
    _fields_ = [("kernel_launches", C.c_int64), ("last_expanded", C.c_int64), ("last_rows", C.c_int64),
                ("last_budget", C.c_int64), ("last_parts", C.c_int32), ("last_max_part_queries", C.c_int32)]


class CoocModel:
    """pio_cooc_model: a trained co-occurrence model (cooc_train's three arrays) that scores batches of
    CooccurrenceAlgorithm queries on `device`.  The arrays are checked and copied when it is created; the device copy is
    made by the first predict_filtered."""

    def __init__(self, top_items, top_counts, top_n, device: int = 0):
        ti = np.ascontiguousarray(top_items, np.int32)
        tc = np.ascontiguousarray(top_counts, np.int32)
        tn = np.ascontiguousarray(top_n, np.int32)
        if ti.ndim != 2 or tc.shape != ti.shape or tn.shape != (ti.shape[0],):
            raise ValueError("top_items / top_counts must be [n_items, n] and top_n [n_items]")
        self.n_items, self.topn = int(ti.shape[0]), int(ti.shape[1])
        self._h = C.c_void_p()
        _check(lib().pio_cooc_model_create(int(device), self.n_items, self.topn, ti.ctypes.data, tc.ctypes.data,
                                           tn.ctypes.data, C.addressof(self._h)))

    def close(self):
        if self._h:
            lib().pio_cooc_model_destroy(self._h)
            self._h = C.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def predict_filtered(self, q_lists, num: int, query_filter=None):
        """q_lists: n item-index sequences; query_filter: QueryFilter with one entry per query, or None.  Returns
        (items int32 [n, num], scores int64 [n, num], count int32 [n])."""
        ptr, flat = _csr(q_lists, len(q_lists))
        n = ptr.shape[0] - 1
        oi = np.full((n, num), -1, np.int32)
        os_ = np.zeros((n, num), np.int64)
        oc = np.zeros(n, np.int32)
        qf = None if query_filter is None else query_filter.struct(n, self.n_items)
        _check(lib().pio_cooc_predict_filtered(self._h, ptr.ctypes.data, flat.ctypes.data, n, int(num),
                                               None if qf is None else C.addressof(qf), oi.ctypes.data,
                                               os_.ctypes.data, oc.ctypes.data))
        return oi, os_, oc

    def stats(self) -> dict:
        st = CoocStats()
        _check(lib().pio_cooc_model_get_stats(self._h, C.addressof(st)))
        return {name: getattr(st, name) for name, _ in CoocStats._fields_}


class PopularStats(C.Structure):
    _fields_ = [("kernel_launches", C.c_int64), ("last_walked", C.c_int64), ("last_listed", C.c_int64),
                ("last_parts", C.c_int32), ("last_max_part_queries", C.c_int32)]


class PopularModel:
    """pio_popular_model: one fixed fp64 score per item (no NaN) that ranks batches of filtered queries on `device`, best
    score first, equal scores by item index.  The scores are checked and copied when it is created; the device copy and
    its ranked order are made by the first predict_filtered."""

    def __init__(self, scores, device: int = 0):
        sc = np.ascontiguousarray(scores, np.float64)
        if sc.ndim != 1:
            raise ValueError("scores must be [n_items]")
        self.n_items = int(sc.shape[0])
        self._h = C.c_void_p()
        _check(lib().pio_popular_model_create(int(device), self.n_items, sc.ctypes.data, C.addressof(self._h)))

    def close(self):
        if self._h:
            lib().pio_popular_model_destroy(self._h)
            self._h = C.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def predict_filtered(self, n_queries: int, topk: int, query_filter=None):
        """n_queries queries, each with its entry of query_filter (QueryFilter, or None: no filter).  Returns
        (items int32 [n, topk], scores float64 [n, topk], count int32 [n])."""
        n = int(n_queries)
        oi = np.full((max(n, 0), topk), -1, np.int32)
        os_ = np.zeros((max(n, 0), topk), np.float64)
        oc = np.zeros(max(n, 0), np.int32)
        qf = None if query_filter is None else query_filter.struct(n, self.n_items)
        _check(lib().pio_popular_predict_filtered(self._h, n, int(topk), None if qf is None else C.addressof(qf),
                                                  oi.ctypes.data, os_.ctypes.data, oc.ctypes.data))
        return oi, os_, oc

    def stats(self) -> dict:
        st = PopularStats()
        _check(lib().pio_popular_model_get_stats(self._h, C.addressof(st)))
        return {name: getattr(st, name) for name, _ in PopularStats._fields_}


@dataclass
class ScoredColumns:
    """A batch of ranked results as arrays: row j holds query j's first count[j] (item id, score) pairs, best first,
    padded with -1 / 0, and names[id] is the item string of an id.  The rows of the queries in `objects` are not used:
    those queries' results are given there as the result objects of predict (or, once served, of serve).  device: the
    GPU whose model computed them, or None."""
    items: np.ndarray                 # int32 [Q, w]
    scores: np.ndarray                # float64 [Q, w]
    count: np.ndarray                 # int32 [Q]
    names: Sequence[str]
    objects: Dict[int, Any] = field(default_factory=dict)
    device: Optional[int] = None


def item_names(string_int) -> List[str]:
    """The item strings of a string -> index map whose indices are 0 .. size - 1, in index order."""
    names = [None] * len(string_int)
    for s, i in string_int.toSeq():
        names[i] = s
    return names


def serve_zscore_merge(items, scores, counts, num, topk: int, n_items: int, device: int = 0):
    """pio_serve_zscore_merge: per algorithm a, items[a] int32 [Q, w_a], scores[a] float64 [Q, w_a] and counts[a] [Q],
    ids in [0, n_items); num [Q] >= 1.  Returns (items int32 [Q, topk], scores float64 [Q, topk], count int32 [Q])."""
    its = [np.ascontiguousarray(x, np.int32) for x in items]
    scs = [np.ascontiguousarray(x, np.float64) for x in scores]
    cns = [np.ascontiguousarray(c, np.int32) for c in counts]
    num = np.ascontiguousarray(num, np.int32)
    n, k = num.shape[0], len(its)
    if not (len(scs) == len(cns) == k) or any(x.ndim != 2 or x.shape[0] != n or s.shape != x.shape or c.shape != (n,)
                                              for x, s, c in zip(its, scs, cns)):
        raise ValueError("items / scores must be [n_queries, w] and counts [n_queries] for every algorithm")
    widths = np.array([x.shape[1] for x in its], np.int32)
    arr = lambda xs: (C.c_void_p * max(k, 1))(*[x.ctypes.data for x in xs])   # noqa: E731
    pi, ps, pc = arr(its), arr(scs), arr(cns)
    oi = np.full((n, topk), -1, np.int32)
    os_ = np.zeros((n, topk), np.float64)
    oc = np.zeros(n, np.int32)
    _check(lib().pio_serve_zscore_merge(int(device), n, k, int(n_items), C.addressof(pi), C.addressof(ps),
                                        C.addressof(pc), widths.ctypes.data, num.ctypes.data, int(topk), oi.ctypes.data,
                                        os_.ctypes.data, oc.ctypes.data))
    return oi, os_, oc


def serve_merge_stats() -> dict:
    """What the last serve_zscore_merge on this thread did: its parts, the most queries in one part, its entries and
    distinct (query, item) rows, the entries budget, and the device milliseconds from the first upload to the last copy
    back."""
    out = (C.c_double * 6)()
    _check(lib().pio_serve_merge_debug_stats(out))
    return {"parts": int(out[0]), "max_part_queries": int(out[1]), "entries": int(out[2]), "rows": int(out[3]),
            "budget": int(out[4]), "device_ms": out[5]}


def nb_train(label, x, n_class, lam, device=0):
    label = np.ascontiguousarray(label, np.int32)
    x = np.ascontiguousarray(x, np.float32)
    n, f = x.shape
    pi = np.zeros(n_class, np.float64)
    theta = np.zeros((n_class, f), np.float64)
    _check(lib().pio_nb_train(C.c_int(device), _ptr(label, C.c_int32), _ptr(x, C.c_float), C.c_int64(n), C.c_int(f),
                              C.c_int(n_class), C.c_double(lam), _ptr(pi, C.c_double), _ptr(theta, C.c_double)))
    return pi, theta


RF_GINI, RF_ENTROPY = 0, 1
RF_FOREST_INT = ("feature", "left", "right", "prediction")
RF_FOREST_F64 = ("threshold", "impurity", "gain")


class RfParams(C.Structure):
    _fields_ = [("num_classes", C.c_int32), ("num_trees", C.c_int32), ("max_depth", C.c_int32),
                ("max_bins", C.c_int32), ("impurity", C.c_int32), ("reserved0", C.c_int32),
                ("feature_subset_strategy", C.c_char_p), ("seed", C.c_int64)]


def rf_train(label, x, num_classes, num_trees, strategy, impurity, max_depth, max_bins, seed=0, device=0):
    """pio_rf_train: a RandomForest classifier (impurity RF_GINI / RF_ENTROPY) as a dict of flat per-node arrays:
    tree_off (int32 [num_trees + 1]), feature, left, right, prediction (int32), threshold, impurity, gain (float64) and
    count (int64)."""
    label = np.ascontiguousarray(label, np.float64)
    x = np.ascontiguousarray(x, np.float64)
    if x.ndim != 2 or label.shape != (x.shape[0],):
        raise ValueError("x must be n x n_feat and label must have n entries")
    p = _rf_params(num_classes, num_trees, strategy, impurity, max_depth, max_bins, seed)
    h = C.c_void_p()
    _check(lib().pio_rf_train(C.c_int(device), C.byref(p), _ptr(label, C.c_double), _ptr(x, C.c_double),
                              C.c_int64(x.shape[0]), C.c_int32(x.shape[1]), C.byref(h)))
    return _rf_forest_take(h)


def _rf_params(num_classes, num_trees, strategy, impurity, max_depth, max_bins, seed) -> RfParams:
    return RfParams(num_classes=int(num_classes), num_trees=int(num_trees), max_depth=int(max_depth),
                    max_bins=int(max_bins), impurity=int(impurity), feature_subset_strategy=str(strategy).encode("utf-8"),
                    seed=int(seed))


def _rf_forest_take(h) -> dict:
    """The flat arrays of the pio_rf_forest h, which is destroyed."""
    try:
        nt, nn = C.c_int32(0), C.c_int64(0)
        _check(lib().pio_rf_forest_size(h, C.byref(nt), C.byref(nn)))
        out = {"tree_off": np.empty(nt.value + 1, np.int32), "count": np.empty(nn.value, np.int64)}
        out.update({k: np.empty(nn.value, np.int32) for k in RF_FOREST_INT})
        out.update({k: np.empty(nn.value, np.float64) for k in RF_FOREST_F64})
        _check(lib().pio_rf_forest_get(h, *_addrs(out, "tree_off", "feature", "threshold", "left", "right", "prediction",
                                                  "impurity", "gain", "count")))
    finally:
        lib().pio_rf_forest_destroy(h)
    return out


def rf_predict(forest, num_classes, x, device=0):
    """pio_rf_predict: the forest's vote (class index, int32 [n]) for the rows of x (n x n_feat)."""
    x = np.ascontiguousarray(x, np.float64)
    n = x.shape[0]
    out = np.empty(n, np.int32)
    vp = C.c_void_p
    args, _arrays = _rf_flat(forest, num_classes)
    _check(lib().pio_rf_predict(C.c_int(device), *args, vp(_addr(x)), C.c_int64(n), C.c_int32(x.shape[1]),
                                vp(_addr(out))))
    return out


def _rf_flat(forest, num_classes):
    """(pio_rf_predict's forest arguments n_trees .. num_classes, the contiguous arrays they point into): the arrays
    must outlive the call."""
    a = {k: np.ascontiguousarray(forest[k], np.int32) for k in ("tree_off", *RF_FOREST_INT)}
    a["threshold"] = np.ascontiguousarray(forest["threshold"], np.float64)
    vp = C.c_void_p
    args = [C.c_int32(a["tree_off"].shape[0] - 1), vp(_addr(a["tree_off"])), C.c_int64(a["threshold"].shape[0]),
            vp(_addr(a["feature"])), vp(_addr(a["threshold"])), vp(_addr(a["left"])), vp(_addr(a["right"])),
            vp(_addr(a["prediction"])), C.c_int32(num_classes)]
    return args, a


def rf_train_timing() -> dict:
    """Where the last rf_train on this thread spent its time (wall ms of phases that each end in a device synchronise)."""
    out = (C.c_double * 70)()
    _check(lib().pio_rf_debug_timing(out))
    levels = int(out[6])
    return {"h2d_ms": out[0], "split_ms": out[1], "bin_ms": out[2], "hist_ms": out[3], "select_ms": out[4],
            "update_ms": out[5], "levels": levels, "groups": int(out[7]),
            "hist_level_ms": list(out[8:8 + levels]), "select_level_ms": list(out[39:39 + levels])}


def rf_train_paths() -> dict:
    """Which paths the last rf_train on this thread took: bin code width in bytes, thresholds staged in shared memory,
    shared-memory and global histogram launches, the most histogram chunks in one level, the most shared-memory passes
    in one chunk, levels and tree groups."""
    out = (C.c_int64 * 8)()
    _check(lib().pio_rf_debug_paths(out))
    keys = ("bin_bytes", "staged", "smem_launches", "global_launches", "max_chunks", "max_passes", "levels", "groups")
    return {k: int(v) for k, v in zip(keys, out)}


class AssocParams(C.Structure):
    """pio_assoc_params"""
    _fields_ = [("basket_window", C.c_int32), ("max_rule_length", C.c_int32), ("min_support", C.c_double),
                ("min_confidence", C.c_double), ("min_lift", C.c_double), ("min_basket_size", C.c_int32),
                ("max_num_rules_per_cond", C.c_int32)]


ASSOC_MAX_CANDIDATES = 1 << 29   # PIO_ASSOC_MAX_CANDIDATES


def assoc_train(user, item, t_ms, n_users, n_items, basket_window, max_rule_length, min_support, min_confidence,
                min_lift, min_basket_size, max_num_rules_per_cond, device=0) -> dict:
    """pio_assoc_train: the complementary purchase template's association rules from buy events (user / item indices,
    t_ms milliseconds).  Returns flat arrays: level_off (int64 [n_levels + 1]); per frequent set set_prefix (int64, -1
    for one item), set_item (int32, the set's largest item) and set_count (int64); per rule, grouped by cond and
    ranked, rule_cond (int64 set index), rule_conseq (int32), support, confidence and lift (float64); and
    n_transactions."""
    user = np.ascontiguousarray(user, np.int32)
    item = np.ascontiguousarray(item, np.int32)
    t_ms = np.ascontiguousarray(t_ms, np.int64)
    n = user.shape[0]
    if item.shape != (n,) or t_ms.shape != (n,):
        raise ValueError("user, item and t_ms must have one entry per event")
    p = AssocParams(int(basket_window), int(max_rule_length), float(min_support), float(min_confidence),
                    float(min_lift), int(min_basket_size), int(max_num_rules_per_cond))
    h = C.c_void_p()
    vp = C.c_void_p
    _check(lib().pio_assoc_train(C.c_int(device), vp(_addr(user)), vp(_addr(item)), vp(_addr(t_ms)), C.c_int64(n),
                                 C.c_int32(n_users), C.c_int32(n_items), C.byref(p), C.byref(h)))
    try:
        nl, ns, nr, nt = C.c_int32(0), C.c_int64(0), C.c_int64(0), C.c_int64(0)
        _check(lib().pio_assoc_model_size(h, C.byref(nl), C.byref(ns), C.byref(nr), C.byref(nt)))
        out = {"level_off": np.zeros(nl.value + 1, np.int64), "set_prefix": np.empty(ns.value, np.int64),
               "set_item": np.empty(ns.value, np.int32), "set_count": np.empty(ns.value, np.int64),
               "rule_cond": np.empty(nr.value, np.int64), "rule_conseq": np.empty(nr.value, np.int32),
               "support": np.empty(nr.value, np.float64), "confidence": np.empty(nr.value, np.float64),
               "lift": np.empty(nr.value, np.float64)}
        _check(lib().pio_assoc_model_get(h, *[vp(_addr(out[k])) for k in ASSOC_ARRAYS]))
    finally:
        lib().pio_assoc_model_destroy(h)
    out["n_transactions"] = int(nt.value)
    return out


ASSOC_ARRAYS = ("level_off", "set_prefix", "set_item", "set_count", "rule_cond", "rule_conseq", "support", "confidence",
                "lift")


def assoc_train_timing() -> dict:
    """Where the last assoc_train on this thread spent its time (wall ms of phases that each end in a device
    synchronise), the baskets before minBasketSize, the transactions, the levels >= 2 enumerated, the level the
    candidate limit rejected (0: none) and the candidates counted for each level k >= 2."""
    out = (C.c_double * 64)()
    _check(lib().pio_assoc_debug_timing(out))
    keys = ("h2d_ms", "baskets_ms", "level1_ms", "levels_ms", "rules_ms", "rank_ms", "d2h_ms", "total_ms")
    res = {k: out[j] for j, k in enumerate(keys)}
    res.update(baskets=int(out[8]), transactions=int(out[9]), levels_run=int(out[10]), rejected_level=int(out[11]),
               candidates={k: int(out[16 + k]) for k in range(2, 33) if out[16 + k]})
    return res


def nb_predict(x, pi, theta, device=0):
    x = np.ascontiguousarray(x, np.float32)
    pi = np.ascontiguousarray(pi, np.float64)
    theta = np.ascontiguousarray(theta, np.float64)
    n, f = x.shape
    out = np.zeros(n, np.int32)
    _check(lib().pio_nb_predict(C.c_int(device), _ptr(x, C.c_float), C.c_int64(n), C.c_int(f), C.c_int(pi.shape[0]),
                                _ptr(pi, C.c_double), _ptr(theta, C.c_double), _ptr(out, C.c_int32)))
    return out
