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
from pathlib import Path

import numpy as np

PKG_DIR = Path(__file__).resolve().parent
REPO_ROOT = PKG_DIR.parent
LIB_PATH = PKG_DIR / "libpio_als.so"
CSRC = PKG_DIR / "csrc"

ABI_VERSION = 2
DEDUP_NONE, DEDUP_SUM, DEDUP_KEEP_LAST = 0, 1, 2
INIT_CALLER, INIT_HASH = 0, 1
SIM_KEEP_QUERY_ITEMS = 1
ERR_ARG, ERR_CUDA, ERR_STATE, ERR_NUMERIC, ERR_IO, ERR_COMM = -1, -2, -3, -4, -5, -6

EXPORTED_SYMBOLS = [
    "pio_als_abi_version", "pio_als_device_count", "pio_als_nccl_unique_id", "pio_als_create",
    "pio_als_destroy", "pio_als_last_error", "pio_als_set_ratings_coo", "pio_als_set_ratings_coo_device", "pio_als_set_ratings_coo_sharded",
    "pio_als_set_ratings_coo_sharded_device",
    "pio_als_set_init", "pio_als_run", "pio_als_get_factors", "pio_als_train", "pio_als_recommend",
    "pio_als_similar", "pio_als_similar_batch", "pio_als_model_import", "pio_als_save", "pio_als_load", "pio_als_get_stats", "pio_als_get_phase_ms",
    "pio_als_synth_ratings_device", "pio_nb_train", "pio_nb_predict", "pio_ids_encode", "pio_cooc_train",
    "pio_events_scan", "pio_events_scan_keys", "pio_events_fold",
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
                   "cos_batched": 0x20, "cos_fallback": 0x40, "multi_pass": 0x80}


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


def device_count() -> int:
    return int(lib().pio_als_device_count())


def nccl_unique_id() -> bytes:
    buf = (C.c_uint8 * 128)()
    rc = lib().pio_als_nccl_unique_id(buf)
    if rc != 0:
        raise NativeError(rc, lib().pio_als_last_error(None).decode())
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
        rc = lib().pio_als_create(C.byref(cfg), C.byref(self._h))
        if rc != 0:
            raise NativeError(rc, lib().pio_als_last_error(None).decode())

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
        if rc != 0:
            raise NativeError(rc, lib().pio_als_last_error(self._h).decode())

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

    def recommend(self, users, topk, item_mask=None, item_weight=None):
        users = np.ascontiguousarray(users, np.int32)
        n = users.shape[0]
        oi = np.full((n, topk), -1, np.int32)
        os_ = np.zeros((n, topk), np.float32)
        oc = np.zeros(n, np.int32)
        mk, wt = self._mask_weight(item_mask, item_weight)
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

    def similar_batch(self, queries, topk, item_mask=None, item_weight=None, keep_query_items=False):
        """queries: sequence of item-index sequences; returns (items [n, topk], scores [n, topk], count [n])."""
        n = len(queries)
        ptr = np.zeros(n + 1, np.int64)
        ptr[1:] = np.cumsum([len(q) for q in queries])
        flat = np.ascontiguousarray(np.concatenate([np.asarray(q, np.int32) for q in queries]) if n and ptr[-1] else
                                    np.zeros(0, np.int32), np.int32)
        oi = np.full((n, topk), -1, np.int32)
        os_ = np.zeros((n, topk), np.float32)
        oc = np.zeros(n, np.int32)
        mk, wt = self._mask_weight(item_mask, item_weight)
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
        rc = lib().pio_als_load(str(path).encode(), C.c_int(device), C.byref(h))
        if rc != 0:
            raise NativeError(rc, lib().pio_als_last_error(None).decode())
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
        rc = lib().pio_als_model_import(C.byref(cfg), _ptr(uf, C.c_float), _ptr(itf, C.c_float), _ptr(uh, C.c_uint8),
                                        _ptr(ih, C.c_uint8), C.byref(h))
        if rc != 0:
            raise NativeError(rc, lib().pio_als_last_error(None).decode())
        return cls(rank=int(k), n_users=max(int(nu), 1), n_items=int(ni), _handle=h)

    def stats(self) -> dict:
        st = Stats()
        self._check(lib().pio_als_get_stats(self._h, C.byref(st)))
        out = {name: getattr(st, name) for name, _ in Stats._fields_}
        # the scoring kernels of the last recommend / similar call, as a set of SCORE_PATH_BITS names
        out["last_score_path"] = {name for name, bit in SCORE_PATH_BITS.items() if st.last_score_path & bit}
        return out

    def phase_ms(self) -> dict:
        """Device-time breakdown of the last run (pio_als_get_phase_ms)."""
        out = (C.c_double * 8)()
        self._check(lib().pio_als_get_phase_ms(self._h, out))
        return {"item_solve_ms": out[0], "user_solve_ms": out[1], "gram_ms": out[2], "comm_ms": out[3],
                "item_kernel": _KERNEL_NAMES[int(out[4])], "user_kernel": _KERNEL_NAMES[int(out[5])],
                "iterations": int(out[6])}


def synth_ratings_device(device, n_users, n_items, nnz, seed, implicit, start, d_user, d_item, d_rating):
    rc = lib().pio_als_synth_ratings_device(C.c_int(device), C.c_int32(n_users), C.c_int32(n_items), C.c_int64(nnz),
                                            C.c_int64(seed), C.c_int(int(implicit)), C.c_int64(start),
                                            C.c_void_p(d_user), C.c_void_p(d_item), C.c_void_p(d_rating))
    if rc != 0:
        raise NativeError(rc, lib().pio_als_last_error(None).decode())


def ids_encode(strings, device=0):
    """BiMap.stringInt on the GPU: (index per string int32[n], first-occurrence position per distinct id int64[n_unique]).
    `strings`: a sequence of str / bytes, or a (bytes_buffer uint8[], offsets int64[n+1]) pair."""
    if isinstance(strings, tuple):
        buf, off = strings
        buf = np.ascontiguousarray(buf, np.uint8)
        off = np.ascontiguousarray(off, np.int64)
    else:
        enc = [s if isinstance(s, (bytes, bytearray)) else str(s).encode("utf-8") for s in strings]
        off = np.zeros(len(enc) + 1, np.int64)
        if enc:
            off[1:] = np.cumsum([len(b) for b in enc])
        buf = np.frombuffer(b"".join(enc), np.uint8) if enc else np.zeros(0, np.uint8)
    n = off.shape[0] - 1
    idx = np.empty(n, np.int32)
    first = np.empty(max(n, 1), np.int64)
    nu = C.c_int32(0)
    rc = lib().pio_ids_encode(C.c_int(device), _ptr(buf, C.c_uint8) if buf.size else None, _ptr(off, C.c_int64),
                              C.c_int64(n), _ptr(idx, C.c_int32), _ptr(first, C.c_int64), C.byref(nu))
    if rc != 0:
        raise NativeError(rc, lib().pio_als_last_error(None).decode())
    return idx, first[:nu.value]


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
    buf = np.frombuffer(text, np.uint8) if isinstance(text, (bytes, bytearray, memoryview)) else \
        np.ascontiguousarray(text, np.uint8)
    n = int(buf.shape[0])
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
    cap = n // EVENTS_MIN_EVENT_BYTES + 1
    out = dict(line=np.empty(cap, np.int64), code=np.empty(cap, np.int32), value=np.empty(cap, np.float64),
               flags=np.empty(cap, np.uint8), time_us=np.empty(cap, np.int64), eid_bytes=np.empty(max(n, 1), np.uint8),
               eid_off=np.empty(cap + 1, np.int64), tid_bytes=np.empty(max(n, 1), np.uint8),
               tid_off=np.empty(cap + 1, np.int64))
    cols = [("line", C.c_int64), ("code", C.c_int32), ("value", C.c_double), ("flags", C.c_uint8),
            ("time_us", C.c_int64), ("eid_bytes", C.c_uint8), ("eid_off", C.c_int64), ("tid_bytes", C.c_uint8),
            ("tid_off", C.c_int64)]
    nk = 0 if keys is None else len(keys)
    if keys is not None:
        kb = [k.encode("utf-8") if isinstance(k, str) else k for k in keys]
        kp = (C.c_char_p * max(nk, 1))(*kb)
        out.update(present=np.empty(cap, np.uint8), number=np.empty(cap, np.uint8), num=np.empty((cap, max(nk, 1))),
                   tok_bytes=np.empty(max(n, 1), np.uint8), tok_off=np.empty(cap * max(nk, 1) + 1, np.int64))
        cols += [("present", C.c_uint8), ("number", C.c_uint8), ("num", C.c_double), ("tok_bytes", C.c_uint8),
                 ("tok_off", C.c_int64)]
    fb_cap = max(1024, n // 4096)
    n_ev, n_fb, n_lines = C.c_int64(0), C.c_int64(0), C.c_int64(0)
    while True:
        fb = [np.empty(fb_cap, np.int64) for _ in range(3)]
        head = (C.c_int(device), _ptr(buf, C.c_uint8) if n else None, C.c_int64(n), C.byref(f))
        tail = (C.byref(n_ev), C.c_int64(fb_cap), *[_ptr(a, C.c_int64) for a in fb], C.byref(n_fb), C.byref(n_lines))
        if keys is None:
            rc = lib().pio_events_scan(*head, C.c_int64(cap), *[_ptr(out[k], t) for k, t in cols], *tail)
        else:
            rc = lib().pio_events_scan_keys(*head, kp, C.c_int(nk), C.c_int64(cap),
                                            *[_ptr(out[k], t) for k, t in cols], *tail)
        if rc != 0:
            raise NativeError(rc, lib().pio_als_last_error(None).decode())
        if n_fb.value <= fb_cap:
            break
        fb_cap = n_fb.value     # more fallback lines than room: once more with room for all of them
    m = n_ev.value
    res = {k: out[k][:m] for k in ("line", "code", "value", "flags", "time_us")}
    res["eid_off"], res["tid_off"] = out["eid_off"][:m + 1], out["tid_off"][:m + 1]
    res["eid_bytes"], res["tid_bytes"] = out["eid_bytes"][:res["eid_off"][-1]], out["tid_bytes"][:res["tid_off"][-1]]
    res["fb_line"], res["fb_begin"], res["fb_end"] = (a[:n_fb.value] for a in fb)
    res["n_lines"] = n_lines.value
    if keys is not None:
        res["present"], res["number"], res["num"] = out["present"][:m], out["number"][:m], out["num"][:m, :nk]
        res["tok_off"] = out["tok_off"][:m * nk + 1]
        res["tok_bytes"] = out["tok_bytes"][:res["tok_off"][-1]]
    return res


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
    rc = lib().pio_events_fold(C.c_int(device), _ptr(buf, C.c_uint8) if buf.size else None, _ptr(off, C.c_int64),
                               _ptr(code, C.c_int32), _ptr(time_us, C.c_int64), _ptr(pm, C.c_uint8), C.c_int64(n),
                               C.c_int(int(n_keys)), _ptr(first, C.c_int64), _ptr(exists, C.c_uint8), _ptr(fus, C.c_int64),
                               _ptr(lus, C.c_int64), _ptr(win, C.c_int64), C.byref(ne))
    if rc != 0:
        raise NativeError(rc, lib().pio_als_last_error(None).decode())
    g = ne.value
    return dict(first_event=first[:g], exists=exists[:g].astype(bool), first_us=fus[:g], last_us=lus[:g],
                winner=win[:g, :int(n_keys)])


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
    rc = lib().pio_cooc_train(C.c_int(device), _ptr(user, C.c_int32), _ptr(item, C.c_int32), C.c_int64(user.shape[0]),
                              C.c_int32(n_users), C.c_int32(n_items), C.c_int(topn), _ptr(oi, C.c_int32),
                              _ptr(oc, C.c_int32), _ptr(on, C.c_int32))
    if rc != 0:
        raise NativeError(rc, lib().pio_als_last_error(None).decode())
    return oi, oc, on


def nb_train(label, x, n_class, lam, device=0):
    label = np.ascontiguousarray(label, np.int32)
    x = np.ascontiguousarray(x, np.float32)
    n, f = x.shape
    pi = np.zeros(n_class, np.float64)
    theta = np.zeros((n_class, f), np.float64)
    rc = lib().pio_nb_train(C.c_int(device), _ptr(label, C.c_int32), _ptr(x, C.c_float), C.c_int64(n), C.c_int(f),
                            C.c_int(n_class), C.c_double(lam), _ptr(pi, C.c_double), _ptr(theta, C.c_double))
    if rc != 0:
        raise NativeError(rc, lib().pio_als_last_error(None).decode())
    return pi, theta


def nb_predict(x, pi, theta, device=0):
    x = np.ascontiguousarray(x, np.float32)
    pi = np.ascontiguousarray(pi, np.float64)
    theta = np.ascontiguousarray(theta, np.float64)
    n, f = x.shape
    out = np.zeros(n, np.int32)
    rc = lib().pio_nb_predict(C.c_int(device), _ptr(x, C.c_float), C.c_int64(n), C.c_int(f), C.c_int(pi.shape[0]),
                              _ptr(pi, C.c_double), _ptr(theta, C.c_double), _ptr(out, C.c_int32))
    if rc != 0:
        raise NativeError(rc, lib().pio_als_last_error(None).decode())
    return out
