"""GPU tests (-m gpu) of the two primitives of csrc/sort_scan.cuh that ingest, dedup, row ranking, the sharded exchange,
ids_encode, the event scan / fold / index, co-occurrence, the forest and the evaluation folds are built on, called
directly through the debug entries pio_debug_radix_sort and pio_debug_scan_u32:

- the stable LSD radix sort of (uint64 key, uint32 payload) by key bits [0, nbits): the payload must come back as numpy's
  stable argsort of key & (2^nbits - 1), and the keys permuted with it.  Sizes step over the warp (RS_WARP_ITEMS) and
  tile (RS_TILE) boundaries and one sort has more than SCAN_TILE^2 / 256 tiles, so the scan of its digit histogram
  recurses three levels; nbits gives odd and even pass counts (the result then lies in either half of the ping-pong);
  the key distributions put whole warps on one digit, and set bits above nbits that must not order the keys.
- the exclusive uint32 scan, in place and out of place: sums mod 2^32 of numpy's uint64 cumsum, at sizes around
  SCAN_TILE and SCAN_TILE^2 (two and three recursion levels).
"""
import ctypes as C

import numpy as np
import pytest

import test_gpu_halfstep as G

pytestmark = pytest.mark.gpu

K = G.source_constants("sort_scan.cuh")
RS_TILE, RS_WARP_ITEMS, SCAN_TILE = K["RS_TILE"], K["RS_WARP_ITEMS"], K["SCAN_TILE"]


def radix_sort(native, keys, nbits):
    k = np.array(keys, np.uint64)
    v = np.arange(k.shape[0], dtype=np.uint32)
    rc = native.lib().pio_debug_radix_sort(C.c_int(0), k.ctypes.data_as(C.c_void_p), v.ctypes.data_as(C.c_void_p),
                                           C.c_int64(k.shape[0]), C.c_int(nbits))
    assert rc == 0, native.lib().pio_als_last_error(None)
    return k, v


def scan(native, x, in_place):
    out = np.zeros_like(x)
    rc = native.lib().pio_debug_scan_u32(C.c_int(0), x.ctypes.data_as(C.c_void_p), out.ctypes.data_as(C.c_void_p),
                                         C.c_int64(x.shape[0]), C.c_int(int(in_place)))
    assert rc == 0, native.lib().pio_als_last_error(None)
    return out


def low_mask(nbits):
    return np.uint64((1 << nbits) - 1)


def make_keys(dist, n, nbits, seed):
    rng = np.random.default_rng(seed)
    m = low_mask(nbits)
    full = rng.integers(0, 2 ** 64, n, dtype=np.uint64, endpoint=False)
    if dist == "uniform":
        return full & m
    if dist == "equal":
        return np.full(n, full[0] & m, np.uint64)
    if dist == "two":
        return np.where(rng.random(n) < 0.5, full[0], full[1 % n]) & m
    if dist == "skew":             # each 8-bit digit: 90 % of the keys share one value
        common = rng.integers(0, 256, 8)
        digits = np.where(rng.random((n, 8)) < 0.9, common, rng.integers(0, 256, (n, 8))).astype(np.uint64)
        return (digits << (np.arange(8, dtype=np.uint64) * np.uint64(8))).sum(1, dtype=np.uint64) & m
    if dist == "sorted":
        return np.sort(full & m)
    if dist == "reversed":
        return np.sort(full & m)[::-1].copy()
    if dist == "high":             # few distinct low parts, random bits at and above nbits
        low = rng.integers(0, min(1 << nbits, 5), n).astype(np.uint64)
        return low | (full & ~m) if nbits < 64 else low
    raise ValueError(dist)


def check_sort(native, keys, nbits):
    k, v = radix_sort(native, keys, nbits)
    want = np.argsort(keys & low_mask(nbits), kind="stable")
    assert np.array_equal(v, want.astype(np.uint32)), (int((v != want).sum()), int(np.argmax(v != want)))
    assert np.array_equal(k, keys[want])


SORT_SIZES = (1, 2, 31, 32, 33, RS_WARP_ITEMS - 1, RS_WARP_ITEMS, RS_WARP_ITEMS + 1, RS_TILE - 1, RS_TILE,
              RS_TILE + 1, 5 * RS_TILE + 317)
NBITS = (1, 7, 8, 9, 17, 20, 32, 33, 40, 63, 64)
DISTS = ("uniform", "equal", "two", "skew", "sorted", "reversed", "high")


@pytest.mark.parametrize("n", SORT_SIZES)
@pytest.mark.parametrize("dist,nbits", [("uniform", 64), ("skew", 20), ("high", 9)])
def test_radix_sort_sizes(native, n, dist, nbits):
    check_sort(native, make_keys(dist, n, nbits, n), nbits)


@pytest.mark.parametrize("nbits", NBITS)
@pytest.mark.parametrize("dist", DISTS)
def test_radix_sort_key_widths_and_distributions(native, nbits, dist):
    n = 3 * RS_TILE + 77
    check_sort(native, make_keys(dist, n, nbits, nbits), nbits)


def test_radix_sort_three_level_histogram_scan(native):
    """More than SCAN_TILE^2 / 256 tiles: the 256 x tiles digit histogram has more than SCAN_TILE^2 entries, so its scan
    recurses three levels.  67 M pairs: about 1.6 GB of device memory.  24 bits: three passes, the result in the half
    that did not hold the input."""
    n = (SCAN_TILE * SCAN_TILE // 256) * RS_TILE + 1
    assert 256 * -(-n // RS_TILE) > SCAN_TILE * SCAN_TILE
    rng = np.random.default_rng(11)
    keys = rng.integers(0, 1 << 24, n, dtype=np.uint64)
    keys[::7] = 12345                  # long runs of one key that only stability orders
    check_sort(native, keys, 24)


SCAN_SIZES = (1, 7, 8, 9, SCAN_TILE - 1, SCAN_TILE, SCAN_TILE + 1, SCAN_TILE ** 2 - 1, SCAN_TILE ** 2,
              SCAN_TILE ** 2 + 1, 3 * SCAN_TILE ** 2 + 5)


def scan_input(kind, n, seed):
    rng = np.random.default_rng(seed)
    if kind == "zeros":
        return np.zeros(n, np.uint32)
    if kind == "ones":
        return np.ones(n, np.uint32)
    if kind == "small":
        return rng.integers(0, 1000, n, dtype=np.uint32)
    return rng.integers(0, 2 ** 32, n, dtype=np.uint32)      # "wrap": totals far above 2^32


@pytest.mark.parametrize("n", SCAN_SIZES)
@pytest.mark.parametrize("kind", ["zeros", "ones", "small", "wrap"])
@pytest.mark.parametrize("in_place", [False, True])
def test_exclusive_scan(native, n, kind, in_place):
    x = scan_input(kind, n, n)
    want = np.zeros(n, np.uint64)
    np.cumsum(x[:-1], dtype=np.uint64, out=want[1:])
    want = (want & np.uint64(0xFFFFFFFF)).astype(np.uint32)
    got = scan(native, x, in_place)
    assert np.array_equal(got, want), (int((got != want).sum()), int(np.argmax(got != want)))
    if kind == "wrap" and n > 2:
        assert int(x.astype(np.uint64).sum()) >= 2 ** 32
