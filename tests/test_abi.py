"""CPU tests of the drop-in boundary: the C-ABI library loads, exports every symbol that
include/pio_als.h declares, and fails loudly (no CPU fallback) when no H100 is visible."""
import re
from pathlib import Path

import pytest

ROOT = Path(__file__).resolve().parent.parent


def test_library_exports_every_declared_symbol(native):
    header = (ROOT / "include" / "pio_als.h").read_text()
    declared = sorted(set(re.findall(r"PIO_API\s+[\w\s\*]+?\b(pio_\w+)\s*\(", header)))
    assert declared, "no PIO_API declarations parsed"
    L = native.lib()
    for name in declared:
        assert hasattr(L, name), f"{name} declared in pio_als.h but not exported"
    assert sorted(native.EXPORTED_SYMBOLS) == declared
    assert L.pio_als_abi_version() == native.ABI_VERSION


def test_no_cpu_fallback_without_gpu(native):
    if native.device_count() > 0:
        pytest.skip("an H100 is visible; the no-GPU failure path cannot be exercised")
    with pytest.raises(native.NativeError) as ei:
        native.NativeALS(rank=10, n_users=10, n_items=10)
    assert ei.value.code == native.ERR_CUDA
    assert "no CPU fallback" in str(ei.value)


def test_argument_validation_precedes_device_work(native):
    for kw in (dict(rank=0), dict(rank=129), dict(n_users=0), dict(world_size=2, world_rank=2)):
        args = dict(rank=8, n_users=4, n_items=4)
        args.update(kw)
        with pytest.raises(native.NativeError) as ei:
            native.NativeALS(**args)
        assert ei.value.code == native.ERR_ARG
