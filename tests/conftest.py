import sys
from pathlib import Path

import pytest

ROOT = Path(__file__).resolve().parent.parent
if str(ROOT) not in sys.path:
    sys.path.insert(0, str(ROOT))
if str(ROOT / "tests") not in sys.path:   # helper modules next to the tests (lowrank_cases.py)
    sys.path.insert(0, str(ROOT / "tests"))

import pio_b200  # noqa: E402,F401  (registers the package under an importable name)


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a real H100 (run with -m gpu on a machine that has one)")


@pytest.fixture(scope="session")
def oracle():
    from oracle import als_oracle
    als_oracle.build()
    return als_oracle


@pytest.fixture(scope="session")
def native():
    from pio_b200 import native as n
    import shutil
    if shutil.which("nvcc"):
        n.build()      # no-op when incubator-predictionio_b200/libpio_als.so is newer than its sources
    n.lib()            # raises if the library is missing: there is no CPU fallback
    return n
