import os
import sys
from pathlib import Path

import pytest

ROOT = Path(__file__).resolve().parents[1]
if str(ROOT) not in sys.path:
    sys.path.insert(0, str(ROOT))


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (an H100; run with -m gpu)")


def _has_gpu() -> bool:
    try:
        from wax_b200 import CUDAVectorEngine
        return CUDAVectorEngine.is_available()
    except Exception:
        return False


def pytest_collection_modifyitems(config, items):
    # `-m gpu` on a box without a GPU must fail loudly rather than silently skip: only auto-skip when the
    # user did not ask for GPU tests explicitly.
    if "gpu" in (config.getoption("-m") or ""):
        return
    if _has_gpu():
        return
    skip = pytest.mark.skip(reason="no CUDA device")
    for item in items:
        if "gpu" in item.keywords:
            item.add_marker(skip)


@pytest.fixture(scope="session")
def oracle():
    from oracle import oracle as o
    o.build()
    return o
