import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (run with -m gpu on an H100)")


def _has_gpu() -> bool:
    try:
        import demodel_b200
        return demodel_b200.load().dm_device_count() > 0
    except Exception:
        return False


def pytest_collection_modifyitems(config, items):
    # `-m gpu` on a box without a GPU should fail loudly, not skip silently;
    # only auto-skip when the marker expression did not ask for gpu tests.
    expr = config.getoption("-m") or ""
    if "gpu" in expr and "not gpu" not in expr:
        return
    if _has_gpu():
        return
    skip = pytest.mark.skip(reason="no CUDA device")
    for item in items:
        if "gpu" in item.keywords:
            item.add_marker(skip)


@pytest.fixture(scope="session")
def oracle():
    from tests import _oracle
    return _oracle.load()


@pytest.fixture(scope="session")
def golden_dir():
    return os.path.join(ROOT, "tests", "golden")
