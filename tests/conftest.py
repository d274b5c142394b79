import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a real H100 (run with -m gpu on a GPU machine)")


def _has_gpu():
    try:
        import torch
        return torch.cuda.is_available()
    except Exception:
        return False


def pytest_collection_modifyitems(config, items):
    # `-m gpu` on a box without a GPU must fail loudly, not silently skip: only skip gpu tests when
    # they were not explicitly selected.
    if _has_gpu():
        return
    markexpr = config.getoption("-m") or ""
    if "gpu" in markexpr and "not gpu" not in markexpr:
        return
    skip = pytest.mark.skip(reason="no GPU in this container")
    for item in items:
        if "gpu" in item.keywords:
            item.add_marker(skip)


@pytest.fixture(scope="session")
def engine():
    from parsec_b200.engine import Engine
    e = Engine(0)
    yield e
    e.close()
