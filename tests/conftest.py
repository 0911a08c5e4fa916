import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for _p in (ROOT, os.path.join(ROOT, "tests")):
    if _p not in sys.path:
        sys.path.insert(0, _p)

GOLDEN = os.path.join(ROOT, "tests", "golden")


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs an sm_90 (H100) CUDA device (pytest -m gpu)")


def pytest_collection_modifyitems(config, items):
    """`gpu` tests need an sm_90 device: without one they are skipped (not failed), so a plain `pytest tests` works
    on a machine without a CUDA driver.  The product path itself still fails loudly without a GPU (test_host_logic)."""
    import torch

    ok = torch.cuda.is_available() and torch.cuda.get_device_capability(0) == (9, 0)
    if ok:
        return
    skip = pytest.mark.skip(reason="needs an sm_90 (H100) CUDA device")
    for item in items:
        if "gpu" in item.keywords:
            item.add_marker(skip)


@pytest.fixture(scope="session")
def golden_dir():
    return GOLDEN


@pytest.fixture(scope="session", autouse=True)
def _built():
    """Build the native library and the C part of the oracle once per session if they are missing."""
    import __graft_entry__ as ge

    if not (os.path.exists(os.path.join(ROOT, "yolort_b200", "libyolort_b200.so"))
            and os.path.exists(os.path.join(ROOT, "oracle", "libnms_ref.so"))):
        ge.build()
