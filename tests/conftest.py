import os
import sys

import pytest

ROOT = os.path.abspath(os.path.join(os.path.dirname(__file__), ".."))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

GOLDEN = os.path.join(ROOT, "tests", "golden")


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (an H100; run with `-m gpu`)")


def _cuda_device_count() -> int:
    try:
        import torch

        return torch.cuda.device_count() if torch.cuda.is_available() else 0
    except Exception:  # pylint: disable=broad-except
        return 0


def pytest_collection_modifyitems(config, items):
    """`gpu`-marked tests are skipped (not failed) on a machine without a CUDA device or without the built library."""
    lib = os.path.join(ROOT, "rectools_b200", "libb200rank.so")
    reason = None
    if not os.path.exists(lib):
        reason = "libb200rank.so is not built"
    elif _cuda_device_count() == 0:
        reason = "no CUDA device"
    if reason is None:
        return
    skip = pytest.mark.skip(reason=reason)
    for item in items:
        if "gpu" in item.keywords:
            item.add_marker(skip)


@pytest.fixture(scope="session")
def golden_dir():
    return GOLDEN


@pytest.fixture(scope="session")
def rb():
    import rectools_b200

    return rectools_b200
