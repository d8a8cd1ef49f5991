import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

GOLDEN = os.path.join(ROOT, "tests", "golden")


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (H100); run with -m gpu")


@pytest.fixture(scope="session")
def golden_dir():
    return GOLDEN


def pytest_collection_modifyitems(config, items):
    """`gpu` tests are SKIPPED (not failed) on a host without a CUDA device or without the built library, so a
    plain `pytest` run on a CPU box reports real CPU-test regressions only."""
    try:
        import torch

        has_cuda = torch.cuda.is_available()
    except Exception:
        has_cuda = False
    has_lib = os.path.exists(os.path.join(ROOT, "kge_b200", "libb200kge.so"))
    if has_cuda and has_lib:
        return
    why = "no CUDA device" if not has_cuda else "libb200kge.so not built"
    skip = pytest.mark.skip(reason=f"gpu test: {why}")
    for item in items:
        if "gpu" in item.keywords:
            item.add_marker(skip)
