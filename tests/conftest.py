import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

GOLDEN = os.path.join(ROOT, "tests", "golden")


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (select with -m gpu)")


@pytest.fixture(scope="session")
def golden_dir():
    return GOLDEN


def pytest_collection_modifyitems(config, items):
    """`gpu`-marked tests are skipped (not failed) on a machine without a CUDA device or without the built library."""
    try:
        import torch
        from bonito_b200 import native
        ok = torch.cuda.is_available() and os.path.exists(native.lib_path())
    except Exception:
        ok = False
    if ok:
        return
    skip = pytest.mark.skip(reason="needs a CUDA device and bonito_b200/libbonito_b200.so")
    for item in items:
        if "gpu" in item.keywords:
            item.add_marker(skip)
