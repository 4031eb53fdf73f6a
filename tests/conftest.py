"""pytest wiring: marker registration and import paths.

`-m "not gpu"` runs everywhere (oracle vs golden fixtures, host logic, C-ABI symbol checks, gloo
multi-process); `-m gpu` needs an H100 and is the parity suite proper (CUDA path through the C-ABI
vs oracle)."""
import os
import sys

import pytest

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PKG = os.path.join(REPO, "wave-u-net_b200")
for p in (REPO, PKG, os.path.join(REPO, "tests")):
    if p not in sys.path:
        sys.path.insert(0, p)


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (H100); run with -m gpu")


def pytest_collection_modifyitems(config, items):
    try:
        import torch
        has_gpu = torch.cuda.is_available()
    except Exception:  # pragma: no cover
        has_gpu = False
    if has_gpu:
        return
    skip = pytest.mark.skip(reason="no CUDA device")
    for item in items:
        if "gpu" in item.keywords:
            item.add_marker(skip)


@pytest.fixture(scope="session")
def golden_dir():
    return os.path.join(REPO, "tests", "golden")
