import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a real H100 (run with -m gpu on the GPU box)")


def pytest_collection_modifyitems(config, items):
    """@pytest.mark.gpu tests are skipped (not failed) on a box without a CUDA device."""
    try:
        import torch
        have = torch.cuda.is_available()
    except Exception:
        have = False
    if have:
        return
    skip = pytest.mark.skip(reason="needs a CUDA device (H100)")
    for it in items:
        if "gpu" in it.keywords:
            it.add_marker(skip)


@pytest.fixture(scope="session")
def golden():
    import json
    with open(os.path.join(ROOT, "tests", "golden", "golden.json")) as f:
        return json.load(f)


@pytest.fixture(scope="session", autouse=True)
def _built():
    """Build the oracle (always) and the CUDA library (if missing; nvcc cross-compiles without a GPU)."""
    import __graft_entry__ as g
    g.build()
