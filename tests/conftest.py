import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (run on an H100 with -m gpu)")


def pytest_collection_modifyitems(config, items):
    """A plain `pytest tests` on a CPU-only box skips the GPU parity tests instead of failing them (the product has no
    CPU fallback, so they cannot run there).  With `-m gpu` the tests are NOT skipped: on the GPU box a missing device must
    fail loudly."""
    if "gpu" in (config.getoption("-m") or ""):
        return
    try:
        import torch
        have = torch.cuda.is_available()
    except Exception:
        have = False
    if have:
        return
    skip = pytest.mark.skip(reason="no CUDA device: commpy_b200 has no CPU fallback")
    for item in items:
        if "gpu" in item.keywords:
            item.add_marker(skip)
