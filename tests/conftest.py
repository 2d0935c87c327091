import os
import subprocess
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "tests")):
    if p not in sys.path:
        sys.path.insert(0, p)


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (an H100)")
    # the oracle is plain C and builds in a second; make sure the checker exists
    if not os.path.exists(os.path.join(ROOT, "oracle", "libcpbus_oracle.so")):
        subprocess.check_call(["make", "-s", "-C", os.path.join(ROOT, "oracle")])


def _has_gpu():
    try:
        import torch
        return torch.cuda.is_available()
    except Exception:
        return False


def pytest_collection_modifyitems(config, items):
    if _has_gpu():
        return
    skip = pytest.mark.skip(reason="no CUDA device here")
    for item in items:
        if "gpu" in item.keywords:
            item.add_marker(skip)
