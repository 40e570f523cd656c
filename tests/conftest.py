import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (run with -m gpu on an H100)")
    # a fresh checkout has no built artefacts (*.so is git-ignored): build the product library and
    # the oracle once, exactly like __graft_entry__.build() (nvcc cross-compiles without a GPU)
    lib = os.path.join(ROOT, "staticmapping_b200", "libsm_b200.so")
    if not os.path.exists(lib):
        import subprocess
        env = dict(os.environ)
        env.pop("CXX", None); env.pop("CC", None)
        subprocess.check_call(["make", "-C", os.path.join(ROOT, "staticmapping_b200", "csrc"), "-j8", "-s"], env=env)


def _has_gpu():
    try:
        import torch
        return torch.cuda.is_available()
    except Exception:
        return False


def pytest_collection_modifyitems(config, items):
    if _has_gpu():
        return
    skip = pytest.mark.skip(reason="no CUDA device in this container")
    for item in items:
        if "gpu" in item.keywords:
            item.add_marker(skip)
