import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


# SPH_EMU_LIB=<path of tests/emu/_build/libsph_b200_emu*.so>: run the `gpu` tests against the host-emulated
# build of the SAME sources (tests/emu/; used by tests/test_kernel_emulation.py in a subprocess).
if os.environ.get("SPH_EMU_LIB"):
    sys.path.insert(0, os.path.join(ROOT, "tests", "emu"))
    import emu_engine
    emu_engine.install(os.environ["SPH_EMU_LIB"])


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (an H100)")


def _has_cuda():
    try:
        import torch
        return torch.cuda.is_available()
    except Exception:
        return False


def pytest_collection_modifyitems(config, items):
    if _has_cuda():
        return
    skip = pytest.mark.skip(reason="no CUDA device")
    for item in items:
        if "gpu" in item.keywords:
            item.add_marker(skip)
