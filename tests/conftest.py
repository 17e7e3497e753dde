import os
import subprocess
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (an H100)")
    config.addinivalue_line("markers", "shipping: run with the default (benchmarked) precision switches")


def pytest_collection_modifyitems(config, items):
    """`gpu`-marked tests need a CUDA device and the built library: skip (not fail) them where either is missing."""
    try:
        import torch
        have = torch.cuda.is_available()
    except Exception:
        have = False
    lib = os.path.join(ROOT, "propainter_b200", "libpropainter_b200.so")
    if have and os.path.exists(lib):
        return
    why = "no CUDA device" if not have else "libpropainter_b200.so not built"
    skip = pytest.mark.skip(reason=f"gpu test: {why}")
    for it in items:
        if "gpu" in it.keywords:
            it.add_marker(skip)


@pytest.fixture(scope="session")
def hostsim():
    """ctypes handle to the host build of pp_elem.cuh (test harness, see tests/hostsim/hostsim.cpp)."""
    import ctypes
    src = os.path.join(ROOT, "tests", "hostsim", "hostsim.cpp")
    lib = os.path.join(ROOT, "tests", "hostsim", "libhostsim.so")
    deps = [src, os.path.join(ROOT, "propainter_b200", "csrc", "pp_elem.cuh"),
            os.path.join(ROOT, "propainter_b200", "csrc", "pp_common.cuh")]
    if not os.path.exists(lib) or any(os.path.getmtime(d) > os.path.getmtime(lib) for d in deps):
        subprocess.check_call(["g++", "-O2", "-ffp-contract=off", "-shared", "-fPIC", "-o", lib, src])
    return ctypes.CDLL(lib)
