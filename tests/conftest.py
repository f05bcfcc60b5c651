import os
import subprocess
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (an H100: run with -m gpu)")


def pytest_sessionstart(session):
    """The CUDA library is built in-tree (git-ignored): build it when it is missing or stale so that a fresh
    checkout can run the suite (nvcc cross-compiles sm_90a without a GPU)."""
    import shutil

    if shutil.which("nvcc") or os.path.exists("/usr/local/cuda/bin/nvcc"):
        import __graft_entry__ as entry

        try:
            entry.build()
        except Exception as e:  # the ABI test then reports the missing library
            print(f"[conftest] build() failed: {e}")


@pytest.fixture(scope="session")
def hostsim():
    """g++ build of the device arithmetic header (tests/hostsim/hostsim.cpp) - test harness only."""
    import ctypes

    src = os.path.join(ROOT, "tests", "hostsim", "hostsim.cpp")
    out = os.path.join(ROOT, "tests", "hostsim", "_hostsim.so")
    hdr = os.path.join(ROOT, "tactics2d_b200", "csrc", "t2d_math.cuh")
    if not os.path.exists(out) or os.path.getmtime(out) < max(os.path.getmtime(src), os.path.getmtime(hdr)):
        subprocess.check_call(["g++", "-O2", "-std=c++17", "-ffp-contract=off", "-shared", "-fPIC", "-o", out, src])
    return ctypes.CDLL(out)


@pytest.fixture(scope="session")
def cuda_device():
    import torch

    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    return torch.device("cuda:0")
