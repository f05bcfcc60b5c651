"""Every header under tactics2d_b200/csrc/ compiles on its own for sm_90a.

A kernel family's header must carry everything it reads (through t2d_world.cuh and the headers it includes), so that
t2d_kernels.cu may include the headers in any order and a new kernel can start from one header.  Each header is compiled
in a translation unit that holds only cuda_runtime.h, the C ABI header and the header itself."""

import glob
import os
import shutil
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "tactics2d_b200", "csrc")
ABI = os.path.join(ROOT, "include", "t2d_b200.h")
HEADERS = sorted(os.path.basename(h) for h in glob.glob(os.path.join(CSRC, "*.cuh")))


def _nvcc():
    nvcc = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
    return nvcc if os.path.exists(nvcc) else shutil.which("nvcc")


def test_headers_found():
    assert "t2d_world.cuh" in HEADERS and "t2d_tick.cuh" in HEADERS, HEADERS


@pytest.mark.parametrize("header", HEADERS)
def test_header_compiles_alone(header, tmp_path):
    nvcc = _nvcc()
    if nvcc is None:
        pytest.skip("nvcc not found")
    tu = tmp_path / "tu.cu"
    tu.write_text(f'#include <cuda_runtime.h>\n#include "{ABI}"\n#include "{os.path.join(CSRC, header)}"\n')
    r = subprocess.run([nvcc, "-gencode", "arch=compute_90a,code=sm_90a", "-std=c++17", "-c", str(tu), "-o",
                        str(tmp_path / "tu.o")], capture_output=True, text=True)
    assert r.returncode == 0, f"{header} does not compile alone:\n{r.stdout}{r.stderr}"
