"""The region lists that lay out the C ABI's scratch and staging blocks (ldso_b200/csrc/scratch_layout.cuh), checked on the CPU by
tests/cpp/scratch_layout_probe.cu over a grid of image sizes, point counts, window sizes and feature capacities: every region inside
the block its list sized, pairwise disjoint, aligned for its type; the groups one copy or one memset covers contiguous; the regions a
context sets once at offsets that do not depend on a call's parameters. No GPU needed: the probe is compiled with nvcc for its argument
structs, and no CUDA call runs."""
import ctypes as C
import hashlib
import os
import shutil
import subprocess
import tempfile

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "ldso_b200", "csrc")
PROBE = os.path.join(ROOT, "tests", "cpp", "scratch_layout_probe.cu")
NVCC = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")


@pytest.fixture(scope="module")
def probe():
    if not os.path.exists(NVCC) and shutil.which("nvcc") is None:
        pytest.skip("nvcc not found")
    srcs = [PROBE, os.path.join(ROOT, "include", "ldso_b200.h")] + sorted(
        os.path.join(CSRC, f) for f in os.listdir(CSRC) if f.endswith((".cuh", ".h")))
    key = hashlib.sha1(b"".join(open(f, "rb").read() for f in srcs)).hexdigest()[:16]
    out = os.path.join(tempfile.gettempdir(), f"ldso_b200_scratch_layout_probe_{os.getuid()}_{key}.so")
    if not os.path.exists(out):
        tmp = out + f".{os.getpid()}"
        nvcc = NVCC if os.path.exists(NVCC) else "nvcc"
        # PTX only: the kernels the argument structs come with are never run here
        subprocess.check_call([nvcc, "-gencode", "arch=compute_90a,code=compute_90a", "-std=c++17", "-O1", "-Xcompiler", "-fPIC", "-shared",
                               "-diag-suppress", "550", PROBE, "-o", tmp])
        os.replace(tmp, out)
    L = C.CDLL(out)
    L.scratch_layout_check.restype = C.c_longlong
    L.scratch_layout_check.argtypes = [C.c_char_p, C.c_char_p, C.c_int]
    return L


@pytest.mark.parametrize("block", ["corners", "pixsel", "actsel", "immature_store", "one_shot", "posegraph"])
def test_region_lists(probe, block):
    err = C.create_string_buffer(512)
    n = probe.scratch_layout_check(block.encode(), err, len(err))
    assert n > 0, err.value.decode()
