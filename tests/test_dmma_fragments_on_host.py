"""The DMMA warp tile of the fp64 GEMM mainloops (tinygp_b200/csrc/dmma.cuh) compiled for the CPU with nvcc: one warp's
64 x 32 tile computed from the header's fragment loads, fragment coordinate maps and accumulator map, against NumPy.
Small-integer operands make every product and sum exact, so the comparison is exact."""

import ctypes
import os
import shutil
import subprocess

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
SRC = os.path.join(HERE, "csrc", "dmma_hostcheck.cu")
OUT = os.path.join(HERE, "csrc", "_build", "libdmma_hostcheck.so")
DEPS = [SRC, os.path.join(HERE, "..", "tinygp_b200", "csrc", "dmma.cuh")]
P = ctypes.c_void_p


@pytest.fixture(scope="module")
def lib():
    nvcc = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    if not os.path.exists(nvcc):
        pytest.skip("nvcc not available")
    if not os.path.exists(OUT) or any(os.path.getmtime(d) > os.path.getmtime(OUT) for d in DEPS):
        os.makedirs(os.path.dirname(OUT), exist_ok=True)
        subprocess.run([nvcc, "-O2", "-std=c++17", "-Wno-deprecated-gpu-targets", "-Xcompiler", "-fPIC", "-shared",
                        "-o", OUT, SRC], check=True)
    return ctypes.CDLL(OUT)


def warp_tile(lib, A, B):
    A, B = np.ascontiguousarray(A, dtype=np.float64), np.ascontiguousarray(B, dtype=np.float64)
    C = np.full((64, 32), np.nan)
    rc = lib.hostcheck_dmma_warp_tile(P(A.ctypes.data), P(B.ctypes.data), A.shape[1], P(C.ctypes.data))
    assert rc == 0, {1: "an atom element is not covered exactly once by the fragments",
                     2: "a fragment load read the row padding",
                     3: "the accumulator map does not write every C element once"}.get(rc, rc)
    return C


@pytest.mark.parametrize("K", [16, 128])
def test_warp_tile_matches_numpy(lib, K):
    rng = np.random.default_rng(K)
    A = rng.integers(-8, 9, (64, K)).astype(np.float64)
    B = rng.integers(-8, 9, (32, K)).astype(np.float64)
    np.testing.assert_array_equal(warp_tile(lib, A, B), A @ B.T)

