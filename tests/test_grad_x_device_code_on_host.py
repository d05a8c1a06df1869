"""The coordinate derivatives of tinygp_b200/csrc/kgrad.cuh (kgrad_eval<true>, used by the contraction epilogue of
b200gp_dense_log_probability_grad_x) compiled for the CPU with nvcc: every opcode, L1 and L2, through the normal form
and the interpreter, every metric kind (Linear, Cholesky, Subspace, nested, a full matrix), against central differences
of the device interpreter (kprog_eval) in each coordinate; exactly 0 and finite at coincident points; and the slot
derivatives bitwise equal to those of kgrad_eval<false>."""

import ctypes
import os
import shutil
import subprocess

import numpy as np
import pytest

from tinygp_b200 import kernels, transforms

HERE = os.path.dirname(os.path.abspath(__file__))
SRC = os.path.join(HERE, "csrc", "kgrad_x_hostcheck.cu")
OUT = os.path.join(HERE, "csrc", "_build", "libkgrad_x_hostcheck.so")
DEPS = [SRC] + [os.path.join(HERE, "..", "tinygp_b200", "csrc", f) for f in ("kgrad.cuh", "kprog.cuh", "common.cuh")] \
    + [os.path.join(HERE, "..", "include", "b200gp.h")]
P = ctypes.c_void_p


@pytest.fixture(scope="module")
def lib():
    nvcc = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    if not os.path.exists(nvcc):
        pytest.skip("nvcc not available")
    if not os.path.exists(OUT) or any(os.path.getmtime(d) > os.path.getmtime(OUT) for d in DEPS):
        os.makedirs(os.path.dirname(OUT), exist_ok=True)
        subprocess.run([nvcc, "-O2", "-std=c++17", "-Wno-deprecated-gpu-targets", "-diag-suppress", "20013",
                        "-Xcompiler", "-fPIC", "-shared", "-o", OUT, SRC], check=True)
    return ctypes.CDLL(OUT)


def _ptr(a):
    return P(a.ctypes.data)


def kgrad_x(lib, prog, X1, X2, mode):
    X1, X2 = np.ascontiguousarray(X1, dtype=np.float64), np.ascontiguousarray(X2, dtype=np.float64)
    npair, ndim = X1.shape
    k = np.empty(npair)
    gx = np.full((npair, lib.hostcheck_kgrad_max_dim()), np.nan)
    same = np.zeros(npair, dtype=np.int32)
    fast = ctypes.c_int()
    err = ctypes.create_string_buffer(256)
    rc = lib.hostcheck_kgrad_x(_ptr(prog), prog.shape[0], _ptr(X1), _ptr(X2), ctypes.c_int64(npair), ndim, mode, _ptr(k),
                               _ptr(gx), _ptr(same), ctypes.byref(fast), err)
    assert rc == 0, (rc, err.value)
    assert np.all(gx[:, ndim:] == 0.0)
    assert np.all(same == 1)                     # the slot derivatives do not depend on whether gx is asked for
    return k, gx[:, :ndim], bool(fast.value)


def keval(lib, prog, X1, X2):
    X1, X2 = np.ascontiguousarray(X1, dtype=np.float64), np.ascontiguousarray(X2, dtype=np.float64)
    k = np.empty(X1.shape[0])
    assert lib.hostcheck_keval_x(_ptr(prog), prog.shape[0], _ptr(X1), _ptr(X2), ctypes.c_int64(X1.shape[0]),
                                 X1.shape[1], _ptr(k)) == 0
    return k


def fd_x(lib, prog, X1, X2, h=1e-6):
    """central differences of kprog_eval by each coordinate of x1"""
    out = []
    for d in range(X1.shape[1]):
        up, dn = X1.copy(), X1.copy()
        up[:, d] += h
        dn[:, d] -= h
        out.append((keval(lib, prog, up, X2) - keval(lib, prog, dn, X2)) / (2 * h))
    return np.stack(out, axis=1)


def _pairs(ndim, seed=0, npair=12):
    rng = np.random.default_rng(seed)
    X1 = rng.uniform(-1, 1, (npair, ndim))
    X2 = rng.uniform(-1, 1, (npair, ndim))
    X2[:3] = X1[:3]                                  # coincident points
    return X1, X2


def _check(lib, prog, X1, X2, mode, fast_expected=None):
    val, gx, fast = kgrad_x(lib, prog, X1, X2, mode)
    if fast_expected is not None:
        assert fast == fast_expected
    np.testing.assert_allclose(val, keval(lib, prog, X1, X2), rtol=1e-14, atol=1e-15)
    assert np.all(np.isfinite(gx))
    assert np.all(gx[:3] == 0.0)                     # defined as 0 at coincident points
    np.testing.assert_allclose(gx[3:], fd_x(lib, prog, X1[3:], X2[3:]), rtol=1e-7, atol=1e-9)
    return gx


LEAVES = [
    ("exp", lambda d: kernels.Exp(1.3, distance=d)),
    ("expsq", lambda d: kernels.ExpSquared(0.8, distance=d)),
    ("m32", lambda d: kernels.Matern32(1.1, distance=d)),
    ("m52", lambda d: kernels.Matern52(0.9, distance=d)),
    ("cos", lambda d: kernels.Cosine(2.7, distance=d)),
    ("ess", lambda d: kernels.ExpSineSquared(1.9, distance=d, gamma=0.7)),
    ("rq", lambda d: kernels.RationalQuadratic(1.2, distance=d, alpha=1.6)),
]
DISTS = {"l1": kernels.L1Distance, "l2": kernels.L2Distance}


@pytest.mark.parametrize("leaf", [name for name, _ in LEAVES])
@pytest.mark.parametrize("dist", list(DISTS))
@pytest.mark.parametrize("mode", [0, 1])
def test_leaf_coordinate_derivatives(lib, leaf, dist, mode):
    k = 0.6 * dict(LEAVES)[leaf](DISTS[dist]()) + 0.3
    prog, _ = k.lower_for(np.zeros((1, 2)))
    X1, X2 = _pairs(2)
    _check(lib, prog, X1, X2, mode, fast_expected=(mode == 0))
    # the same leaf under a transform takes the metric path of the interpreter
    kt = 0.6 * transforms.Linear(np.array([0.7, 1.8]), dict(LEAVES)[leaf](DISTS[dist]()))
    prog_t, _ = kt.lower_for(np.zeros((1, 2)))
    _check(lib, prog_t, X1, X2, mode, fast_expected=False)


def test_fast_and_interpreter_agree(lib):
    k = 1.4 * kernels.ExpSquared(0.7) * kernels.Matern32(1.2) + 0.5 * (kernels.RationalQuadratic(1.0, alpha=0.9) + 0.2) \
        + kernels.Exp(0.9, distance=kernels.L2Distance())
    prog, _ = k.lower_for(np.zeros((1, 3)))
    X1, X2 = _pairs(3, 1)
    g0 = _check(lib, prog, X1, X2, 0, fast_expected=True)
    g1 = _check(lib, prog, X1, X2, 1, fast_expected=False)
    np.testing.assert_allclose(g0, g1, rtol=1e-12, atol=1e-15)


METRICS = {
    "linear_ard": (lambda: 1.2 * transforms.Linear(np.array([0.5, 1.5, 2.0]), kernels.ExpSquared()), 3),
    "linear_scalar_l1": (lambda: transforms.Linear(0.8, kernels.Matern32(1.1)), 3),
    "cholesky_l1": (lambda: transforms.Cholesky(np.array([0.7, 1.3, 0.9]), kernels.Matern52(1.1)), 3),
    "cholesky_matrix": (lambda: transforms.Cholesky(np.array([[1.1, 0.0, 0.0], [0.3, 0.9, 0.0], [-0.2, 0.4, 1.3]]),
                                                    kernels.Exp(1.0, distance=kernels.L2Distance())), 3),
    "linear_matrix_l1": (lambda: transforms.Linear(np.array([[0.5, 1.0, -0.3], [0.2, -0.7, 1.1]]),
                                                   kernels.RationalQuadratic(alpha=1.5)), 3),
    "subspace_axis": (lambda: transforms.Subspace(1, kernels.Matern32(0.6)), 3),
    "subspace_nested": (lambda: transforms.Subspace([0, 2], transforms.Linear(0.8, kernels.RationalQuadratic(alpha=1.5))), 3),
    "two_metrics_and_identity": (lambda: transforms.Linear(np.array([0.5, 1.5, 2.0]), kernels.Exp(1.0, distance=kernels.L2Distance()))
                                 * transforms.Subspace(1, kernels.Matern32(0.6)) + kernels.Cosine(4.0), 3),
    "eight_dims": (lambda: transforms.Linear(np.linspace(0.4, 1.8, 8), kernels.ExpSquared(1.5))
                   + kernels.Matern52(2.0, distance=kernels.L2Distance()), 8),
}


@pytest.mark.parametrize("case", list(METRICS))
def test_metric_coordinate_derivatives(lib, case):
    build, ndim = METRICS[case]
    prog, _ = build().lower_for(np.zeros((1, ndim)))
    X1, X2 = _pairs(ndim, 2)
    _check(lib, prog, X1, X2, 0, fast_expected=False)
