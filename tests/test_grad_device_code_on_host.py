"""The kernel-program derivatives of the dense gradient (tinygp_b200/csrc/kgrad.cuh) compiled for the CPU with nvcc:
every opcode at zero and non-zero distance, L1 and L2, through the normal form and the interpreter, and the metric
row-scale sensitivities, against central differences of the device interpreter (kprog_eval) and the oracle's closed
forms (oracle/grad_np.py)."""

import ctypes
import os
import shutil
import subprocess

import numpy as np
import pytest

from oracle import grad_np
from oracle import tinygp_np as o
from tinygp_b200 import kernels, transforms

HERE = os.path.dirname(os.path.abspath(__file__))
SRC = os.path.join(HERE, "csrc", "kgrad_hostcheck.cu")
OUT = os.path.join(HERE, "csrc", "_build", "libkgrad_hostcheck.so")
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


def kgrad(lib, prog, X1, X2, mode):
    X1, X2 = np.ascontiguousarray(X1, dtype=np.float64), np.ascontiguousarray(X2, dtype=np.float64)
    npair, ndim = X1.shape
    k = np.empty(npair)
    dk = np.zeros((npair, lib.hostcheck_kgrad_max_slots()))
    ns, fast = ctypes.c_int(), ctypes.c_int()
    err = ctypes.create_string_buffer(256)
    rc = lib.hostcheck_kgrad(_ptr(prog), prog.shape[0], _ptr(X1), _ptr(X2), ctypes.c_int64(npair), ndim, mode, _ptr(k),
                             _ptr(dk), ctypes.byref(ns), ctypes.byref(fast), err)
    assert rc == 0, (rc, err.value)
    return k, dk[:, :ns.value], bool(fast.value)


def keval(lib, prog, X1, X2):
    prog = np.ascontiguousarray(prog)
    X1, X2 = np.ascontiguousarray(X1, dtype=np.float64), np.ascontiguousarray(X2, dtype=np.float64)
    k = np.empty(X1.shape[0])
    assert lib.hostcheck_keval(_ptr(prog), prog.shape[0], _ptr(X1), _ptr(X2), ctypes.c_int64(X1.shape[0]), X1.shape[1],
                               _ptr(k)) == 0
    return k


def fd_slots(lib, prog, X1, X2):
    """central differences of kprog_eval by every slot: p0 / p1 of the instructions, then the metric rows"""
    rows, metric_rows = [], []
    r = 0
    while int(prog[r, 0]) == 32:
        mr, mc = int(prog[r, 2]), int(prog[r, 3])
        metric_rows.append((r + 1, mr, mc))
        r += 1 + -(-mr * mc // 4)
    for i in range(r, prog.shape[0]):
        op = int(prog[i, 0])
        if op in (16, 17):
            continue
        rows.append((i, 2))
        if op in (6, 7):
            rows.append((i, 3))
    out = []

    def central(mod, h):
        up, dn = prog.copy(), prog.copy()
        mod(up, 1 + h)
        mod(dn, 1 - h)
        return (keval(lib, up, X1, X2) - keval(lib, dn, X1, X2)) / (2 * h)

    for i, c in rows:
        v = prog[i, c]
        h = 1e-6 * max(abs(v), 1e-3)
        up, dn = prog.copy(), prog.copy()
        up[i, c] += h
        dn[i, c] -= h
        out.append((keval(lib, up, X1, X2) - keval(lib, dn, X1, X2)) / (2 * h))
    for start, mr, mc in metric_rows:
        for rr in range(mr):
            def mod(p, lam, start=start, rr=rr, mc=mc):
                flat = p[start:].reshape(-1)
                flat[rr * mc:(rr + 1) * mc] *= lam
                p[start:] = flat.reshape(p[start:].shape)
            out.append(central(mod, 1e-6))
    return np.stack(out, axis=1)


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


def _pairs(ndim, seed=0):
    rng = np.random.default_rng(seed)
    X1 = rng.uniform(-1, 1, (12, ndim))
    X2 = rng.uniform(-1, 1, (12, ndim))
    X2[:3] = X1[:3]                                  # r = 0
    return X1, X2


@pytest.mark.parametrize("leaf", [name for name, _ in LEAVES])
@pytest.mark.parametrize("dist", list(DISTS))
@pytest.mark.parametrize("mode", [0, 1])
def test_leaf_derivatives(lib, leaf, dist, mode):
    make = dict(LEAVES)[leaf]
    k = 0.6 * make(DISTS[dist]()) + 0.3
    prog, _ = k.lower_for(np.zeros((1, 2)))
    X1, X2 = _pairs(2)
    val, dk, fast = kgrad(lib, prog, X1, X2, mode)
    assert fast == (mode == 0)
    np.testing.assert_allclose(val, keval(lib, prog, X1, X2), rtol=1e-14, atol=1e-15)
    assert np.all(np.isfinite(dk))
    np.testing.assert_allclose(dk, fd_slots(lib, prog, X1, X2), rtol=1e-7, atol=1e-9)
    assert np.all(dk[:3, 1] == 0.0)                  # d k / d scale at r = 0
    # the oracle's closed form of d k / d scale (and gamma / alpha) for the same leaf
    onode = {"exp": lambda d: o.Exp(1.3, d), "expsq": lambda d: o.ExpSquared(0.8, d), "m32": lambda d: o.Matern32(1.1, d),
             "m52": lambda d: o.Matern52(0.9, d), "cos": lambda d: o.Cosine(2.7, d),
             "ess": lambda d: o.ExpSineSquared(1.9, d, gamma=0.7),
             "rq": lambda d: o.RationalQuadratic(1.2, d, alpha=1.6)}[leaf]({"l1": o.L1Distance, "l2": o.L2Distance}[dist]())
    for p in range(X1.shape[0]):
        acc = {}
        grad_np._walk(onode, (X1[p] - X2[p])[None, None, :], np.ones((1, 1)), acc, False)
        got = {f: float(v[1]) for (_, f), v in acc.items()}
        assert dk[p, 1] == pytest.approx(0.6 * got["scale"], rel=1e-12, abs=1e-15)
        if leaf in ("ess", "rq"):
            assert dk[p, 2] == pytest.approx(0.6 * got["gamma" if leaf == "ess" else "alpha"], rel=1e-12, abs=1e-15)


def test_fast_and_interpreter_agree(lib):
    k = 1.4 * kernels.ExpSquared(0.7) * kernels.Matern32(1.2) + 0.5 * (kernels.RationalQuadratic(1.0, alpha=0.9) + 0.2)
    prog, _ = k.lower_for(np.zeros((1, 3)))
    X1, X2 = _pairs(3, 1)
    v0, d0, f0 = kgrad(lib, prog, X1, X2, 0)
    v1, d1, f1 = kgrad(lib, prog, X1, X2, 1)
    assert f0 and not f1
    np.testing.assert_allclose(v0, v1, rtol=1e-14)
    np.testing.assert_allclose(d0, d1, rtol=1e-12, atol=1e-15)
    np.testing.assert_allclose(d0, fd_slots(lib, prog, X1, X2), rtol=1e-7, atol=1e-9)


@pytest.mark.parametrize("case", ["linear_ard", "cholesky_l1", "subspace_nested", "two_metrics"])
def test_metric_row_scales(lib, case):
    k = {
        "linear_ard": lambda: 1.2 * transforms.Linear(np.array([0.5, 1.5, 2.0]), kernels.ExpSquared()),
        "cholesky_l1": lambda: transforms.Cholesky(np.array([0.7, 1.3, 0.9]), kernels.Matern52(1.1)),
        "subspace_nested": lambda: transforms.Subspace([0, 2], transforms.Linear(0.8, kernels.RationalQuadratic(alpha=1.5))),
        "two_metrics": lambda: transforms.Linear(np.array([0.5, 1.5, 2.0]), kernels.Exp(1.0, distance=kernels.L2Distance()))
        * transforms.Subspace(1, kernels.Matern32(0.6)) + kernels.Cosine(4.0),
    }[case]()
    prog, _ = k.lower_for(np.zeros((1, 3)))
    X1, X2 = _pairs(3, 2)
    val, dk, fast = kgrad(lib, prog, X1, X2, 0)
    assert not fast                                   # input transforms always take the interpreter
    np.testing.assert_allclose(val, keval(lib, prog, X1, X2), rtol=1e-14)
    assert np.all(np.isfinite(dk))
    np.testing.assert_allclose(dk, fd_slots(lib, prog, X1, X2), rtol=1e-7, atol=1e-9)


def test_refused_programs(lib):
    k = kernels.quasisep.Celerite(1.1, 0.8, 0.9, 0.1)
    prog, _ = k.lower_for(np.zeros(1))
    X = np.zeros((1, 1))
    assert lib.hostcheck_kgrad(_ptr(prog), prog.shape[0], _ptr(X), _ptr(X), ctypes.c_int64(1), 1, 0, _ptr(np.empty(1)),
                               _ptr(np.empty(16)), ctypes.byref(ctypes.c_int()), ctypes.byref(ctypes.c_int()),
                               ctypes.create_string_buffer(256)) == 3
    big = sum(kernels.RationalQuadratic(1.0 + i, alpha=1.0) for i in range(9))   # 18 slots
    prog, _ = big.lower_for(np.zeros((1, 1)))
    assert lib.hostcheck_kgrad(_ptr(prog), prog.shape[0], _ptr(X), _ptr(X), ctypes.c_int64(1), 1, 0, _ptr(np.empty(1)),
                               _ptr(np.empty(16)), ctypes.byref(ctypes.c_int()), ctypes.byref(ctypes.c_int()),
                               ctypes.create_string_buffer(256)) == 3
