"""The derivative build of the Fisher information (kgrad_element in tinygp_b200/csrc/kgrad.cuh, run by grad.cu's
dk_build_kernel for every element of the np x np work buffer) compiled for the CPU with nvcc: every slot's dK / d slot,
mapped to the kernel's fields, against the complex-step derivatives of oracle/fisher_np.py; the noise slot's identity;
zeros in the padding."""

import ctypes
import os
import shutil
import subprocess

import numpy as np
import pytest

from oracle import fisher_np
from oracle import tinygp_np as o
from tinygp_b200 import kernels, transforms

HERE = os.path.dirname(os.path.abspath(__file__))
SRC = os.path.join(HERE, "csrc", "fisher_hostcheck.cu")
OUT = os.path.join(HERE, "csrc", "_build", "libfisher_hostcheck.so")
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


def build(lib, prog, x, np_, slot):
    D = np.full((np_, np_), np.nan)
    ns = ctypes.c_int()
    err = ctypes.create_string_buffer(256)
    rc = lib.hostcheck_dk_build(P(prog.ctypes.data), prog.shape[0], P(x.ctypes.data), ctypes.c_int64(x.shape[0]),
                                ctypes.c_int64(np_), x.shape[1], slot, P(D.ctypes.data), ctypes.byref(ns), err)
    assert rc == 0, (rc, err.value)
    return D, ns.value


CASES = {
    "sum_product": (lambda m: 1.3 * m.ExpSquared(0.9) * m.Matern32(1.7) + m.RationalQuadratic(1.1, alpha=0.7) + 0.2, 2),
    "periodic_l1": (lambda m: m.Cosine(2.5) + m.ExpSineSquared(1.7, gamma=0.6) * m.Exp(0.9, distance=m.L1Distance()), 1),
    "ard": (lambda m: 1.5 * m.Linear(np.array([0.5, 1.5, 2.0]), m.ExpSquared())
            + m.Subspace([0, 2], m.Cholesky(np.array([0.8, 1.1]), m.Matern52(1.2, distance=m.L2Distance()))), 3),
    "nested": (lambda m: m.Cholesky(0.9, m.Linear(np.array([1.4]), m.RationalQuadratic(1.0, alpha=2.0))), 1),
}


class _P:
    Exp, ExpSquared, Matern32, Matern52 = kernels.Exp, kernels.ExpSquared, kernels.Matern32, kernels.Matern52
    Cosine, ExpSineSquared, RationalQuadratic = kernels.Cosine, kernels.ExpSineSquared, kernels.RationalQuadratic
    L1Distance, L2Distance = kernels.L1Distance, kernels.L2Distance
    Linear, Cholesky, Subspace = transforms.Linear, transforms.Cholesky, transforms.Subspace


@pytest.mark.parametrize("name", list(CASES))
def test_derivative_build_matches_complex_step(lib, name):
    make, dim = CASES[name]
    rng = np.random.default_rng(4)
    n, np_ = 21, 24
    X = rng.uniform(0, 3, n) if dim == 1 else rng.uniform(0, 3, (n, dim))
    X[3] = X[7]                                          # coincident points
    k = make(_P)
    prog, x, leaves, owners = k.lower_for_grad(X)
    x = np.ascontiguousarray(x)
    # each slot as the fields it moves (the map of DirectSolver.fisher_information): leaf slots in program order, then
    # metric rows; a row scale lambda moves with d lambda / d s = 1 / s (Linear), -1 / f (Cholesky)
    slot_fields = [[(node, f, None, 1.0)] for node, f0, f1 in leaves for f in ((f0,) if f1 is None else (f0, f1))]
    for rows in owners:
        for chain in rows:
            ents = []
            for node, field, idx, how in chain:
                v = np.asarray(getattr(node, field), dtype=np.float64)
                s = float(v) if v.ndim == 0 else float(v[idx])
                ents.append((node, field, None if v.ndim == 0 else idx, 1.0 / s if how == "linear" else -1.0 / s))
            slot_fields.append(ents)
    labels, dKo = fisher_np.derivatives(make(o), X)
    ref = dict(zip(labels, dKo))
    from tinygp_b200.gp import _param_walk
    label_of = {key: label for label, key in _param_walk(k)}
    # dK / d field = sum over the slots that move the field of (d slot / d field) dK / d slot
    got = {}
    for s, ents in enumerate(slot_fields):
        D, ns = build(lib, prog, x, np_, s)
        assert ns == len(slot_fields)
        assert np.all(D[n:] == 0.0) and np.all(D[:, n:] == 0.0)
        for node, field, idx, coef in ents:
            lab = label_of[(id(node), field, idx)]
            got[lab] = got.get(lab, 0.0) + coef * D[:n, :n]
    assert sorted(got, key=str) == sorted(labels[:-1], key=str)
    for lab, d in got.items():
        np.testing.assert_allclose(d, ref[lab], rtol=1e-12, atol=1e-13 * max(1.0, np.max(np.abs(ref[lab]))), err_msg=str(lab))
    D, _ = build(lib, prog, x, np_, len(slot_fields))      # the noise slot
    np.testing.assert_array_equal(D, np.diag((np.arange(np_) < n).astype(float)))
