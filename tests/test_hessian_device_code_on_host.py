"""The second derivatives of a kernel program (khess_eval in tinygp_b200/csrc/kgrad.cuh, what grad.cu's
hess_contract_kernel runs for every element of a W tile) compiled for the CPU with nvcc: against central differences of
kgrad_eval (normal form and interpreter) over every opcode, L1 and L2, zero and non-zero distance and metric row scales,
and against oracle/hessian_np.py's contraction."""

import ctypes
import os

import numpy as np
import pytest

from oracle import fisher_np, hessian_np
from oracle import tinygp_np as o
from tinygp_b200 import kernels, transforms
from util import host_library

HERE = os.path.dirname(os.path.abspath(__file__))
SRC = os.path.join(HERE, "csrc", "khess_hostcheck.cu")
OUT = os.path.join(HERE, "csrc", "_build", "libkhess_hostcheck.so")
DEPS = [SRC] + [os.path.join(HERE, "..", "tinygp_b200", "csrc", f) for f in ("kgrad.cuh", "kprog.cuh", "common.cuh")] \
    + [os.path.join(HERE, "..", "include", "b200gp.h")]
P = ctypes.c_void_p
MAXS = 16


@pytest.fixture(scope="module")
def lib():
    return host_library(SRC, OUT, DEPS, ["-diag-suppress", "20013"])


def khess(lib, prog, X1, X2, pairs):
    ne, nd = X1.shape
    pa = np.array([a for a, _ in pairs], dtype=np.int32)
    pb = np.array([b for _, b in pairs], dtype=np.int32)
    h = np.full((ne, len(pairs)), np.nan)
    ns = ctypes.c_int()
    err = ctypes.create_string_buffer(256)
    rc = lib.hostcheck_khess(P(prog.ctypes.data), prog.shape[0], P(X1.ctypes.data), P(X2.ctypes.data),
                             ctypes.c_int64(ne), nd, P(pa.ctypes.data), P(pb.ctypes.data), len(pairs),
                             P(h.ctypes.data), ctypes.byref(ns), err)
    assert rc == 0, (rc, err.value)
    return h, ns.value


def kgrad(lib, prog, X1, X2, mode):
    dk = np.zeros((X1.shape[0], MAXS))
    rc = lib.hostcheck_kgrad1(P(prog.ctypes.data), prog.shape[0], P(X1.ctypes.data), P(X2.ctypes.data),
                              ctypes.c_int64(X1.shape[0]), X1.shape[1], mode, P(dk.ctypes.data))
    assert rc == 0
    return dk


def _slot_places(prog, nslot):
    """for each slot, ("p", row, col) or ("m", header row, rows, cols, r), in kgrad_prepare's order"""
    places, metrics, row = [], [], 0
    while row < prog.shape[0] and int(prog[row, 0]) == 32 and int(prog[row, 1]) == len(metrics) + 1:
        mr, mc = int(prog[row, 2]), int(prog[row, 3])
        metrics.append((row, mr, mc))
        row += 1 + -(-mr * mc // 4)
    for i in range(row, prog.shape[0]):
        op = int(prog[i, 0])
        if op in (16, 17):
            continue
        places.append(("p", i, 2))
        if op in (6, 7):
            places.append(("p", i, 3))
    for st, mr, mc in metrics:
        places += [("m", st, mr, mc, r) for r in range(mr)]
    assert len(places) == nslot
    return places


def _moved(prog, place, h):
    p = prog.copy()
    if place[0] == "p":
        p[place[1], place[2]] += h
    else:
        _, st, mr, mc, r = place
        nd = -(-mr * mc // 4)
        flat = p[st + 1:st + 1 + nd].reshape(-1)
        flat[r * mc:(r + 1) * mc] *= 1.0 + h
        p[st + 1:st + 1 + nd] = flat.reshape(-1, 4)
    return p


class _P:
    Exp, ExpSquared, Matern32, Matern52 = kernels.Exp, kernels.ExpSquared, kernels.Matern32, kernels.Matern52
    Cosine, ExpSineSquared, RationalQuadratic = kernels.Cosine, kernels.ExpSineSquared, kernels.RationalQuadratic
    L1Distance, L2Distance = kernels.L1Distance, kernels.L2Distance
    Linear, Cholesky, Subspace = transforms.Linear, transforms.Cholesky, transforms.Subspace


CASES = {   # (kernel, input dimensions); the first three have a normal form, the others run the interpreter only
    "l1_all_leaves": (lambda m: 1.3 * m.ExpSquared(0.9, distance=m.L1Distance()) * m.Matern32(1.7, distance=m.L1Distance())
                      + m.RationalQuadratic(1.1, distance=m.L1Distance(), alpha=0.7) + 0.2, 2),
    "l2_all_leaves": (lambda m: m.Exp(1.1, distance=m.L2Distance()) * m.Matern52(1.4, distance=m.L2Distance())
                      + m.ExpSquared(0.8) * m.RationalQuadratic(1.2, distance=m.L2Distance(), alpha=1.6), 2),
    "periodic": (lambda m: m.Cosine(2.5) * 0.7 + m.ExpSineSquared(1.7, gamma=0.6) * m.Exp(0.9), 1),
    "ard_l2": (lambda m: 1.5 * m.Linear(np.array([0.5, 1.5, 2.0]), m.ExpSquared())
               + m.Subspace([0, 2], m.Cholesky(np.array([0.8, 1.1]), m.Matern52(1.2, distance=m.L2Distance()))), 3),
    "ard_l1": (lambda m: m.Linear(np.array([0.7, 1.2]), m.Exp(1.3, distance=m.L1Distance()))
               * m.Linear(np.array([1.1, 0.6]), m.RationalQuadratic(0.9, distance=m.L1Distance(), alpha=1.4)), 2),
    "ard_periodic": (lambda m: m.Linear(np.array([0.9, 1.3]), m.ExpSineSquared(2.0, distance=m.L2Distance(), gamma=0.5))
                     + m.Linear(np.array([1.2, 0.4]), m.Matern32(1.5, distance=m.L2Distance()) * m.Cosine(3.0, distance=m.L2Distance())), 2),
}


def _points(dim, ne=40, seed=6):
    rng = np.random.default_rng(seed)
    X1 = rng.uniform(0, 2, (ne, dim))
    X2 = rng.uniform(0, 2, (ne, dim))
    X2[:4] = X1[:4]                                       # zero distance
    return np.ascontiguousarray(X1), np.ascontiguousarray(X2)


@pytest.mark.parametrize("mode", [0, 1])
@pytest.mark.parametrize("name", list(CASES))
def test_against_central_differences_of_kgrad(lib, name, mode):
    make, dim = CASES[name]
    X1, X2 = _points(dim)
    prog, _, _, _ = make(_P).lower_for_grad(X1)
    prog = np.ascontiguousarray(prog)
    _, ns = khess(lib, prog, X1, X2, [(0, 0)])
    places = _slot_places(prog, ns)
    pairs = [(a, b) for a in range(ns) for b in range(a, ns)]
    got = np.concatenate([khess(lib, prog, X1, X2, pairs[i:i + 16])[0] for i in range(0, len(pairs), 16)], axis=1)
    dk0 = kgrad(lib, prog, X1, X2, mode)
    for b in range(ns):
        h = 1e-6 * (max(abs(prog[places[b][1], places[b][2]]), 1e-2) if places[b][0] == "p" else 1.0)
        d = (kgrad(lib, _moved(prog, places[b], h), X1, X2, mode) - kgrad(lib, _moved(prog, places[b], -h), X1, X2, mode)) / (2 * h)
        for a in range(ns):
            col = pairs.index((min(a, b), max(a, b)))
            ref = d[:, a].copy()
            if a == b and places[a][0] == "m":
                ref -= dk0[:, a]             # kgrad's row sensitivity is lambda dk / dlambda: d / dlambda adds dk / dlambda
            np.testing.assert_allclose(got[:, col], ref, rtol=1e-6, atol=1e-7 * max(1.0, np.max(np.abs(ref))),
                                       err_msg=f"{name} slots {a}, {b}")


@pytest.mark.parametrize("name", ["l1_all_leaves", "l2_all_leaves", "periodic"])
def test_contraction_against_oracle(lib, name):
    """without transforms every slot is a field: sum_ij A_ij d2k(x_i, x_j) / da db / 2 against hessian_np.second_term"""
    make, dim = CASES[name]
    rng = np.random.default_rng(8)
    n = 14
    X = rng.uniform(0, 2, (n, dim))
    X[5] = X[2]
    A = rng.normal(size=(n, n))
    A = A + A.T
    k = make(_P)
    prog, x, leaves, _ = k.lower_for_grad(X)
    prog = np.ascontiguousarray(prog)
    I, J = np.meshgrid(np.arange(n), np.arange(n), indexing="ij")
    X1, X2 = np.ascontiguousarray(X[I.ravel()]), np.ascontiguousarray(X[J.ravel()])
    _, ns = khess(lib, prog, X1, X2, [(0, 0)])
    pairs = [(a, b) for a in range(ns) for b in range(a, ns)]
    got = np.concatenate([khess(lib, prog, X1, X2, pairs[i:i + 16])[0] for i in range(0, len(pairs), 16)], axis=1)
    from tinygp_b200.gp import _param_walk
    label_of = {key: label for label, key in _param_walk(k)}
    slot_label = [label_of[(id(node), f, None)] for node, f0, f1 in leaves for f in ((f0,) if f1 is None else (f0, f1))]
    labels, So = hessian_np.second_term(make(o), X, A)
    idx = {lab: i for i, lab in enumerate(labels)}
    for col, (a, b) in enumerate(pairs):
        val = 0.5 * np.sum(A.ravel() * got[:, col])
        ref = So[idx[slot_label[a]], idx[slot_label[b]]]
        assert val == pytest.approx(ref, rel=1e-10, abs=1e-11 * np.max(np.abs(So))), (name, a, b)
