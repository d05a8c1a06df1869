"""Expected Fisher information of the oracle GP's log-likelihood with NumPy / LAPACK (TEST ORACLE).

    F_ab = 1/2 tr(W dK/da W dK/db),   W = K^-1 (LAPACK dpotrf then dpotri).

dK/da comes from complex-step differentiation of the oracle's kernel matrix (oracle/tinygp_np.py): the parameter is
moved to p + i h and dK/da = Im K / h, exact to rounding and independent of the closed forms of grad_np.py and of the
CUDA code.  The kernel is evaluated on the pairwise differences D as grad_np does (a 0- / 1-D Linear or Cholesky maps the
differences as it maps the points); an L1 distance takes |z| as z sign(Re z), the analytic continuation of |.| that the
complex step needs.

Parameters are labelled as GaussianProcess.fisher_information labels them: (path, None) for a scalar field, (path, i)
for entry i of a 1-D field, depth-first over vars(node), a shared node once; ("diag", None) last for a scalar diag.
"""

from __future__ import annotations

import copy

import numpy as np
import scipy.linalg as sla
from scipy.linalg import lapack

from oracle import tinygp_np as o

H = 1e-30


def _fields(node):
    if isinstance(node, o.Constant):
        return ("value",)
    if isinstance(node, o.ExpSineSquared):
        return ("scale", "gamma")
    if isinstance(node, o.RationalQuadratic):
        return ("scale", "alpha")
    if isinstance(node, o.Stationary):
        return ("scale",)
    if isinstance(node, o.Linear):
        return ("scale",)
    if isinstance(node, o.Cholesky):
        return ("factor",)
    return ()


def params(kernel, path="", memo=None):
    """[(label, node, field, index)] of every differentiable scalar of the kernel"""
    memo = set() if memo is None else memo
    if id(kernel) in memo:
        return []
    memo.add(id(kernel))
    out = []
    fields = _fields(kernel)
    for name, value in vars(kernel).items():
        if isinstance(value, o.Kernel):
            out += params(value, path + name + ".", memo)
        elif name in fields:
            if np.ndim(value) == 0:
                out.append(((path + name, None), kernel, name, None))
            else:
                out += [((path + name, i), kernel, name, i) for i in range(np.size(value))]
    return out


class _AbsL1(o.L1Distance):
    def distance(self, d):
        return np.sum(d * np.sign(d.real), axis=-1)


def _value(node, D):
    if isinstance(node, o.Sum):
        return _value(node.kernel1, D) + _value(node.kernel2, D)
    if isinstance(node, o.Product):
        return _value(node.kernel1, D) * _value(node.kernel2, D)
    if isinstance(node, o.Constant):
        return np.full(D.shape[:-1], node.value, dtype=np.result_type(node.value, D))
    if isinstance(node, o.Subspace):
        return _value(node.kernel, D[..., [node.axis]] if np.ndim(node.axis) == 0 else D[..., list(node.axis)])
    if isinstance(node, (o.Linear, o.Cholesky)):
        p = node.scale if isinstance(node, o.Linear) else node.factor
        if np.ndim(p) >= 2:
            raise TypeError("matrix-valued transforms have no oracle Fisher information")
        return _value(node.kernel, p * D if isinstance(node, o.Linear) else D / p)
    if isinstance(node, o.Stationary) and isinstance(node.distance, o.L1Distance):
        node = copy.copy(node)
        node.distance = _AbsL1()
    return node.evaluate_diff(D)


def _diffs(X):
    X = np.asarray(X, dtype=np.float64)
    X2 = X[:, None] if X.ndim == 1 else X
    return X2[:, None, :] - X2[None, :, :]


def kernel_matrix(kernel, X):
    return np.real(_value(kernel, _diffs(X)))


def derivatives(kernel, X, scalar_diag=True):
    """(labels, [dK/da]) by complex step; the scalar diag's dK/d diag = I last"""
    D = _diffs(X)
    labels, dK = [], []
    for label, node, field, idx in params(kernel):
        old = getattr(node, field)
        new = np.array(old, dtype=np.complex128)
        if idx is None:
            new = new + 1j * H
        else:
            new[idx] += 1j * H
        setattr(node, field, new if np.ndim(old) else complex(new))
        try:
            dK.append(np.imag(_value(kernel, D)) / H)
        finally:
            setattr(node, field, old)
        labels.append(label)
    if scalar_diag:
        labels.append(("diag", None))
        dK.append(np.eye(D.shape[0]))
    return labels, dK


def inverse(kernel, X, diag):
    """W = K^-1 by dpotrf / dpotri, or None if K is not positive definite"""
    K = kernel_matrix(kernel, X) + np.diag(np.broadcast_to(np.asarray(diag, dtype=np.float64), (_diffs(X).shape[0],)))
    c, info = lapack.dpotrf(K, lower=1, clean=1)
    if info != 0:
        return None
    Wl, _ = lapack.dpotri(c, lower=1)
    return np.tril(Wl) + np.tril(Wl, -1).T


def fisher(kernel, X, diag, scalar_diag=None):
    """(labels, F) of GaussianProcess(kernel, X, diag=diag).fisher_information(); all-NaN F for a non-PD K"""
    scalar_diag = np.ndim(diag) == 0 if scalar_diag is None else scalar_diag
    labels, dK = derivatives(kernel, X, scalar_diag)
    W = inverse(kernel, X, diag)
    if W is None:
        return labels, np.full((len(labels), len(labels)), np.nan)
    A = [W @ d for d in dK]
    F = np.array([[0.5 * np.sum(a * b.T) for b in A] for a in A])
    return labels, 0.5 * (F + F.T)


def score_samples(kernel, X, diag, ndraw, rng):
    """d logp / d theta (labels order, diag last for a scalar diag) for ndraw draws y ~ N(0, K): shape (ndraw, P)"""
    labels, dK = derivatives(kernel, X, np.ndim(diag) == 0)
    W = inverse(kernel, X, diag)
    L = sla.cholesky(np.linalg.inv(W), lower=True)
    alpha = W @ (L @ rng.standard_normal((L.shape[0], ndraw)))
    return labels, np.stack([0.5 * (np.sum(alpha * (d @ alpha), axis=0) - np.sum(W * d)) for d in dK], axis=1)
