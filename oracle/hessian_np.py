"""Hessian of the oracle GP's log-likelihood with respect to the kernel parameters and a scalar noise diagonal, with
NumPy / LAPACK (TEST ORACLE).  With W = K^-1 (LAPACK dpotrf then dpotri), alpha = W r, K_a = dK/da, K_ab = d2K/dadb:

    H_ab = 1/2 <alpha alpha^T - W, K_ab>  -  (K_a alpha)^T W (K_b alpha)  +  1/2 tr(W K_a W K_b)

For the scalar diag sigma, K_sigma = I and K_sigma,sigma = K_a,sigma = 0.

- K_a: complex step of the oracle kernel matrix (fisher_np.derivatives);
- the second-derivative term: complex step, parameter by parameter, of grad_np's closed-form contraction
  sum_ij (A_ij / 2) dK_ij / da with A = alpha alpha^T - W held fixed.  The L1 distance is continued analytically as
  z sign(Re z) (and its derivative as sign(Re z)), and the kernel values that weight the factors of a Product come from
  fisher_np's complex-safe evaluation, so that the step goes through transforms and products.

Parameters are labelled and ordered as GaussianProcess.fisher_information labels them (fisher_np.params).
"""

from __future__ import annotations

import contextlib

import numpy as np
import scipy.linalg as sla
from scipy.linalg import lapack

from oracle import fisher_np
from oracle import grad_np

H = 1e-30


class _AnalyticNumpy:
    """numpy with abs / sign continued analytically off the real axis (|z| -> z sign(Re z), sign(z) -> sign(Re z)),
    and complex zeros, so that adjoints accumulate the imaginary part"""

    def __getattr__(self, name):
        return getattr(np, name)

    @staticmethod
    def abs(z):
        return z * np.sign(np.real(z)) if np.iscomplexobj(z) else np.abs(z)

    @staticmethod
    def zeros(shape):
        return np.zeros(shape, dtype=np.complex128)

    @staticmethod
    def sign(z):
        return np.sign(np.real(z))


@contextlib.contextmanager
def _analytic_grad_np():
    """grad_np on complex parameters: its numpy continued analytically, and its kernel values (the weights a Product
    passes to each factor) from fisher_np's complex-safe evaluation"""
    saved = grad_np.np, grad_np._value
    grad_np.np, grad_np._value = _AnalyticNumpy(), fisher_np._value
    try:
        yield
    finally:
        grad_np.np, grad_np._value = saved


def _key_value(acc, node, field, idx):
    v = acc.get((id(node), field), [None, 0.0])[1]
    return v if idx is None else np.asarray(v)[idx]


def second_term(kernel, X, A):
    """(labels, S) with S_ab = 1/2 sum_ij A_ij d2K_ij / da db over the kernel's parameters (no diag)"""
    X = np.asarray(X, dtype=np.float64)
    D = fisher_np._diffs(X)
    plist = fisher_np.params(kernel)
    S = np.zeros((len(plist), len(plist)))
    with _analytic_grad_np():
        for b, (_, node, field, idx) in enumerate(plist):
            old = getattr(node, field)
            new = np.array(old, dtype=np.complex128)
            if idx is None:
                new = new + 1j * H
            else:
                new[idx] += 1j * H
            setattr(node, field, new if np.ndim(old) else np.complex128(new))
            try:
                acc: dict = {}
                grad_np._walk(kernel, D.astype(np.complex128), 0.5 * A, acc, False)
            finally:
                setattr(node, field, old)
            for a, (_, na, fa, ia) in enumerate(plist):
                S[a, b] = np.imag(_key_value(acc, na, fa, ia)) / H
    return [p[0] for p in plist], 0.5 * (S + S.T)


def hessian(kernel, X, y, diag, mean=0.0, scalar_diag=None, terms=False):
    """(labels, H) of GaussianProcess(kernel, X, diag=diag, mean=mean).log_probability_hessian(y); all-NaN H for a non-PD
    K.  terms: (labels, H, (S, G, F)) with the second-derivative term S, the alpha term G = (K_a alpha)^T W (K_b alpha)
    and F, H = S - G + F."""
    scalar_diag = np.ndim(diag) == 0 if scalar_diag is None else scalar_diag
    labels, dK = fisher_np.derivatives(kernel, X, scalar_diag)
    W = fisher_np.inverse(kernel, X, diag)
    if W is None:
        nan = np.full((len(labels), len(labels)), np.nan)
        return (labels, nan, (nan, nan, nan)) if terms else (labels, nan)
    r = np.asarray(y, dtype=np.float64) - mean
    alpha = W @ r
    A = np.outer(alpha, alpha) - W
    _, S0 = second_term(kernel, X, A)
    S = np.zeros((len(labels), len(labels)))
    S[:S0.shape[0], :S0.shape[1]] = S0
    V = np.stack([d @ alpha for d in dK], axis=1)
    G = V.T @ W @ V
    G = 0.5 * (G + G.T)
    WK = [W @ d for d in dK]
    F = np.array([[0.5 * np.sum(a * b.T) for b in WK] for a in WK])
    F = 0.5 * (F + F.T)
    Hm = S - G + F
    return (labels, Hm, (S, G, F)) if terms else (labels, Hm)


def log_probability(kernel, X, y, diag, mean=0.0):
    """log N(y | mean, K + diag) by LAPACK, -inf for a non-PD K"""
    K = fisher_np.kernel_matrix(kernel, X)
    K = K + np.diag(np.broadcast_to(np.asarray(diag, dtype=np.float64), (K.shape[0],)))
    c, info = lapack.dpotrf(K, lower=1, clean=1)
    if info != 0:
        return -np.inf
    r = np.asarray(y, dtype=np.float64) - mean
    z = sla.solve_triangular(c, r, lower=True)
    return -0.5 * z @ z - np.sum(np.log(np.diag(c))) - 0.5 * K.shape[0] * np.log(2 * np.pi)
