"""Gradient of the oracle GP's log-likelihood with respect to the coordinates X, with NumPy / LAPACK (TEST ORACLE).

For r = y - mean, alpha = K^-1 r and W = K^-1 (LAPACK dpotrf then dpotri), and a stationary kernel k(x_i, x_j) =
k(D_ij) of the difference D_ij = x_i - x_j:
    d logp / d x_i = sum_{j != i} (alpha_i alpha_j - W_ij) dk/dD (D_ij)
(K_ij and K_ji both depend on x_i; dk/dD is odd in D, so both halves of 1/2 sum_ij (...) dK_ij add up).  dk/dD is
written in closed form per leaf from the kernel formulas of the reference's kernels/stationary.py (:76-235); a linear
input transform (transforms.py:40-161) maps D by its matrix J and the gradient by J^T.  At coincident points (D = 0) the
gradient is taken as 0: sign(0) = 0 for the L1 distance, and 0 for leaves on the L2 distance (the Exp leaf has no
derivative there).
"""

from __future__ import annotations

import numpy as np
import scipy.linalg as sla
from scipy.linalg import lapack

from oracle import tinygp_np as o


def _leaf(node, D):
    """(k, dk/dD) of a stationary leaf over the differences D (..., dims)"""
    l2 = isinstance(node.distance, o.L2Distance)
    l1, l2sq = np.sum(np.abs(D), axis=-1), np.sum(D * D, axis=-1)
    ell = node.scale
    if isinstance(node, (o.ExpSquared, o.RationalQuadratic)):
        sq = l2sq if l2 else l1 * l1                      # squared_distance
        r2 = sq / ell**2
        if isinstance(node, o.ExpSquared):               # exp(-r2 / 2)
            k = np.exp(-0.5 * r2)
            dk_dsq = -0.5 * k / ell**2
        else:                                            # (1 + r2 / (2 alpha))^-alpha
            b = 1.0 + 0.5 * r2 / node.alpha
            k = b ** (-node.alpha)
            dk_dsq = -0.5 * k / (b * ell**2)
        dsq_dD = 2.0 * D if l2 else 2.0 * l1[..., None] * np.sign(D)
        return k, dk_dsq[..., None] * dsq_dD
    dist = np.sqrt(l2sq) if l2 else l1
    r = dist / ell
    if isinstance(node, o.Exp):
        k = np.exp(-r)
        dk_dr = -k
    elif isinstance(node, o.Matern32):
        e = np.exp(-np.sqrt(3.0) * r)
        k = (1.0 + np.sqrt(3.0) * r) * e
        dk_dr = -3.0 * r * e
    elif isinstance(node, o.Matern52):
        e = np.exp(-np.sqrt(5.0) * r)
        k = (1.0 + np.sqrt(5.0) * r + 5.0 * r * r / 3.0) * e
        dk_dr = -(5.0 / 3.0) * r * (1.0 + np.sqrt(5.0) * r) * e
    elif isinstance(node, o.Cosine):
        k = np.cos(2 * np.pi * r)
        dk_dr = -2 * np.pi * np.sin(2 * np.pi * r)
    elif isinstance(node, o.ExpSineSquared):
        k = np.exp(-node.gamma * np.sin(np.pi * r) ** 2)
        dk_dr = -node.gamma * np.pi * np.sin(2 * np.pi * r) * k
    else:
        raise TypeError(f"no closed-form coordinate gradient for {type(node).__name__}")
    if l2:
        safe = np.where(dist == 0.0, 1.0, dist)
        ddist_dD = np.where((dist == 0.0)[..., None], 0.0, D / safe[..., None])
    else:
        ddist_dD = np.sign(D)
    return k, (dk_dr / ell)[..., None] * ddist_dD


def _jacobian(node, dims):
    """matrix J of a linear input transform: transformed differences = D @ J^T"""
    return np.stack([np.atleast_1d(node._map(e)) for e in np.eye(dims)], axis=-1)


def kernel_and_grad(node, D):
    """(K, dK/dD) of a kernel expression over the differences D (..., dims)"""
    if isinstance(node, o.Sum):
        ka, ga = kernel_and_grad(node.kernel1, D)
        kb, gb = kernel_and_grad(node.kernel2, D)
        return ka + kb, ga + gb
    if isinstance(node, o.Product):
        ka, ga = kernel_and_grad(node.kernel1, D)
        kb, gb = kernel_and_grad(node.kernel2, D)
        return ka * kb, kb[..., None] * ga + ka[..., None] * gb
    if isinstance(node, o.Constant):
        return np.full(D.shape[:-1], node.value), np.zeros(D.shape)
    if isinstance(node, (o.Linear, o.Cholesky, o.Subspace)):
        J = _jacobian(node, D.shape[-1])
        k, g = kernel_and_grad(node.kernel, D @ J.T)
        return k, g @ J
    return _leaf(node, D)


def log_probability_grad_x(kernel, X, y, diag, mean=0.0, with_scale=False):
    """(logp, d logp / d X, alpha) of GaussianProcess(kernel, X, diag=diag, mean=mean).log_probability(y) for a constant
    mean; d logp / d X has the shape of X.  with_scale: a fourth item, sum_j |(alpha_i alpha_j - W_ij) dk/dD (D_ij)| per
    point and dimension, the scale of the rounding error a computed gradient may carry."""
    X = np.asarray(X, dtype=np.float64)
    X2 = X[:, None] if X.ndim == 1 else X
    n = X2.shape[0]
    d = np.broadcast_to(np.asarray(diag, dtype=np.float64), (n,))
    r = np.asarray(y, dtype=np.float64) - mean
    D = X2[:, None, :] - X2[None, :, :]
    Kx, G = kernel_and_grad(kernel, D)
    c, info = lapack.dpotrf(Kx + np.diag(d), lower=1, clean=1)
    if info != 0:
        out = (-np.inf, np.full(X.shape, np.nan), np.full(n, np.nan))
        return out + (np.full(X.shape, np.nan),) if with_scale else out
    alpha = sla.cho_solve((c, True), r)
    Wl, info = lapack.dpotri(c, lower=1)
    W = np.tril(Wl) + np.tril(Wl, -1).T
    logp = -0.5 * r @ alpha - np.sum(np.log(np.diag(c))) - 0.5 * n * np.log(2 * np.pi)
    omega = np.outer(alpha, alpha) - W
    np.fill_diagonal(omega, 0.0)
    terms = omega[..., None] * G
    dX = np.sum(terms, axis=1).reshape(X.shape)
    if not with_scale:
        return logp, dX, alpha
    return logp, dX, alpha, np.sum(np.abs(terms), axis=1).reshape(X.shape)
