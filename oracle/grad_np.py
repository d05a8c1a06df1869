"""Gradient of the oracle GP's log-likelihood with NumPy / LAPACK (TEST ORACLE).

For r = y - mean, alpha = K^-1 r and W = K^-1 (LAPACK dpotrf then dpotri):
    d logp / d theta  = 1/2 sum_ij (alpha_i alpha_j - W_ij) dK_ij / d theta
    d logp / d diag_i = 1/2 (alpha_i^2 - W_ii),   d logp / d mean = alpha.
dK / d theta is written in closed form per leaf, from the kernel formulas of the reference's kernels/stationary.py
(:76-235) and the linear maps of transforms.py (:40-161), independently of the CUDA code.  A kernel is walked over the
pairwise coordinate differences D (N1, N2, dims): the weight of a subtree is (alpha alpha^T - W) / 2 times the values
of its Product siblings, and a subtree under a transform returns its D-adjoint sum-free, dK/dD weighted, so that the
transform can form d / d scale.
"""

from __future__ import annotations

import numpy as np
import scipy.linalg as sla
from scipy.linalg import lapack

from oracle import tinygp_np as o


def _dist(node, D):
    """(l1, l2sq, uses_l2) of the leaf's distance (kernels/distance.py:41-59)"""
    return np.sum(np.abs(D), axis=-1), np.sum(D * D, axis=-1), isinstance(node.distance, o.L2Distance)


def _leaf(node, D, Wt, acc, need_adj):
    """value of a stationary leaf; accumulates sum(Wt * dk/dparam); returns Wt * dk/dD when asked"""
    l1, l2sq, l2 = _dist(node, D)
    ell = node.scale
    if isinstance(node, (o.ExpSquared, o.RationalQuadratic)):
        sq = l2sq if l2 else l1 * l1                      # squared_distance
        r2 = sq / ell**2
        if isinstance(node, o.ExpSquared):               # exp(-r2 / 2)
            k = np.exp(-0.5 * r2)
            dk_dr2 = -0.5 * k
        else:                                            # (1 + r2 / (2 alpha))^-alpha
            a = node.alpha
            b = 1.0 + 0.5 * r2 / a
            k = b ** (-a)
            dk_dr2 = -0.5 * k / b
            _add(acc, node, "alpha", np.sum(Wt * k * (0.5 * r2 / (a * b) - np.log(b))))
        _add(acc, node, "scale", np.sum(Wt * dk_dr2 * (-2.0 * r2 / ell)))
        if not need_adj:
            return k, None
        dk_dsq = dk_dr2 / ell**2
        dsq_dD = 2.0 * D if l2 else 2.0 * l1[..., None] * np.sign(D)
        return k, (Wt * dk_dsq)[..., None] * dsq_dD
    dist = np.where(l2sq == 0.0, l1, np.sqrt(np.where(l2sq == 0.0, 1.0, l2sq))) if l2 else l1
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
        s2 = np.sin(np.pi * r) ** 2
        k = np.exp(-node.gamma * s2)
        dk_dr = -node.gamma * np.pi * np.sin(2 * np.pi * r) * k
        _add(acc, node, "gamma", np.sum(Wt * (-s2) * k))
    else:
        raise TypeError(f"no closed-form gradient for {type(node).__name__}")
    _add(acc, node, "scale", np.sum(Wt * dk_dr * (-r / ell)))
    if not need_adj:
        return k, None
    if l2:
        safe = np.where(dist == 0.0, 1.0, dist)
        ddist_dD = np.where((dist == 0.0)[..., None], 0.0, D / safe[..., None])
    else:
        ddist_dD = np.sign(D)
    return k, (Wt * dk_dr / ell)[..., None] * ddist_dD


def _add(acc, node, field, value, index=None):
    key = (id(node), field)
    if key not in acc:
        shape = np.shape(getattr(node, field))
        acc[key] = [node, np.zeros(shape) if shape else 0.0]
    if index is None:
        acc[key][1] = acc[key][1] + value
    else:
        acc[key][1][index] += value


def _value(node, D):
    if isinstance(node, o.Sum):
        return _value(node.kernel1, D) + _value(node.kernel2, D)
    if isinstance(node, o.Product):
        return _value(node.kernel1, D) * _value(node.kernel2, D)
    if isinstance(node, o.Constant):
        return np.full(D.shape[:-1], node.value)
    if isinstance(node, o.Subspace):
        return _value(node.kernel, _subspace(node, D))
    if isinstance(node, (o.Linear, o.Cholesky)):
        return _value(node.kernel, node._map(D))         # linear map of the points = the same map of differences
    return node.evaluate_diff(D)


def _subspace(node, D):
    return D[..., [node.axis]] if np.ndim(node.axis) == 0 else D[..., list(node.axis)]


def _walk(node, D, Wt, acc, need_adj):
    """K of the subtree, sum(Wt * dK/dtheta) into acc, and Wt * dK/dD (element-wise, not summed) if need_adj"""
    if isinstance(node, o.Sum):
        ka, aa = _walk(node.kernel1, D, Wt, acc, need_adj)
        kb, ab = _walk(node.kernel2, D, Wt, acc, need_adj)
        return ka + kb, (aa + ab if need_adj else None)
    if isinstance(node, o.Product):
        va, vb = _value(node.kernel1, D), _value(node.kernel2, D)
        _, aa = _walk(node.kernel1, D, Wt * vb, acc, need_adj)
        _, ab = _walk(node.kernel2, D, Wt * va, acc, need_adj)
        return va * vb, (aa + ab if need_adj else None)
    if isinstance(node, o.Constant):
        _add(acc, node, "value", np.sum(Wt))
        return np.full(D.shape[:-1], node.value), (np.zeros(D.shape) if need_adj else None)
    if isinstance(node, o.Subspace):
        k, a = _walk(node.kernel, _subspace(node, D), Wt, acc, True)
        adj = np.zeros(D.shape)
        for j, ax in enumerate(np.atleast_1d(node.axis)):
            adj[..., ax] += a[..., j]
        return k, adj
    if isinstance(node, (o.Linear, o.Cholesky)):
        p = node.scale if isinstance(node, o.Linear) else node.factor
        if p.ndim >= 2:
            raise TypeError("matrix-valued transforms have no oracle gradient")
        field = "scale" if isinstance(node, o.Linear) else "factor"
        # transforms.py:71-74 (scale * X) and :98-101 (X / factor): D_in = p * D, resp. D / p
        Din = p * D if isinstance(node, o.Linear) else D / p
        k, a = _walk(node.kernel, Din, Wt, acc, True)
        dDin_dp = D if isinstance(node, o.Linear) else -D / p**2
        g = a * dDin_dp
        if p.ndim == 0:
            _add(acc, node, field, np.sum(g))
        else:
            _add(acc, node, field, np.sum(g.reshape(-1, g.shape[-1]), axis=0))
        return k, (a * p if isinstance(node, o.Linear) else a / p)
    return _leaf(node, D, Wt, acc, need_adj)


def log_probability_grad(kernel, X, y, diag, mean=0.0, with_scale=False):
    """(logp, grads, d logp / d diag, alpha) of GaussianProcess(kernel, X, diag=diag, mean=mean).log_probability(y);
    grads maps (id(node), field) -> [node, d logp / d field].  with_scale: a fifth item, the magnitudes of the two terms
    of each gradient, 1/2 |alpha^T K_theta alpha| + 1/2 |tr(W K_theta)| (same keys; for diag 1/2 alpha^2 + 1/2 W_ii),
    the scale of the rounding error a computed gradient may carry"""
    X = np.asarray(X, dtype=np.float64)
    X2 = X[:, None] if X.ndim == 1 else X
    n = X2.shape[0]
    d = np.broadcast_to(np.asarray(diag, dtype=np.float64), (n,))
    r = np.asarray(y, dtype=np.float64) - mean
    D = X2[:, None, :] - X2[None, :, :]
    K = _value(kernel, D) + np.diag(d)
    c, info = lapack.dpotrf(K, lower=1, clean=1)
    if info != 0:
        return -np.inf, None, np.full(n, np.nan), np.full(n, np.nan)
    alpha = sla.cho_solve((c, True), r)
    Wl, info = lapack.dpotri(c, lower=1)
    W = np.tril(Wl) + np.tril(Wl, -1).T
    logp = -0.5 * r @ alpha - np.sum(np.log(np.diag(c))) - 0.5 * n * np.log(2 * np.pi)
    acc: dict = {}
    _walk(kernel, D, 0.5 * (np.outer(alpha, alpha) - W), acc, False)
    ddiag = 0.5 * (alpha * alpha - np.diag(W))
    if not with_scale:
        return logp, acc, ddiag, alpha
    t1: dict = {}
    t2: dict = {}
    _walk(kernel, D, 0.5 * np.outer(alpha, alpha), t1, False)
    _walk(kernel, D, 0.5 * W, t2, False)
    scale = {key: np.abs(t1[key][1]) + np.abs(t2[key][1]) for key in acc}
    scale["diag"] = 0.5 * (alpha * alpha + np.abs(np.diag(W)))
    return logp, acc, ddiag, alpha, scale
