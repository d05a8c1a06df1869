"""Predictive mean and variance of the oracle GP and their gradients with respect to the test inputs, with NumPy /
LAPACK (TEST ORACLE).

For the training covariance K = k(X, X) + diag = L L^T (LAPACK dpotrf), alpha = K^-1 (y - mean), a predictive kernel
k and test points x*_m (the dense branch of the reference's gp.py:225-271 predict, solvers/direct.py:75-95 condition):
    mu_m  = sum_j k(x*_m, x_j) alpha_j + mean
    var_m = k(x*_m, x*_m) + sqrt(eps) - |L^-1 k(X, x*_m)|^2
    d mu_m  / d x*_m = sum_j dk/dD (x*_m - x_j) alpha_j
    d var_m / d x*_m = -2 sum_j dk/dD (x*_m - x_j) v_m,j,   v_m = K^-1 k(X, x*_m)
with dk/dD of grad_x_np.kernel_and_grad (0 at coincident points).  k(x*, x*) does not depend on x* for a stationary k.
"""

from __future__ import annotations

import numpy as np
import scipy.linalg as sla
from scipy.linalg import lapack

from oracle.grad_x_np import kernel_and_grad


def _coords(X):
    X = np.asarray(X, dtype=np.float64)
    return X[:, None] if X.ndim == 1 else X


def predict_and_grad(kernel, X, y, diag, X_test, mean=0.0, pred_kernel=None, with_scale=False):
    """(mu, var, dmu, dvar) of GaussianProcess(kernel, X, diag=diag, mean=mean).predict(y, X_test, kernel=pred_kernel,
    return_var=True) for a constant mean; dmu and dvar have the shape of X_test.  with_scale: two more items, the sums
    of |terms| of dmu and dvar per point and dimension, the scale of the rounding error a computed gradient may carry.
    A non positive-definite K gives NaN everywhere."""
    pred_kernel = kernel if pred_kernel is None else pred_kernel
    X2, Xt = _coords(X), _coords(X_test)
    n, m = X2.shape[0], Xt.shape[0]
    shape = np.shape(X_test)
    d = np.broadcast_to(np.asarray(diag, dtype=np.float64), (n,))
    K, _ = kernel_and_grad(kernel, X2[:, None, :] - X2[None, :, :])
    c, info = lapack.dpotrf(K + np.diag(d), lower=1, clean=1)
    if info != 0:
        nan = (np.full(m, np.nan), np.full(m, np.nan), np.full(shape, np.nan), np.full(shape, np.nan))
        return nan + (np.full(shape, np.nan), np.full(shape, np.nan)) if with_scale else nan
    alpha = sla.cho_solve((c, True), np.asarray(y, dtype=np.float64) - mean)
    Ks, G = kernel_and_grad(pred_kernel, Xt[:, None, :] - X2[None, :, :])       # (m, n), (m, n, dims)
    kss, _ = kernel_and_grad(pred_kernel, np.zeros((m, Xt.shape[1])))
    A = sla.solve_triangular(c, Ks.T, lower=True)                              # L^-1 k(X, X*)
    V = sla.cho_solve((c, True), Ks.T)                                          # K^-1 k(X, X*)
    mu = Ks @ alpha + mean
    var = kss + np.sqrt(np.finfo(np.float64).eps) - np.sum(A * A, axis=0)
    tm = G * alpha[None, :, None]
    tv = -2.0 * G * V.T[:, :, None]
    out = (mu, var, tm.sum(axis=1).reshape(shape), tv.sum(axis=1).reshape(shape))
    if not with_scale:
        return out
    return out + (np.abs(tm).sum(axis=1).reshape(shape), np.abs(tv).sum(axis=1).reshape(shape))
