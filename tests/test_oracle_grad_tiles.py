"""oracle/grad_tiles_np.py, the NumPy restatement of the gradient's tile schedules that test_grad_tiles_exact_gpu.py
compares the kernel with, checked on a factor whose inverse is known exactly.

L = (I + E) D with E strictly lower, integer, nonzero only on rows R x columns S for disjoint R and S, so that E^2 = 0,
L^-1 = D^-1 (I - E) and K^-1 = L^-T L^-1 = (I - E)^T D^-2 (I - E).  With D's entries in {1, 2} every product and
partial sum of the schedules is a short dyadic fraction, exact in fp64 in any order: the driver's inverse must equal
L^-1 bitwise and the contraction K^-1 bitwise."""

import numpy as np
import pytest
from scipy.linalg import lapack

from oracle import grad_tiles_np as gt

TILE = gt.TILE


def _factor(n, T, seed):
    """(L, L^-1, K^-1) padded to 128 T with the identity"""
    rng = np.random.default_rng(seed)
    np_ = T * TILE
    in_r = np.zeros(np_, dtype=bool)
    in_r[:n] = rng.random(n) < 0.5
    in_s = np.zeros(np_, dtype=bool)
    in_s[:n] = ~in_r[:n]
    E = rng.integers(-2, 3, (np_, np_)).astype(np.float64) * (rng.random((np_, np_)) < 0.3)
    E = np.tril(E, -1) * np.outer(in_r, in_s)
    assert not np.any(E @ E)
    d = np.ones(np_)
    d[:n] = rng.integers(1, 3, n)
    eye = np.eye(np_)
    L = (eye + E) * d[None, :]
    Linv = (eye - E) / d[:, None]
    Kinv = (eye - E).T @ np.diag(d ** -2.0) @ (eye - E)
    return L, Linv, Kinv


@pytest.mark.parametrize("n,T", [(128, 1), (129, 2), (256, 2), (300, 3), (1100, 9), (1111, 9)])
def test_inverse_and_contraction_are_exact(n, T):
    L, Linv, Kinv = _factor(n, T, seed=n)
    X, linv = gt.inverse(L, T)
    assert np.array_equal(X, Linv)
    U = X.T.copy()                                      # the driver mirrors X's lower triangle into the upper one
    U[np.tril_indices_from(U, -1)] = np.nan             # blocks below the diagonal are never read
    for b in range(T):
        U[b * TILE:(b + 1) * TILE, b * TILE:(b + 1) * TILE] = np.nan
    W = gt.contract(U, np.ascontiguousarray(linv.transpose(0, 2, 1)), T)
    assert len(W) == T * (T + 1) // 2
    for (ti, tj), w in W.items():
        assert np.array_equal(w, Kinv[ti * TILE:(ti + 1) * TILE, tj * TILE:(tj + 1) * TILE]), (ti, tj)


def test_lapack_factors_the_construction_exactly():
    """the construction is a Cholesky factor as LAPACK computes it, so K = L L^T is a fair stand-in for a real K"""
    L, _, _ = _factor(300, 3, seed=5)
    c, info = lapack.dpotrf(L @ L.T, lower=1, clean=1)
    assert info == 0 and np.array_equal(c, L)


def test_epilogue_weights_and_reduction():
    """wdiag, the per-tile sums of wt and the dX reduction against direct sums over the whole matrix"""
    from oracle import tinygp_np as o
    from oracle import grad_x_np

    rng = np.random.default_rng(2)
    T, n = 3, 300
    _, _, Kinv = _factor(n, T, seed=3)
    W = {(ti, tj): Kinv[ti * TILE:(ti + 1) * TILE, tj * TILE:(tj + 1) * TILE] for ti in range(T) for tj in range(ti + 1)}
    alpha = rng.integers(-3, 4, n).astype(np.float64)
    X = rng.uniform(0, 3, (n, 2))
    k = o.Matern32(1.1) + o.Linear(np.array([0.7, 1.3]), o.ExpSquared(1.0))
    wdiag, wsum, (rows, cols, _, _, dX, sc) = gt.epilogue(W, alpha, n, T, k, X)
    Wn = Kinv[:n, :n]
    assert np.array_equal(wdiag, np.diag(Wn))
    om = np.outer(alpha, alpha) - Wn
    assert np.sum(wsum) == np.sum(np.tril(om, -1)) * 2 + np.sum(np.diag(om))
    _, g = grad_x_np.kernel_and_grad(k, X[:, None, :] - X[None, :, :])
    terms = np.tril(om, -1)[..., None] * g
    # the lower triangle of (om g) adds to row i and subtracts from column j
    ref = terms.sum(axis=1) - terms.sum(axis=0)
    assert np.all(np.abs(dX - ref) <= 1e-13 * sc)
    assert rows.shape == cols.shape == (T * (T + 1) // 2, 2, TILE)
    # the full-matrix form of oracle/grad_x_np.py agrees: it sums (om g)_ij over j != i, om symmetric and g odd
    om_full = om.copy()
    np.fill_diagonal(om_full, 0.0)
    assert np.allclose(dX, np.sum(om_full[..., None] * g, axis=1), rtol=0, atol=1e-12 * np.max(sc))
