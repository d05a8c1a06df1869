"""The tile schedules of the gradient's triangular GEMM kernel, restated with NumPy (TEST ORACLE).

grad.cu's tri_gemm_kernel computes 128 x 128 tiles over a per-tile range of 128-blocks of K, with the diagonal blocks
of an operand taken from a separate array:
    TRMM      block column j of X = L^-1:  C(ti, j) = sum_{k=j+1..ti} A(ti, k) B(0, k)^T   for ti = j+1..T-1,
              A(ti, ti) read from diagA (B is 128 x np);
    CONTRACT  W = K^-1 = U U^T:  W(ti, tj) = sum_{k=ti..T-1} U(ti, k) U(tj, k)^T   for ti >= tj,
              U's diagonal blocks read from diagU;
and the CONTRACT epilogue weights each element i >= j (i, j < n) of a W tile by
    wt = (1 if i == j else 2) (alpha_i alpha_j - W_ij)
and, for the coordinate gradient, adds om g_ij (om = alpha_i alpha_j - W_ij for i > j, g_ij = d k / d delta at
x_i - x_j) to the tile's row sum of i and to its column sum of j; dX_i = sum_{J <= I} row sums of tile (I, J) -
sum_{I' >= I} column sums of tile (I', I).
Each function reads only the blocks in its ranges, so NaN anywhere else stays out of the result.  With operands whose
products and sums are exact in fp64 (small integers), the block products below equal the kernel's bitwise whatever
the summation order.
"""

from __future__ import annotations

import numpy as np
import scipy.linalg as sla

from oracle import grad_x_np

TILE = 128


def _blk(M, r, k, diag=None):
    if diag is not None and r == k:
        return diag[r]
    return M[r * TILE:(r + 1) * TILE, k * TILE:(k + 1) * TILE]


def tile_index(ti, tj):
    """CTA / partial index of the W tile (ti, tj), ti >= tj"""
    return ti * (ti + 1) // 2 + tj


def trmm(C, A, diagA, B, T, j):
    """C with the tiles of the inverse step for block column j written; diagA: (T, 128, 128)"""
    C = C.copy()
    for ti in range(j + 1, T):
        acc = np.zeros((TILE, TILE))
        for k in range(j + 1, ti + 1):
            acc += _blk(A, ti, k, diagA) @ B[:, k * TILE:(k + 1) * TILE].T
        C[ti * TILE:(ti + 1) * TILE, j * TILE:(j + 1) * TILE] = acc
    return C


def contract(U, diagU, T):
    """{(ti, tj): W tile} for ti >= tj"""
    W = {}
    for ti in range(T):
        for tj in range(ti + 1):
            acc = np.zeros((TILE, TILE))
            for k in range(ti, T):
                acc += _blk(U, ti, k, diagU) @ _blk(U, tj, k, diagU).T
            W[(ti, tj)] = acc
    return W


def inverse(L, T):
    """(X = L^-1, the diagonal blocks' inverses) by the gradient's driver: for j = T-2 .. 0 the panel
    Pt(k) = -X_jj^T L_kj^T for k > j, then the TRMM step into block column j of L, in place"""
    M = np.array(L, dtype=np.float64)
    eye = np.eye(TILE)
    linv = np.stack([sla.solve_triangular(_blk(M, b, b), eye, lower=True) for b in range(T)])
    np_ = T * TILE
    Pt = np.full((TILE, np_), np.nan)
    for j in range(T - 2, -1, -1):
        Pt[:, (j + 1) * TILE:] = -(linv[j].T @ M[(j + 1) * TILE:, j * TILE:(j + 1) * TILE].T)
        M = trmm(M, M, linv, Pt, T, j)
    for b in range(T):
        M[b * TILE:(b + 1) * TILE, b * TILE:(b + 1) * TILE] = linv[b]
    return np.tril(M), linv


def epilogue(W, alpha, n, T, kernel=None, X=None):
    """what the CONTRACT epilogue derives from the W tiles: (wdiag (n), wsum, dx) with wsum[t] = the tile's sum of wt
    (the partial of a slot whose d k / d slot is 1 everywhere, e.g. an added Constant).  With an oracle kernel
    expression and X (n, ndim): dx = (rows, cols, rows_scale, cols_scale, dX, dX_scale), rows / cols the per-tile
    (ntiles, ndim, 128) sums and the scales the same sums of |om g|; else dx = None."""
    np_ = T * TILE
    a = np.zeros(np_)
    a[:n] = alpha
    idx = np.arange(TILE)
    ntiles = T * (T + 1) // 2
    wdiag = np.zeros(np_)
    wsum = np.zeros(ntiles)
    nd = None if X is None else X.shape[1]
    if nd is not None:
        rows, cols = np.zeros((ntiles, nd, TILE)), np.zeros((ntiles, nd, TILE))
        rows_s, cols_s = np.zeros((ntiles, nd, TILE)), np.zeros((ntiles, nd, TILE))
    for (ti, tj), w in W.items():
        t = tile_index(ti, tj)
        i, jj = ti * TILE + idx[:, None], tj * TILE + idx[None, :]
        valid = (i < n) & (jj < n) & (jj <= i)
        om = np.outer(a[ti * TILE:(ti + 1) * TILE], a[tj * TILE:(tj + 1) * TILE]) - w
        wt = np.where(i == jj, 1.0, 2.0) * om
        wsum[t] = np.sum(wt[valid])
        if ti == tj:
            wdiag[ti * TILE:(ti + 1) * TILE] = np.diag(w)
        if nd is None:
            continue
        ri, cj = np.minimum(i[:, 0], n - 1), np.minimum(jj[0], n - 1)
        D = X[ri][:, None, :] - X[cj][None, :, :]
        _, g = grad_x_np.kernel_and_grad(kernel, D)
        terms = np.where((valid & (i > jj))[..., None], om[..., None] * g, 0.0)
        rows[t], cols[t] = np.sum(terms, axis=1).T, np.sum(terms, axis=0).T
        rows_s[t], cols_s[t] = np.sum(np.abs(terms), axis=1).T, np.sum(np.abs(terms), axis=0).T
    if nd is None:
        return wdiag[:n], wsum, None
    return wdiag[:n], wsum, (rows, cols, rows_s, cols_s) + reduce_dx(rows, cols, rows_s, cols_s, T, n)


def reduce_dx(rows, cols, rows_s, cols_s, T, n):
    """(dX, its scale) from the per-tile sums, as dx_reduce_kernel adds them"""
    nd = rows.shape[1]
    dX, sc = np.zeros((T * TILE, nd)), np.zeros((T * TILE, nd))
    for I in range(T):
        s = slice(I * TILE, (I + 1) * TILE)
        for J in range(I + 1):
            dX[s] += rows[tile_index(I, J)].T
            sc[s] += rows_s[tile_index(I, J)].T
        for I2 in range(I, T):
            dX[s] -= cols[tile_index(I2, I)].T
            sc[s] += cols_s[tile_index(I2, I)].T
    return dX[:n], sc[:n]
