"""The fp64 GEMM and the diagonal-block step of the dense factorisation, restated with NumPy (TEST ORACLE).

dense.cu's gemm_nt_kernel computes 128 x 128 tiles of C (op)= alpha A B^T over K columns, for `batch` problems whose
operands lie strideA / strideB / strideC elements apart in one buffer each:
    tiles      lower: every (ti, tj) with tj <= ti < tiles_m (C square); else every ti < tiles_m, tj < tiles_n
    beta_mode  0: C = alpha A B^T;   1: C += alpha A B^T;   2: C = G + alpha A B^T with the generated tile
               G(i, j) = k(x_gr, x_gc) + [gr == gc] diag[gr]   for gr = row0 + i < n_valid and gc = col0 + j < n_valid,
                       = [gr == gc]                            otherwise (the identity pad of the factorisation).
Every other element of C is left as it is.  The functions read only the operand elements inside those ranges, so NaN
anywhere else stays out of the result.  With small-integer operands every product and partial sum is exact in fp64, so
these block products equal the kernel's bitwise whatever the summation order.

potf2_trtri_kernel factors one 128 x 128 diagonal block, L L^T = A, inverts L, and reports the first pivot that is not
> 0 as a 1-based column.  exact_factor builds factors for which LAPACK and any other Cholesky / inverse order are exact.
"""

from __future__ import annotations

import numpy as np

TILE = 128


def tiles(tiles_m, tiles_n, lower):
    """the (ti, tj) tiles one launch computes"""
    if lower:
        return [(ti, tj) for ti in range(tiles_m) for tj in range(ti + 1)]
    return [(ti, tj) for ti in range(tiles_m) for tj in range(tiles_n)]


def view(buf, off, rows, cols, ld):
    """rows x cols matrix with row stride ld starting at element off of the flat buffer (a view)"""
    assert off + (rows - 1) * ld + cols <= buf.size
    return np.lib.stride_tricks.as_strided(buf[off:], shape=(rows, cols), strides=(ld * buf.itemsize, buf.itemsize))


def generator(kernel, X, diag, n_valid, gr, gc):
    """G for global row indices gr and column indices gc (1-D arrays); kernel(X1, X2) -> matrix"""
    G = (gr[:, None] == gc[None, :]).astype(np.float64)
    rv, cv = gr[gr < n_valid], gc[gc < n_valid]
    if rv.size and cv.size:
        k = kernel(X[rv], X[cv]) + np.where(rv[:, None] == cv[None, :], diag[rv][:, None], 0.0)
        G[np.ix_(gr < n_valid, gc < n_valid)] = k
    return G


def gemm_nt(C, A, lda, strideA, B, ldb, strideB, ldc, strideC, batch, tiles_m, tiles_n, K, alpha, beta_mode, lower,
            kernel=None, X=None, diag=None, n_valid=0, row0=0, col0=0):
    """a copy of the flat buffer C with every computed tile written, and the boolean mask of the written elements"""
    C = np.array(C, dtype=np.float64)
    written = np.zeros(C.shape, dtype=bool)
    rows = np.arange(TILE)
    for p in range(batch):
        for ti in range(tiles_m):
            a = view(A, p * strideA + ti * TILE * lda, TILE, K, lda)
            tjs = [tj for (i, tj) in tiles(tiles_m, tiles_n, lower) if i == ti]
            b = view(B, p * strideB, (max(tjs) + 1) * TILE, K, ldb)
            prod = a @ b.T                                      # the row of tiles at once: exact for integer operands
            for tj in tjs:
                off = p * strideC + ti * TILE * ldc + tj * TILE
                c = view(C, off, TILE, TILE, ldc)
                acc = prod[:, tj * TILE:(tj + 1) * TILE]
                if beta_mode == 0:
                    c[:] = alpha * acc
                elif beta_mode == 1:
                    c[:] = c + alpha * acc
                else:
                    c[:] = generator(kernel, X, diag, n_valid, row0 + ti * TILE + rows, col0 + tj * TILE + rows) + alpha * acc
                view(written, off, TILE, TILE, ldc)[:] = True
    return C, written


def exact_factor(rng, n=TILE):
    """(L, L^-1) with L = (I + E) D: D_j in {1, 2, 4}; E strictly lower, entries in [-3, 3], nonzero only on rows R x
    columns S with R and S disjoint, so E^2 = 0 and L^-1 = D^-1 (I - E).  K = L L^T is an integer matrix, and every
    intermediate of a Cholesky factorisation of K or of an inversion of L, in any order, is exact in fp64."""
    in_r = rng.random(n) < 0.5
    E = np.tril(rng.integers(-3, 4, (n, n)).astype(np.float64), -1) * np.outer(in_r, ~in_r)
    d = 2.0 ** rng.integers(0, 3, n)
    eye = np.eye(n)
    return (eye + E) * d[None, :], (eye - E) / d[:, None]


def plant_pivot(K, L, c, value):
    """K with the pivot of column c (its Schur complement L_cc^2) changed to `value` (exact for exact_factor's K);
    value = NaN puts NaN on the diagonal"""
    K = K.copy()
    K[c, c] = np.nan if np.isnan(value) else K[c, c] - L[c, c] ** 2 + value
    return K
