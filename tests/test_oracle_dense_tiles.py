"""oracle/dense_tiles_np.py, the NumPy restatement of the dense factorisation's GEMM tiles and diagonal-block step that
test_dense_tiles_exact_gpu.py compares the kernels with, checked against direct whole-matrix computations and LAPACK."""

import numpy as np
import pytest
from scipy.linalg import lapack

from oracle import dense_tiles_np as dt
from oracle import tinygp_np as o

TILE = dt.TILE


def test_tile_sets():
    for T in (1, 2, 15, 16, 17, 33):
        low = dt.tiles(T, T, True)
        assert len(low) == len(set(low)) == T * (T + 1) // 2
        assert set(low) == {(ti, tj) for ti in range(T) for tj in range(T) if tj <= ti}
    assert dt.tiles(3, 4, False) == [(ti, tj) for ti in range(3) for tj in range(4)]


@pytest.mark.parametrize("beta_mode", [0, 1])
@pytest.mark.parametrize("lower", [0, 1])
def test_gemm_tiles_against_whole_products(beta_mode, lower):
    """two problems in one buffer, with NaN in every operand element outside the tiles' rows and K columns"""
    rng = np.random.default_rng(3 + lower)
    tm, tn, K, batch, alpha = (3, 3, 256, 2, -1.0) if lower else (2, 3, 256, 2, 1.0)
    lda, ldb, ldc = K + 4, K + 2, tn * TILE + 6
    sA, sB, sC = (tm * TILE + 1) * lda, (tn * TILE + 2) * ldb + 2, (tm * TILE + 3) * ldc
    A, B, C0 = np.full(batch * sA, np.nan), np.full(batch * sB, np.nan), np.full(batch * sC, -7.0)
    for p in range(batch):
        dt.view(A, p * sA, tm * TILE, K, lda)[:] = rng.integers(-4, 5, (tm * TILE, K))
        dt.view(B, p * sB, tn * TILE, K, ldb)[:] = rng.integers(-4, 5, (tn * TILE, K))
        dt.view(C0, p * sC, tm * TILE, tn * TILE, ldc)[:] = rng.integers(-4, 5, (tm * TILE, tn * TILE))
    C, written = dt.gemm_nt(C0, A, lda, sA, B, ldb, sB, ldc, sC, batch, tm, tn, K, alpha, beta_mode, lower)
    assert np.all(C[~written] == C0[~written])
    for p in range(batch):
        a, b = dt.view(A, p * sA, tm * TILE, K, lda), dt.view(B, p * sB, tn * TILE, K, ldb)
        c0, c = dt.view(C0, p * sC, tm * TILE, tn * TILE, ldc), dt.view(C, p * sC, tm * TILE, tn * TILE, ldc)
        want = alpha * (a @ b.T) + (c0 if beta_mode else 0.0)
        mask = np.kron(np.tril(np.ones((tm, tn))) if lower else np.ones((tm, tn)), np.ones((TILE, TILE))) > 0
        assert np.array_equal(c[mask], want[mask])
        assert np.array_equal(c[~mask], c0[~mask])
        assert np.all(dt.view(written, p * sC, tm * TILE, tn * TILE, ldc) == mask)


def test_generator_diag_and_identity_pad():
    rng = np.random.default_rng(4)
    n_valid, nd = 300, 2
    X = rng.uniform(0, 3, (n_valid, nd))
    diag = rng.integers(1, 8, n_valid) / 4.0
    k = o.Constant(0.75) + o.ExpSquared(1.1)
    gr, gc = np.arange(256, 384), np.arange(128, 384)
    G = dt.generator(k, X, diag, n_valid, gr, gc)
    full = np.eye(384)
    full[:n_valid, :n_valid] = k(X, X) + np.diag(diag)
    assert np.array_equal(G, full[256:384, 128:384])
    assert np.all(G[n_valid - 256:, :][:, gc < n_valid] == 0.0)          # pad rows: 0 off the diagonal ...
    assert np.all(np.diag(G[:, 128:])[n_valid - 256:] == 1.0)             # ... and 1 on it


@pytest.mark.parametrize("seed", range(20))
def test_lapack_reproduces_the_exact_factor(seed):
    L, Linv = dt.exact_factor(np.random.default_rng(seed))
    assert np.array_equal(L @ Linv, np.eye(TILE))
    K = L @ L.T
    assert np.array_equal(K, np.round(K)) and np.max(np.abs(K)) < 2.0 ** 30
    c, info = lapack.dpotrf(K, lower=1, clean=1)
    assert info == 0 and np.array_equal(c, L)
    inv, info = lapack.dtrtri(c, lower=1)
    assert info == 0 and np.array_equal(np.tril(inv), Linv)


@pytest.mark.parametrize("value", [-1.0, 0.0])     # NaN is not checked: some LAPACK builds let a NaN pivot pass
@pytest.mark.parametrize("col", [0, 7, 8, 63, 127])
def test_lapack_reports_the_planted_pivot(col, value):
    L, _ = dt.exact_factor(np.random.default_rng(col))
    K = dt.plant_pivot(L @ L.T, L, col, value)
    _, info = lapack.dpotrf(K, lower=1)
    assert info == col + 1
    if col < 100:       # a second bad pivot further on does not change the report
        _, info = lapack.dpotrf(dt.plant_pivot(K, L, col + 20, -1.0), lower=1)
        assert info == col + 1
