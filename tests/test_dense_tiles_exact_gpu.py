"""The dense factorisation's fp64 GEMM (dense.cu gemm_nt_kernel, through b200gp_gemm_nt_test) and its diagonal-block
kernel (potf2_trtri_kernel, through b200gp_potf2_test) against the NumPy restatement in oracle/dense_tiles_np.py.

GEMM operands are integers in [-4, 4], so every tile is exact in fp64 in any summation order and results are compared
exactly.  Every operand element a tile must not read (columns >= K, rows outside the launched tiles, the gaps between
the problems of a batch) holds NaN, and C starts as a sentinel outside the tiles a launch computes, so a read outside
a range shows up as NaN and a write outside the tiles as a changed sentinel.  The diagonal-block kernel is run on
L = (I + E) D blocks whose factor and inverse are exact in any order, with NaN in the strict upper triangle it must not
read."""

import numpy as np
import pytest
import scipy.linalg as sla

from oracle import dense_tiles_np as dt
from tinygp_b200 import _cabi, kernels
from util import to_oracle

pytestmark = pytest.mark.gpu

TILE = dt.TILE
SENTINEL = -1234.5


def _p(a):
    return None if a is None else _cabi.ptr(a)


def _gemm(A, lda, sA, B, ldb, sB, C, ldc, sC, batch, tm, tn, K, alpha, beta, lower, prog=None, X=None, diag=None,
          n_valid=0, row0=0, col0=0):
    ctx = _cabi.get_context()
    C = C.copy()
    nd = 0 if X is None else X.shape[1]
    ctx.check(ctx.lib.b200gp_gemm_nt_test(
        ctx.handle, _p(A), A.size, lda, sA, _p(B), B.size, ldb, sB, _p(C), C.size, ldc, sC, batch, tm, tn, K, alpha,
        beta, lower, _p(prog), 0 if prog is None else prog.shape[0], _p(X), nd, _p(diag), n_valid, row0, col0))
    return C


def _operands(tm, tn, K, batch, seed):
    """A, B and C buffers for `batch` problems with unequal strides: NaN in A and B outside the tiles' rows and K
    columns, C all sentinel"""
    rng = np.random.default_rng(seed)
    lda, ldb, ldc = K + 4, K + 2, tn * TILE + 6
    sA, sB, sC = (tm * TILE + 1) * lda + 2, (tn * TILE + 2) * ldb, (tm * TILE + 3) * ldc + 4
    A, B, C = np.full(batch * sA, np.nan), np.full(batch * sB, np.nan), np.full(batch * sC, SENTINEL)
    for p in range(batch):
        dt.view(A, p * sA, tm * TILE, K, lda)[:] = rng.integers(-4, 5, (tm * TILE, K))
        dt.view(B, p * sB, tn * TILE, K, ldb)[:] = rng.integers(-4, 5, (tn * TILE, K))
    return A, (lda, sA), B, (ldb, sB), C, (ldc, sC), rng


def _fill_tiles(C, ldc, sC, batch, tiles, values):
    for p in range(batch):
        for ti, tj in tiles:
            dt.view(C, p * sC + ti * TILE * ldc + tj * TILE, TILE, TILE, ldc)[:] = values()


def _check(got, want, written, what):
    bad = ~((got == want) | (np.isnan(got) & np.isnan(want)))
    assert not np.any(bad & ~written), (what, "elements outside the computed tiles changed", int(np.sum(bad & ~written)))
    assert not np.any(bad), (what, "tile elements differ", int(np.sum(bad)), int(np.sum(np.isnan(got[written]))))


# lower: T crosses the band heights 16 and 32 of the tile rasterisation; rectangular: one column and a full grid
GEMM_SHAPES = [(T, T, 1) for T in (1, 2, 15, 16, 17, 32, 33)] + [(1, 1, 0), (5, 1, 0), (3, 4, 0)]


@pytest.mark.parametrize("beta", [0, 1])
@pytest.mark.parametrize("K", [128, 256, 1024])
@pytest.mark.parametrize("tm,tn,lower", GEMM_SHAPES)
def test_gemm_tiles_exact(tm, tn, lower, K, beta):
    alpha = (-1.0) ** (K // TILE + beta)        # each beta_mode runs with alpha = +1 and -1 over the K values
    batch = 3 if tm <= 17 else 2
    A, (lda, sA), B, (ldb, sB), C, (ldc, sC), rng = _operands(tm, tn, K, batch, seed=tm * 1000 + tn * 10 + K + beta)
    tiles = dt.tiles(tm, tn, lower)
    # the computed tiles start as NaN where C must not be read (beta 0), as integers where it is added to (beta 1)
    _fill_tiles(C, ldc, sC, batch, tiles,
                (lambda: np.nan) if beta == 0 else (lambda: rng.integers(-4, 5, (TILE, TILE))))
    want, written = dt.gemm_nt(C, A, lda, sA, B, ldb, sB, ldc, sC, batch, tm, tn, K, alpha, beta, lower)
    got = _gemm(A, lda, sA, B, ldb, sB, C, ldc, sC, batch, tm, tn, K, alpha, beta, lower)
    _check(got, want, written, (tm, tn, lower, K, beta))


def _generator_case(tm, tn, lower, row0, seed):
    n_valid = row0 + min(tm, tn) * TILE - 37            # ragged inside the last tile of the shorter side
    A, (lda, sA), B, (ldb, sB), C, (ldc, sC), rng = _operands(tm, tn, 256, 1, seed)
    _fill_tiles(C, ldc, sC, 1, dt.tiles(tm, tn, lower), lambda: np.nan)
    return n_valid, A, (lda, sA), B, (ldb, sB), C, (ldc, sC), rng


@pytest.mark.parametrize("row0", [0, 256])
@pytest.mark.parametrize("tm,tn,lower", [(1, 1, 1), (3, 3, 1), (17, 17, 1), (3, 3, 0), (4, 2, 0)])
def test_generator_epilogue_exact(tm, tn, lower, row0):
    """beta_mode 2 with a constant kernel and dyadic diag, so that the generated tile is exact: diag at the global
    diagonal row0 + i == col0 + j, the identity pad from n_valid on"""
    n_valid, A, (lda, sA), B, (ldb, sB), C, (ldc, sC), rng = _generator_case(tm, tn, lower, row0, seed=tm + row0)
    X = rng.uniform(0, 3, (n_valid, 2))
    diag = rng.integers(1, 8, n_valid) / 4.0
    k = kernels.Constant(0.75)
    want, written = dt.gemm_nt(C, A, lda, sA, B, ldb, sB, ldc, sC, 1, tm, tn, 256, -1.0, 2, lower, kernel=to_oracle(k),
                               X=X, diag=diag, n_valid=n_valid, row0=row0, col0=row0)
    got = _gemm(A, lda, sA, B, ldb, sB, C, ldc, sC, 1, tm, tn, 256, -1.0, 2, lower, prog=k.program(), X=X, diag=diag,
                n_valid=n_valid, row0=row0, col0=row0)
    _check(got, want, written, (tm, tn, lower, row0))


def test_generator_epilogue_real_kernel():
    """a two-leaf program in 3-D: the generated tile against the oracle's kernel within 2e-15 (|k| + |AB|)"""
    tm = tn = 3
    row0 = 256
    n_valid, A, (lda, sA), B, (ldb, sB), C, (ldc, sC), rng = _generator_case(tm, tn, 1, row0, seed=9)
    X = rng.uniform(0, 3, (n_valid, 3))
    diag = rng.uniform(0.05, 0.2, n_valid)
    k = 1.3 * kernels.ExpSquared(0.8) + 0.4 * kernels.Matern32(1.1, kernels.L2Distance())
    ko = to_oracle(k)
    common = (C, A, lda, sA, B, ldb, sB, ldc, sC, 1, tm, tn, 256)
    gen = dict(kernel=ko, X=X, diag=diag, n_valid=n_valid, row0=row0, col0=row0)
    want, written = dt.gemm_nt(*common, -1.0, 2, 1, **gen)
    G, _ = dt.gemm_nt(*common, 0.0, 2, 1, **gen)
    AB, _ = dt.gemm_nt(*common, 1.0, 0, 1)
    got = _gemm(A, lda, sA, B, ldb, sB, C, ldc, sC, 1, tm, tn, 256, -1.0, 2, 1, prog=k.program(), X=X, diag=diag,
                n_valid=n_valid, row0=row0, col0=row0)
    assert np.all(got[~written] == SENTINEL)
    err = np.abs(got[written] - want[written])
    tol = 2e-15 * (np.abs(G[written]) + np.abs(AB[written]))
    assert np.all(err <= tol), (int(np.sum(~(err <= tol))), float(np.max(err - tol)))


# ---- the diagonal-block kernel ----
LDA = 384


def _potf2(A, sA, batch, global_off):
    ctx = _cabi.get_context()
    A = A.copy()
    linv = np.full((batch, TILE, TILE), np.nan)
    info = np.full(batch, -1, dtype=np.int32)
    ctx.check(ctx.lib.b200gp_potf2_test(ctx.handle, _cabi.ptr(A), A.size, LDA, sA, batch, global_off,
                                        _cabi.ptr(linv), _cabi.ptr(info)))
    return A, linv, info


def _blocks(Ks):
    """the blocks at A + p sA (row stride 384, columns shifted by 64 p): lower triangles of Ks, NaN in the strict
    upper triangles, the sentinel everywhere else"""
    sA = (TILE + 2) * LDA + 64
    A = np.full(len(Ks) * sA, SENTINEL)
    upper = np.triu(np.ones((TILE, TILE), dtype=bool), 1)
    for p, K in enumerate(Ks):
        dt.view(A, p * sA, TILE, TILE, LDA)[:] = np.where(upper, np.nan, K)
    return A, sA


def _same(got, want):
    return np.array_equal(got, want, equal_nan=True)


@pytest.mark.parametrize("global_off", [0, 1024])
def test_diagonal_block_exact(global_off):
    rng = np.random.default_rng(global_off + 1)
    Ls = [dt.exact_factor(rng) for _ in range(3)]
    A, sA = _blocks([L @ L.T for L, _ in Ls])
    got, linv, info = _potf2(A, sA, 3, global_off)
    want, _ = _blocks([L for L, _ in Ls])            # L below, the upper NaN and the sentinel untouched
    assert _same(got, want), int(np.sum(~((got == want) | (np.isnan(got) & np.isnan(want)))))
    for p, (_, Linv) in enumerate(Ls):
        assert np.array_equal(linv[p], Linv), (p, float(np.max(np.abs(linv[p] - Linv))))
        assert np.all(linv[p][np.triu_indices(TILE, 1)] == 0.0)
    assert np.all(info == 0)


def test_diagonal_block_random_spd():
    """condition number about 1e3: L and L^-1 against LAPACK within 1e-12 of their largest entries"""
    rng = np.random.default_rng(77)
    Ks = []
    for _ in range(3):
        Q, _ = np.linalg.qr(rng.normal(size=(TILE, TILE)))
        K = (Q * np.logspace(0, -3, TILE)) @ Q.T
        Ks.append(0.5 * (K + K.T))
    A, sA = _blocks(Ks)
    got, linv, info = _potf2(A, sA, 3, 0)
    assert np.all(info == 0)
    for p, K in enumerate(Ks):
        L = np.linalg.cholesky(K)
        Li = sla.solve_triangular(L, np.eye(TILE), lower=True)
        Lg = np.tril(dt.view(got, p * sA, TILE, TILE, LDA))
        assert np.max(np.abs(Lg - L)) <= 1e-12 * np.max(np.abs(L))
        assert np.max(np.abs(linv[p] - Li)) <= 1e-12 * np.max(np.abs(Li))


@pytest.mark.parametrize("global_off", [0, 1024])
@pytest.mark.parametrize("value", [-1.0, 0.0, np.nan])
@pytest.mark.parametrize("col", [0, 7, 8, 63, 127])
def test_first_bad_pivot_index(col, value, global_off):
    """problem 0: one bad pivot at col; problem 1: none; problem 2: bad pivots at c2 and c2 + 9, reported as c2"""
    rng = np.random.default_rng(col)
    Ls = [dt.exact_factor(rng)[0] for _ in range(3)]
    c2 = (col * 5 + 3) % 118
    Ks = [dt.plant_pivot(Ls[0] @ Ls[0].T, Ls[0], col, value), Ls[1] @ Ls[1].T,
          dt.plant_pivot(dt.plant_pivot(Ls[2] @ Ls[2].T, Ls[2], c2 + 9, -1.0), Ls[2], c2, value)]
    A, sA = _blocks(Ks)
    got, _, info = _potf2(A, sA, 3, global_off)
    assert info.tolist() == [global_off + col + 1, 0, global_off + c2 + 1]
    # the columns before the bad pivot are the exact factor's
    assert np.array_equal(np.tril(dt.view(got, 0, TILE, TILE, LDA))[:, :col], np.tril(Ls[0])[:, :col])


def test_sizes_are_checked_before_launch():
    ctx = _cabi.get_context()
    lib, h = ctx.lib, ctx.handle
    A, B, C = np.zeros(256 * 130), np.zeros(256 * 130), np.zeros(256 * 256)
    X, d = np.zeros((10, 2)), np.zeros(10)
    prog = kernels.Constant(0.75).program()
    P = _cabi.ptr

    def gemm(lda=130, sA=0, tm=2, tn=2, K=128, beta=0, lower=1, batch=1, a=A, ldc=256, n_valid=10, pr=prog):
        return lib.b200gp_gemm_nt_test(h, P(a), a.size, lda, sA, P(B), B.size, 130, 0, P(C), C.size, ldc, 0, batch,
                                       tm, tn, K, 1.0, beta, lower, P(pr), pr.shape[0], P(X), 2, P(d), n_valid, 0, 0)
    for kw in [dict(K=0), dict(K=192), dict(lda=129), dict(lda=100), dict(sA=1), dict(tm=3, tn=3), dict(tn=1),
               dict(beta=3), dict(batch=0), dict(ldc=200), dict(beta=2, n_valid=0), dict(a=A[:-3])]:
        assert gemm(**kw) != 0, kw
    assert gemm(beta=2, pr=np.array([[99.0, 0, 0, 0]])) != 0
    assert gemm() == 0 and gemm(beta=2) == 0 and gemm(lower=0, tn=1) == 0          # valid calls still run
    D = np.zeros(130 * 384)
    linv, info = np.zeros((2, TILE, TILE)), np.zeros(2, dtype=np.int32)
    potf2 = lambda lda=384, sA=0, batch=1, off=0, a=D: lib.b200gp_potf2_test(h, P(a), a.size, lda, sA, batch, off,
                                                                               P(linv), P(info))
    for kw in [dict(lda=127), dict(batch=0), dict(batch=2, sA=384 * 3), dict(off=-1), dict(off=2 ** 31 - 100),
               dict(a=D[:127 * 384 + 127])]:
        assert potf2(**kw) != 0, kw
    assert potf2() == 0 and potf2(batch=2, sA=64) == 0
