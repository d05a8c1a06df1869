"""The gradient's triangular tile kernel (grad.cu tri_gemm_kernel, through b200gp_grad_tiles_test) against the NumPy
restatement of its schedules in oracle/grad_tiles_np.py, exactly.

Operands are small integers in [-4, 4], so every tile product and every weighted sum is exact in fp64 in any summation
order: results are compared bitwise, whatever order a mainloop uses.  Every operand block a tile must not read (outside
its K range, and the diagonal blocks that come from the separate diagonal-block array) holds NaN, so a read outside a
range shows up as NaN; the inverse step's C starts as a sentinel that every element outside the written tiles must keep.
The coordinate-gradient partials involve the kernel's derivatives, so they are compared with the closed forms of
oracle/grad_x_np.py within 1e-13 of the sum of the magnitudes of their terms."""

import numpy as np
import pytest

from oracle import grad_tiles_np as gt
from oracle import tinygp_np as o
from tinygp_b200 import _cabi, kernels, transforms

pytestmark = pytest.mark.gpu

TILE = gt.TILE
SENTINEL = -1234.5
TRMM, CONTRACT = 0, 1


class _P:   # the product's names under the oracle's spelling
    Exp, ExpSquared, Matern32, Matern52 = kernels.Exp, kernels.ExpSquared, kernels.Matern32, kernels.Matern52
    RationalQuadratic, Constant = kernels.RationalQuadratic, kernels.Constant
    L1Distance, L2Distance = kernels.L1Distance, kernels.L2Distance
    Linear, Cholesky, Subspace = transforms.Linear, transforms.Cholesky, transforms.Subspace


def _ints(rng, shape):
    return rng.integers(-4, 5, shape).astype(np.float64)


def _bits(a):
    return np.ascontiguousarray(a).view(np.uint64)


def _run_trmm(T, j, A, diagA, B, C):
    ctx = _cabi.get_context()
    C = C.copy()
    ctx.check(ctx.lib.b200gp_grad_tiles_test(ctx.handle, TRMM, T, j, _cabi.ptr(A), _cabi.ptr(diagA), _cabi.ptr(B),
                                             _cabi.ptr(C), None, 0, None, 0, 0, None, None, None, None, None))
    return C


def _run_contract(T, U, diagU, prog, X, alpha, dx):
    ctx = _cabi.get_context()
    n, nd = X.shape
    ntiles = T * (T + 1) // 2
    wdiag, partial = np.full(n, np.nan), np.full((ntiles, 16), np.nan)
    dxpart = np.full((ntiles, 2, nd, TILE), np.nan) if dx else None
    dX = np.full((n, nd), np.nan) if dx else None
    p = lambda a: None if a is None else _cabi.ptr(a)
    ctx.check(ctx.lib.b200gp_grad_tiles_test(ctx.handle, CONTRACT, T, 0, _cabi.ptr(U), _cabi.ptr(diagU), None, None,
                                             _cabi.ptr(prog), prog.shape[0], _cabi.ptr(X), n, nd, _cabi.ptr(alpha),
                                             _cabi.ptr(wdiag), _cabi.ptr(partial), p(dxpart), p(dX)))
    return wdiag, partial, dxpart, dX


def _trmm_operands(T, j, seed):
    """A, diagA, B with NaN in every block the step must not read, and C all sentinel"""
    rng = np.random.default_rng(seed)
    np_ = T * TILE
    A = np.full((np_, np_), np.nan)
    for ti in range(j + 1, T):
        A[ti * TILE:(ti + 1) * TILE, (j + 1) * TILE:ti * TILE] = _ints(rng, (TILE, (ti - j - 1) * TILE))
    diagA = np.full((T, TILE, TILE), np.nan)
    diagA[j + 1:] = _ints(rng, (T - j - 1, TILE, TILE))
    B = np.full((TILE, np_), np.nan)
    B[:, (j + 1) * TILE:] = _ints(rng, (TILE, np_ - (j + 1) * TILE))
    return A, diagA, B, np.full((np_, np_), SENTINEL)


TRMM_STEPS = [(T, j) for T in (2, 3, 9) for j in range(T - 1)] + [(17, j) for j in (0, 1, 7, 14, 15)]


@pytest.mark.parametrize("T,j", TRMM_STEPS)
def test_inverse_step_tiles_exact(T, j):
    A, diagA, B, C = _trmm_operands(T, j, seed=100 * T + j)
    got = _run_trmm(T, j, A, diagA, B, C)
    ref = gt.trmm(C, A, diagA, B, T, j)
    written = np.zeros(got.shape, dtype=bool)
    written[(j + 1) * TILE:, j * TILE:(j + 1) * TILE] = True
    assert np.all(got[~written] == SENTINEL), "the step wrote outside block column j below the diagonal"
    for ti in range(j + 1, T):
        r = slice(ti * TILE, (ti + 1) * TILE)
        g, e = got[r, j * TILE:(j + 1) * TILE], ref[r, j * TILE:(j + 1) * TILE]
        assert np.array_equal(_bits(g), _bits(e)), (T, j, ti, int(np.sum(np.isnan(g))), float(np.nanmax(np.abs(g - e))))


def _contract_operands(T, n, nd, seed):
    """U (upper blocks only; NaN below and on the diagonal), its diagonal blocks, integer alpha, X in [0, 3]^nd"""
    rng = np.random.default_rng(seed)
    np_ = T * TILE
    U = np.full((np_, np_), np.nan)
    for r in range(T - 1):
        U[r * TILE:(r + 1) * TILE, (r + 1) * TILE:] = _ints(rng, (TILE, np_ - (r + 1) * TILE))
    diagU = _ints(rng, (T, TILE, TILE))
    alpha = rng.integers(-3, 4, n).astype(np.float64)
    X = rng.uniform(0.0, 3.0, (n, nd))
    return U, diagU, alpha, X


def _program(build, X):
    """(program, device coordinates, slot of the trailing Constant) of build(kernels) + Constant(0.25)"""
    k = build(_P) + _P.Constant(0.25)
    prog, x, leaves, owners = k.lower_for_grad(X)
    nslot = sum(2 if f1 is not None else 1 for _, _, f1 in leaves)
    assert leaves[-1][0] is k.kernel2 and nslot + sum(len(r) for r in owners) <= 16
    return prog, x, nslot - 1


def _check_contract(T, n, build, nd, seed, check_dx=True):
    U, diagU, alpha, X = _contract_operands(T, n, nd, seed)
    prog, x, cslot = _program(build, X)
    assert np.array_equal(x, X)
    W = gt.contract(U, diagU, T)
    okern = build(o) + o.Constant(0.25)
    wdiag_ref, wsum, dx = gt.epilogue(W, alpha, n, T, okern if check_dx else None, X if check_dx else None)

    wdiag, partial, _, _ = _run_contract(T, U, diagU, prog, x, alpha, dx=False)
    assert np.array_equal(_bits(wdiag), _bits(wdiag_ref)), ("wdiag", T, n)
    assert np.array_equal(_bits(partial[:, cslot]), _bits(wsum)), ("Constant partials", T, n, partial[:, cslot] - wsum)

    wdiag_x, partial_x, dxpart, dX = _run_contract(T, U, diagU, prog, x, alpha, dx=True)
    assert np.array_equal(_bits(wdiag_x), _bits(wdiag)), "wdiag differs between the plain and the dX kernel"
    assert np.array_equal(_bits(partial_x), _bits(partial)), "slot partials differ between the plain and the dX kernel"
    if not check_dx:
        return
    rows, cols, rows_s, cols_s, dX_ref, dX_s = dx
    for what, got, ref, sc in (("row sums", dxpart[:, 0], rows, rows_s), ("column sums", dxpart[:, 1], cols, cols_s),
                               ("dX", dX, dX_ref, dX_s)):
        err = np.abs(got - ref)
        bad = ~(err <= 1e-13 * sc)
        assert not np.any(bad), (what, T, n, nd, np.argwhere(bad)[:5].tolist(), float(np.max(err - 1e-13 * sc)))


def _ard3(m):
    return (1.5 * m.Linear(np.array([0.5, 1.5, 2.0]), m.ExpSquared())
            + m.Subspace(1, m.Exp(0.7))
            + m.Subspace([0, 2], m.Cholesky(np.array([0.8, 1.1]), m.Matern52(1.2, distance=m.L2Distance()))))


CONTRACT_SHAPES = [(T, n) for T in (1, 2, 5, 17) for n in sorted({128 * T, 128 * T - 37, 128 * (T - 1) + 1})]


@pytest.mark.parametrize("T,n", CONTRACT_SHAPES)
def test_w_tiles_exact(T, n):
    _check_contract(T, n, _ard3, 3, seed=T * 1000 + n)


def _full_d(nd):
    """an ARD Linear over all nd axes plus a Subspace on the last one"""
    scales = np.linspace(0.4, 1.6, nd)
    return lambda m: (1.2 * m.Linear(scales, m.ExpSquared())
                      + m.Subspace(nd - 1, m.Matern32(1.1, distance=m.L2Distance())))


@pytest.mark.parametrize("T,n", [(2, 219), (3, 347)])
@pytest.mark.parametrize("nd", [1, 2, 3, 4, 7, 8])
def test_dx_partials_every_ndim(nd, T, n):
    _check_contract(T, n, _full_d(nd), nd, seed=nd * 10 + T)


def test_sizes_are_checked_before_launch():
    ctx = _cabi.get_context()
    lib, h = ctx.lib, ctx.handle
    A = np.zeros((256, 256))
    D = np.zeros((2, TILE, TILE))
    B = np.zeros((TILE, 256))
    C = np.zeros((256, 256))
    prog, _, _ = _program(_ard3, np.zeros((10, 3)))
    X, alpha = np.zeros((256, 8)), np.zeros(256)
    out = [np.zeros(256), np.zeros((3, 16)), np.zeros((3, 2, 8, TILE)), np.zeros((256, 8))]
    P = _cabi.ptr
    trmm = lambda T, j, mode=TRMM: lib.b200gp_grad_tiles_test(h, mode, T, j, P(A), P(D), P(B), P(C), None, 0, None, 0,
                                                              0, None, None, None, None, None)
    for T, j in [(0, 0), (1, 0), (2, -1), (2, 1)]:
        assert trmm(T, j) != 0, (T, j)
    assert trmm(2, 0, mode=2) != 0
    contract = lambda n, nd, pr=prog: lib.b200gp_grad_tiles_test(
        h, CONTRACT, 2, 0, P(A), P(D), None, None, P(pr), pr.shape[0], P(X), n, nd, P(alpha), P(out[0]), P(out[1]),
        P(out[2]), P(out[3]))
    for n, nd in [(0, 3), (257, 3), (10, 0), (10, 9), (10, 2)]:     # nd = 2: the program's transforms are 3-D
        assert contract(n, nd) != 0, (n, nd)
    # one differentiable scalar too many
    rq = lambda s: _P.RationalQuadratic(s, alpha=0.8)
    k17 = _ard3(_P) + rq(1.0) * rq(2.0) * rq(3.0) + _P.Exp(1.5)
    seventeen, _, leaves, owners = k17.lower_for_grad(np.zeros((10, 3)))
    assert sum(2 if f1 is not None else 1 for _, _, f1 in leaves) + sum(len(r) for r in owners) == 17
    assert contract(10, 3, pr=seventeen) != 0
    assert b"more than 16" in lib.b200gp_last_error(h)
    assert contract(256, 3) == 0 and trmm(2, 0) == 0                   # and valid calls still run
