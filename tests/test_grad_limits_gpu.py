"""GaussianProcess.log_probability_and_grad at the limits it advertises, with and without wrt_X, against the LAPACK
gradients of oracle/grad_np.py and oracle/grad_x_np.py at the tolerances of test_grad_gpu.py / test_grad_x_gpu.py
(1e-8 of each value's scale): 4 to 8 input dimensions (the coordinate gradient's cap), exactly 16 differentiable scalars
(the slot cap) and the refusal of a 17th by the library itself, sizes around one and two 128-tiles, and the int8
trailing update at the library's own panel width and digit-plane count."""

import numpy as np
import pytest
from ctypes import byref, c_double

from oracle import grad_np, grad_x_np
from oracle import tinygp_np as o
from tinygp_b200 import GaussianProcess, _cabi, kernels, transforms

pytestmark = pytest.mark.gpu


class _P:   # the product's names under the oracle's spelling
    Exp, ExpSquared, Matern32, Matern52 = kernels.Exp, kernels.ExpSquared, kernels.Matern32, kernels.Matern52
    ExpSineSquared, RationalQuadratic = kernels.ExpSineSquared, kernels.RationalQuadratic
    L1Distance, L2Distance = kernels.L1Distance, kernels.L2Distance
    Linear, Cholesky, Subspace = transforms.Linear, transforms.Cholesky, transforms.Subspace


def _ard(D):
    s = np.linspace(0.5, 1.5, D)
    return lambda m: 1.3 * m.Linear(s, m.ExpSquared()) + m.Subspace(D - 1, m.Exp(0.7))


def _chol(D):
    f = np.linspace(1.4, 0.7, D)
    return lambda m: (m.Cholesky(f, m.Matern52(1.2, distance=m.L2Distance()))
                      * m.RationalQuadratic(2.5, distance=m.L2Distance(), alpha=0.9))


def _mix(D):
    s = np.linspace(0.6, 1.2, D)
    return lambda m: (m.Linear(s, m.ExpSquared(1.1)) * m.Subspace(D - 1, m.Cholesky(0.8, m.Matern32(1.0)))
                      + m.Subspace(0, m.Exp(1.5, distance=m.L2Distance())) + 0.2)


def _sixteen(m):
    """exactly 16 differentiable scalars: 8 leaf / constant parameters, 2 gamma / alpha and 6 transform rows"""
    return (1.3 * m.Linear(np.array([0.6, 1.1, 0.9]), m.ExpSquared())
            + m.Subspace(0, m.ExpSineSquared(1.7, gamma=0.6)) * m.RationalQuadratic(0.9, distance=m.L2Distance(), alpha=1.3)
            + m.Subspace([0, 2], m.Cholesky(np.array([0.8, 1.1]), m.Matern52(1.2, distance=m.L2Distance())))
            + m.Matern32(1.4, distance=m.L2Distance()) * m.Exp(2.0) + 0.3)


CASES = {f"{name}{D}": (make(D), D) for D in (4, 5, 8) for name, make in (("ard", _ard), ("chol", _chol), ("mix", _mix))}
CASES["sixteen"] = (_sixteen, 3)
CASES["expsq_const"] = (lambda m: 1.3 * m.ExpSquared(0.9) + 0.2, 3)
CASES["ard3"] = (lambda m: 1.5 * m.Linear(np.array([0.5, 1.5, 2.0]), m.ExpSquared())
                 + m.Subspace(1, m.Exp(0.7))
                 + m.Subspace([0, 2], m.Cholesky(np.array([0.8, 1.1]), m.Matern52(1.2, distance=m.L2Distance()))), 3)


def _data(dim, n, seed=3):
    rng = np.random.default_rng(seed)
    side = 3.0 * (n / 300.0) ** (1.0 / dim)
    X = rng.uniform(0, side, (n, dim))
    y = np.sin(2 * X[:, 0]) + 0.3 * rng.normal(size=n)
    diag = rng.uniform(0.1, 0.3, n)
    return X, y, diag


def _nodes(g, on):
    yield g, on
    for a in ("kernel1", "kernel2", "kernel"):
        if hasattr(on, a):
            yield from _nodes(getattr(g, a), getattr(on, a))


def _nslot(k, X):
    _, _, leaves, owners = k.lower_for_grad(X)
    return sum(2 if f1 is not None else 1 for _, _, f1 in leaves) + sum(len(r) for r in owners)


_ORACLE = {}


def _oracle(name, n):
    if (name, n) not in _ORACLE:
        build, dim = CASES[name]
        X, y, diag = _data(dim, n)
        ok = build(o)
        _ORACLE[(name, n)] = ((ok,) + grad_np.log_probability_grad(ok, X, y, diag, with_scale=True),
                              grad_x_np.log_probability_grad_x(build(o), X, y, diag, with_scale=True))
    return _ORACLE[(name, n)]


def _check(name, n, wrt_X):
    build, dim = CASES[name]
    X, y, diag = _data(dim, n)
    gp = GaussianProcess(build(_P), X, diag=diag)
    logp, g = gp.log_probability_and_grad(y, wrt_X=wrt_X)
    (ok, lpo, acc, ddiag, alpha, scale), (_, dXo, _, xscale) = _oracle(name, n)
    assert logp == pytest.approx(lpo, rel=1e-9)
    checked = 0
    for gn, on in _nodes(g.kernel, ok):
        for (nid, field), (_, ref) in acc.items():
            if nid != id(on):
                continue
            got = np.asarray(getattr(gn, field))
            tol = 1e-8 * np.asarray(scale[(nid, field)]) + 1e-300
            assert np.all(np.abs(got - ref) <= tol), (name, n, wrt_X, type(on).__name__, field, got, ref, tol)
            checked += 1
    assert checked == len(acc)
    assert np.all(np.abs(g.diag - ddiag) <= 1e-8 * scale["diag"])
    np.testing.assert_allclose(g.mean, alpha, rtol=1e-9, atol=1e-9 * np.max(np.abs(alpha)))
    if wrt_X:
        assert g.X.shape == X.shape
        err = np.abs(g.X - dXo)
        assert np.all(err <= 1e-8 * xscale + 1e-300), (name, n, float(np.max(err / (xscale + 1e-300))))
    return g


@pytest.mark.parametrize("wrt_X", [False, True])
@pytest.mark.parametrize("n", [300, 1000])
@pytest.mark.parametrize("name", [c for c in CASES if c[-1] in "458"])
def test_four_to_eight_dims(name, n, wrt_X):
    _check(name, n, wrt_X)


@pytest.mark.parametrize("wrt_X", [False, True])
@pytest.mark.parametrize("n", [300, 1000])
def test_sixteen_differentiable_scalars(n, wrt_X):
    X, _, _ = _data(3, n)
    assert _nslot(_sixteen(_P), X) == 16
    _check("sixteen", n, wrt_X)


@pytest.mark.parametrize("entry", ["b200gp_dense_log_probability_grad", "b200gp_dense_log_probability_grad_x"])
def test_seventeenth_scalar_refused_by_the_library(entry):
    X, y, diag = _data(3, 300)
    k = _sixteen(_P) + kernels.Matern52(2.0)
    assert _nslot(k, X) == 17
    with pytest.raises(NotImplementedError, match="at most 16"):
        GaussianProcess(k, X, diag=diag).log_probability_and_grad(y)
    ctx = _cabi.get_context()
    prog, x = k.lower_for(X)
    logp = c_double()
    dprog, dmetric = np.zeros_like(prog), np.zeros((3, 8))
    ddiag, alpha, dX = np.empty(300), np.empty(300), np.empty((300, 3))
    args = [ctx.handle, _cabi.ptr(prog), prog.shape[0], _cabi.ptr(x), 300, 3, _cabi.ptr(diag), _cabi.ptr(y), byref(logp),
            _cabi.ptr(dprog), _cabi.ptr(dmetric), _cabi.ptr(ddiag), _cabi.ptr(alpha)]
    if entry.endswith("_x"):
        args.append(_cabi.ptr(dX))
    assert getattr(ctx.lib, entry)(*args) != 0
    assert b"more than 16" in ctx.lib.b200gp_last_error(ctx.handle)


@pytest.mark.parametrize("wrt_X", [False, True])
@pytest.mark.parametrize("n", [1, 2, 127, 128, 129, 256, 257])
def test_tile_edges(n, wrt_X):
    g = _check("ard3", n, wrt_X)
    if wrt_X and n == 1:
        assert np.array_equal(g.X, np.zeros((1, 3)))


@pytest.mark.parametrize("wrt_X", [False, True])
@pytest.mark.parametrize("name", ["expsq_const", "ard3"])
def test_int8_update_at_library_defaults(name, wrt_X):
    """the int8 trailing update forced on, at the default panel width (nb = 1024) and digit planes (7)"""
    ctx = _cabi.get_context()
    assert ctx.get_option("nb") == 1024 and ctx.get_option("ozaki_slices") == 7
    ctx.set_option("ozaki_min_n", 0)
    ctx.set_option("profile", 1)
    ctx.profile(reset=True)
    try:
        _check(name, 4099, wrt_X)
        assert ctx.profile()["i8_ops"] > 0
    finally:
        ctx.reset_options()
