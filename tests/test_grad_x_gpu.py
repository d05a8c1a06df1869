"""GaussianProcess.log_probability_and_grad(y, wrt_X=True) on the GPU: d logp / d X against the LAPACK gradient of
oracle/grad_x_np.py on the native fp64 and the int8-update factorisations; the other gradients bitwise equal to the
plain call's; bitwise reproducibility; non positive-definite input; duplicate points; translation and rotation
invariance; and the full-size benchmark problem against central differences of the device's own log_probability."""

import numpy as np
import pytest

from oracle import grad_x_np
from oracle import tinygp_np as o
from tinygp_b200 import GaussianProcess, _cabi, kernels, transforms

pytestmark = pytest.mark.gpu

CASES = {
    "expsq_const": (lambda m: 1.3 * m.ExpSquared(0.9) + 0.2, 3),
    "exp_matern": (lambda m: m.Exp(1.1) + m.Matern32(0.8, distance=m.L2Distance()) * m.Matern52(1.4), 2),
    "periodic": (lambda m: m.Cosine(2.5) + m.ExpSineSquared(1.7, gamma=0.6) * m.RationalQuadratic(0.9, distance=m.L2Distance(), alpha=1.3), 1),
    "rq_l1": (lambda m: m.RationalQuadratic(1.2, alpha=0.8) + 0.5 * m.ExpSquared(1.4, distance=m.L1Distance()), 1),
    "ard": (lambda m: 1.5 * m.Linear(np.array([0.5, 1.5, 2.0]), m.ExpSquared())
            + m.Subspace(1, m.Exp(0.7)) + m.Subspace([0, 2], m.Cholesky(np.array([0.8, 1.1]), m.Matern52(1.2, distance=m.L2Distance()))), 3),
    "linear0d": (lambda m: m.Cholesky(0.9, m.Linear(0.7, m.Matern32(1.0))) * m.ExpSineSquared(3.0, gamma=0.4), 1),
}


class _P:   # the product's names under the oracle's spelling
    Exp, ExpSquared, Matern32, Matern52 = kernels.Exp, kernels.ExpSquared, kernels.Matern32, kernels.Matern52
    Cosine, ExpSineSquared, RationalQuadratic = kernels.Cosine, kernels.ExpSineSquared, kernels.RationalQuadratic
    L1Distance, L2Distance = kernels.L1Distance, kernels.L2Distance
    Linear, Cholesky, Subspace = transforms.Linear, transforms.Cholesky, transforms.Subspace


def _data(dim, n, seed=3):
    rng = np.random.default_rng(seed)
    side = 3.0 * (n / 300.0) ** (1.0 / dim)
    X = rng.uniform(0, side, n) if dim == 1 else rng.uniform(0, side, (n, dim))
    y = np.sin(2 * (X if dim == 1 else X[:, 0])) + 0.3 * rng.normal(size=n)
    diag = rng.uniform(0.1, 0.3, n)
    return X, y, diag


def _nodes(g):
    yield g
    for a in ("kernel1", "kernel2", "kernel"):
        if isinstance(getattr(g, a, None), kernels.Kernel):
            yield from _nodes(getattr(g, a))


def _same_kernel_grads(ga, gb):
    for a, b in zip(_nodes(ga), _nodes(gb)):
        for f in ("value", "scale", "factor", "gamma", "alpha"):
            va, vb = getattr(a, f, None), getattr(b, f, None)
            if va is not None or vb is not None:
                assert np.array_equal(np.asarray(va), np.asarray(vb)), (type(a).__name__, f, va, vb)


_ORACLE = {}


def _oracle(name, n):
    if (name, n) not in _ORACLE:
        build, dim = CASES[name]
        X, y, diag = _data(dim, n)
        _ORACLE[(name, n)] = grad_x_np.log_probability_grad_x(build(o), X, y, diag, with_scale=True)
    return _ORACLE[(name, n)]


def _check(name, n):
    build, dim = CASES[name]
    X, y, diag = _data(dim, n)
    gp = GaussianProcess(build(_P), X, diag=diag)
    logp, g = gp.log_probability_and_grad(y, wrt_X=True)
    lp0, g0 = gp.log_probability_and_grad(y)
    assert logp == lp0
    _same_kernel_grads(g.kernel, g0.kernel)
    assert np.array_equal(g.diag, g0.diag) and np.array_equal(g.mean, g0.mean)
    lpo, dXo, _, scale = _oracle(name, n)
    assert logp == pytest.approx(lpo, rel=1e-9)
    assert g.X.shape == X.shape
    err = np.abs(g.X - dXo)
    assert np.all(err <= 1e-8 * scale + 1e-300), (name, n, float(np.max(err / (scale + 1e-300))))


@pytest.mark.parametrize("n", [300, 1000, 4099])
@pytest.mark.parametrize("name", list(CASES))
def test_dX_matches_lapack(name, n):
    if n == 4099 and name not in ("expsq_const", "ard", "periodic"):
        pytest.skip("the largest size runs a representative subset")
    _check(name, n)


@pytest.mark.parametrize("n", [300, 1000, 4099])
@pytest.mark.parametrize("name", ["expsq_const", "ard", "periodic"])
def test_dX_matches_lapack_int8_update(name, n):
    ctx = _cabi.get_context()
    ctx.set_option("ozaki_min_n", 0)
    ctx.set_option("nb", 256)
    try:
        _check(name, n)
    finally:
        ctx.reset_options()


def test_bitwise_reproducible():
    X, y, diag = _data(3, 1500)
    gp = GaussianProcess(CASES["ard"][0](_P), X, diag=diag)
    l1, g1 = gp.log_probability_and_grad(y, wrt_X=True)
    l2, g2 = gp.log_probability_and_grad(y, wrt_X=True)
    assert l1 == l2
    assert np.array_equal(g1.X, g2.X) and np.array_equal(g1.diag, g2.diag) and np.array_equal(g1.mean, g2.mean)
    _same_kernel_grads(g1.kernel, g2.kernel)


def test_non_pd_gives_nan():
    X = np.random.default_rng(1).uniform(0, 1, (200, 2))
    gp = GaussianProcess(kernels.ExpSquared(1.0) + 0.3, X, diag=-0.5)
    logp, g = gp.log_probability_and_grad(np.sin(X[:, 0]), wrt_X=True)
    assert logp == -np.inf
    assert np.isnan(g.kernel.kernel1.scale) and np.isnan(g.diag) and np.all(np.isnan(g.mean))
    assert g.X.shape == X.shape and np.all(np.isnan(g.X))


def test_duplicate_points_are_finite():
    X, y, diag = _data(2, 400)
    X[10:20] = X[0]                                   # eleven coincident points
    X[30] = X[31]
    k = kernels.Exp(1.1, distance=kernels.L2Distance()) + kernels.Matern32(0.9) * kernels.ExpSquared(1.5)
    logp, g = GaussianProcess(k, X, diag=diag).log_probability_and_grad(y, wrt_X=True)
    assert np.isfinite(logp) and np.all(np.isfinite(g.X))
    _, dXo, _, scale = grad_x_np.log_probability_grad_x(
        o.Exp(1.1, distance=o.L2Distance()) + o.Matern32(0.9) * o.ExpSquared(1.5), X, y, diag, with_scale=True)
    assert np.all(np.abs(g.X - dXo) <= 1e-8 * scale + 1e-300)


@pytest.mark.parametrize("name", ["expsq_const", "exp_matern", "ard"])
def test_translation_invariance(name):
    build, dim = CASES[name]
    X, y, diag = _data(dim, 2000)
    _, g = GaussianProcess(build(_P), X, diag=diag).log_probability_and_grad(y, wrt_X=True)
    assert np.linalg.norm(g.X.sum(axis=0)) <= 1e-10 * np.sum(np.linalg.norm(g.X, axis=1))


@pytest.mark.parametrize("k", [
    lambda: 1.3 * kernels.ExpSquared(0.9) + 0.2,
    lambda: kernels.Exp(1.2, distance=kernels.L2Distance()) * kernels.RationalQuadratic(1.5, distance=kernels.L2Distance(), alpha=0.8),
    lambda: kernels.Matern52(1.1, distance=kernels.L2Distance()) + kernels.Matern32(0.7, distance=kernels.L2Distance()),
])
def test_rotation_invariance_isotropic_l2(k):
    X, y, diag = _data(3, 2000)
    X = X - X.mean(axis=0)
    _, g = GaussianProcess(k(), X, diag=diag).log_probability_and_grad(y, wrt_X=True)
    M = g.X.T @ X                                      # sum_i dX_i x_i^T
    scale = np.sum(np.linalg.norm(g.X, axis=1) * np.linalg.norm(X, axis=1))
    assert np.max(np.abs(M - M.T)) <= 1e-10 * scale


def test_full_size_directional_derivative():
    """the bench.py dense problem (N = 65536): v . dX for a random unit v against central differences of the device's
    log_probability along v (Richardson-extrapolated from steps h and 2h)"""
    from bench import N_DENSE, make_dense_problem
    X, y, _, _ = make_dense_problem(N_DENSE)
    k = 1.0 * kernels.ExpSquared(1.0)
    logp, g = GaussianProcess(k, X, diag=0.1).log_probability_and_grad(y, wrt_X=True)
    f = lambda Xp: GaussianProcess(k, Xp, diag=0.1).log_probability(y)
    assert logp == pytest.approx(f(X), rel=1e-12)
    v = np.random.default_rng(7).normal(size=X.shape)
    v /= np.linalg.norm(v)
    h = 0.05
    d1 = (f(X + h * v) - f(X - h * v)) / (2 * h)
    d2 = (f(X + 2 * h * v) - f(X - 2 * h * v)) / (4 * h)
    fd = (4 * d1 - d2) / 3
    got = float(np.sum(v * g.X))
    print(f"N={N_DENSE}: v . dX {got:.9e}, central differences {fd:.9e} (h: {d1:.9e}, 2h: {d2:.9e}), "
          f"|dX| {np.linalg.norm(g.X):.6e}")
    assert got == pytest.approx(fd, rel=1e-5)
