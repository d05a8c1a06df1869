"""GaussianProcess.log_probability_and_grad on the GPU: parity with the LAPACK gradient of oracle/grad_np.py on the
native fp64 and the int8-update factorisations, non positive-definite input, bitwise reproducibility, solver state, and
the full-size benchmark problem against central differences of the device's own log_probability."""

import numpy as np
import pytest

from oracle import grad_np
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


def _nodes(g, on):
    yield g, on
    for a in ("kernel1", "kernel2", "kernel"):
        if hasattr(on, a):
            yield from _nodes(getattr(g, a), getattr(on, a))


_ORACLE = {}


def _oracle(name, n):
    if (name, n) not in _ORACLE:
        build, dim = CASES[name]
        X, y, diag = _data(dim, n)
        ok = build(o)
        _ORACLE[(name, n)] = (ok,) + grad_np.log_probability_grad(ok, X, y, diag, with_scale=True)
    return _ORACLE[(name, n)]


def _check(name, n):
    build, dim = CASES[name]
    X, y, diag = _data(dim, n)
    gp = GaussianProcess(build(_P), X, diag=diag)
    logp, g = gp.log_probability_and_grad(y)
    assert logp == pytest.approx(GaussianProcess(build(_P), X, diag=diag).log_probability(y), rel=1e-12)
    ok, lpo, acc, ddiag, alpha, scale = _oracle(name, n)
    assert logp == pytest.approx(lpo, rel=1e-9)
    checked = 0
    for gn, on in _nodes(g.kernel, ok):
        for (nid, field), (_, ref) in acc.items():
            if nid != id(on):
                continue
            got = np.asarray(getattr(gn, field))
            tol = 1e-8 * np.asarray(scale[(nid, field)]) + 1e-300
            assert np.all(np.abs(got - ref) <= tol), (name, n, type(on).__name__, field, got, ref, tol)
            checked += 1
    assert checked == len(acc)
    assert np.all(np.abs(g.diag - ddiag) <= 1e-8 * scale["diag"])
    np.testing.assert_allclose(g.mean, alpha, rtol=1e-9, atol=1e-9 * np.max(np.abs(alpha)))


@pytest.mark.parametrize("n", [300, 1000, 4099])
@pytest.mark.parametrize("name", list(CASES))
def test_grad_matches_lapack(name, n):
    if n == 4099 and name not in ("expsq_const", "ard", "periodic"):
        pytest.skip("the largest size runs a representative subset")
    _check(name, n)


@pytest.mark.parametrize("n", [300, 1000, 4099])
@pytest.mark.parametrize("name", ["expsq_const", "ard", "periodic"])
def test_grad_matches_lapack_int8_update(name, n):
    ctx = _cabi.get_context()
    ctx.set_option("ozaki_min_n", 0)
    ctx.set_option("nb", 256)
    try:
        _check(name, n)
    finally:
        ctx.reset_options()


def test_non_pd_gives_nan_gradients():
    X = np.linspace(0, 1, 200)
    gp = GaussianProcess(kernels.ExpSquared(1.0) + 0.3, X, diag=-0.5)
    logp, g = gp.log_probability_and_grad(np.sin(X))
    assert logp == -np.inf
    assert np.isnan(g.kernel.kernel1.scale) and np.isnan(g.kernel.kernel2.value) and np.isnan(g.diag)
    assert np.all(np.isnan(g.mean))


def test_bitwise_reproducible_and_solver_untouched():
    X, y, diag = _data(3, 1500)
    gp = GaussianProcess(CASES["ard"][0](_P), X, diag=diag)
    Xt = X[:7] + 0.05
    before = gp.predict(y, Xt, return_var=True)
    l1, g1 = gp.log_probability_and_grad(y)
    l2, g2 = gp.log_probability_and_grad(y)
    after = gp.predict(y, Xt, return_var=True)
    assert l1 == l2
    assert np.array_equal(g1.diag, g2.diag) and np.array_equal(g1.mean, g2.mean)
    for a, b in zip(_nodes(g1.kernel, CASES["ard"][0](o)), _nodes(g2.kernel, CASES["ard"][0](o))):
        for f in ("value", "scale", "factor"):
            if getattr(a[0], f, None) is not None:
                assert np.array_equal(getattr(a[0], f), getattr(b[0], f))
    for u, v in zip(before, after):
        assert np.array_equal(u, v)


def test_full_size_against_central_differences():
    """the bench.py dense problem (N = 65536): one call fits in memory and agrees with the device's log_probability"""
    from bench import N_DENSE, make_dense_problem
    X, y, _, _ = make_dense_problem(N_DENSE)
    amp, scale, diag = 1.0, 1.0, 0.1
    logp, g = GaussianProcess(amp * kernels.ExpSquared(scale), X, diag=diag).log_probability_and_grad(y)
    f = lambda a, s, d: GaussianProcess(a * kernels.ExpSquared(s), X, diag=d).log_probability(y)
    assert logp == pytest.approx(f(amp, scale, diag), rel=1e-12)
    h = 1e-4
    fd_amp = (f(amp * (1 + h), scale, diag) - f(amp * (1 - h), scale, diag)) / (2 * h * amp)
    fd_scale = (f(amp, scale * (1 + h), diag) - f(amp, scale * (1 - h), diag)) / (2 * h * scale)
    fd_diag = (f(amp, scale, diag * (1 + h)) - f(amp, scale, diag * (1 - h))) / (2 * h * diag)
    print(f"N={N_DENSE}: d/d amp {g.kernel.kernel1.value:.9e} (fd {fd_amp:.9e}), d/d scale {g.kernel.kernel2.scale:.9e} "
          f"(fd {fd_scale:.9e}), d/d diag {g.diag:.9e} (fd {fd_diag:.9e})")
    assert g.kernel.kernel1.value == pytest.approx(fd_amp, rel=1e-5)
    assert g.kernel.kernel2.scale == pytest.approx(fd_scale, rel=1e-5)
    assert g.diag == pytest.approx(fd_diag, rel=1e-5)
