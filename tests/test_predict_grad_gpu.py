"""GaussianProcess.predict_and_grad on the GPU: d mu / d X_test and d var / d X_test against the LAPACK values of
oracle/predict_grad_np.py (1-, 2-, 3- and 8-D inputs, N up to 2500, M on both sides of the 128-point tile, a predictive
kernel that is one component of a sum); mu bit for bit predict's and var within the rounding of its sum of squares of
predict(return_var=True)'s; blocks of test points (M above the 4096-point block) against single-point and permuted calls;
bitwise reproducibility; test points on training points; a failed factorisation; and N = 16384 against central
differences of the device's own predict, with the native fp64 and the int8 trailing update."""

import numpy as np
import pytest

from oracle import predict_grad_np
from oracle import tinygp_np as o
from tinygp_b200 import GaussianProcess, _cabi, kernels, transforms

pytestmark = pytest.mark.gpu

EPS = np.finfo(np.float64).eps

KERNELS = {
    "expsq_const": (lambda m: 1.3 * m.ExpSquared(0.9) + 0.2, 3),
    "exp_matern": (lambda m: m.Exp(1.1) + m.Matern32(0.8, distance=m.L2Distance()) * m.Matern52(1.4), 2),
    "periodic": (lambda m: m.Cosine(2.5) + m.ExpSineSquared(1.7, gamma=0.6) * m.RationalQuadratic(0.9, distance=m.L2Distance(), alpha=1.3), 1),
    "rq_l1": (lambda m: m.RationalQuadratic(1.2, alpha=0.8) + 0.5 * m.ExpSquared(1.4, distance=m.L1Distance()), 1),
    "ard": (lambda m: 1.5 * m.Linear(np.array([0.5, 1.5, 2.0]), m.ExpSquared())
            + m.Subspace(1, m.Exp(0.7)) + m.Subspace([0, 2], m.Cholesky(np.array([0.8, 1.1]), m.Matern52(1.2, distance=m.L2Distance()))), 3),
    "linear0d": (lambda m: m.Cholesky(0.9, m.Linear(0.7, m.Matern32(1.0))) * m.ExpSineSquared(3.0, gamma=0.4), 1),
    "expsq_8d": (lambda m: 1.2 * m.ExpSquared(2.5) + 0.1, 8),
    "ard_matern_8d": (lambda m: m.Linear(np.linspace(0.3, 1.0, 8), m.Matern52(1.0, distance=m.L2Distance())), 8),
}

# (kernel, N, M)
PARITY = [("expsq_const", 1000, 129), ("exp_matern", 300, 1), ("periodic", 2500, 1000), ("rq_l1", 300, 127),
          ("ard", 2500, 128), ("linear0d", 1000, 1000), ("expsq_8d", 1000, 129), ("ard_matern_8d", 2500, 127),
          ("ard", 300, 1000), ("exp_matern", 1000, 128)]


class _P:   # the product's names under the oracle's spelling
    Exp, ExpSquared, Matern32, Matern52 = kernels.Exp, kernels.ExpSquared, kernels.Matern32, kernels.Matern52
    Cosine, ExpSineSquared, RationalQuadratic = kernels.Cosine, kernels.ExpSineSquared, kernels.RationalQuadratic
    L1Distance, L2Distance = kernels.L1Distance, kernels.L2Distance
    Linear, Cholesky, Subspace = transforms.Linear, transforms.Cholesky, transforms.Subspace


def _data(dim, n, m, seed=3):
    rng = np.random.default_rng(seed)
    side = 3.0 * (n / 300.0) ** (1.0 / dim)
    X = rng.uniform(0, side, n) if dim == 1 else rng.uniform(0, side, (n, dim))
    y = np.sin(2 * (X if dim == 1 else X[:, 0])) + 0.3 * rng.normal(size=n)
    diag = rng.uniform(0.1, 0.3, n)
    Xt = rng.uniform(-0.2 * side, 1.2 * side, m if dim == 1 else (m, dim))
    return X, y, diag, Xt


def _check_against_oracle(gp, ok, X, y, diag, Xt, pred=None, opred=None, include_mean=True):
    mu, var, g = gp.predict_and_grad(y, Xt, kernel=pred, include_mean=include_mean, return_var=True)
    mu1, g1 = gp.predict_and_grad(y, Xt, kernel=pred, include_mean=include_mean)
    assert np.array_equal(mu, mu1) and np.array_equal(g.mean, g1.mean) and g1.var is None
    assert g.mean.shape == Xt.shape and g.var.shape == Xt.shape and var.shape == (Xt.shape[0],)
    mo, vo, dmo, dvo, sm, sv = predict_grad_np.predict_and_grad(ok, X, y, diag, Xt, pred_kernel=opred, with_scale=True)
    np.testing.assert_allclose(mu, mo, rtol=1e-8, atol=1e-9 * np.max(np.abs(mo)))
    np.testing.assert_allclose(var, vo, rtol=0, atol=1e-9 * np.max(np.abs(vo)))
    for got, ref, scale in ((g.mean, dmo, sm), (g.var, dvo, sv)):
        err = np.abs(got - ref)
        assert np.all(err <= 1e-8 * scale + 1e-300), float(np.max(err / (scale + 1e-300)))
    return mu, var, g


@pytest.mark.parametrize("name,n,m", PARITY)
def test_matches_lapack(name, n, m):
    build, dim = KERNELS[name]
    X, y, diag, Xt = _data(dim, n, m)
    _check_against_oracle(GaussianProcess(build(_P), X, diag=diag), build(o), X, y, diag, Xt)


@pytest.mark.parametrize("n,m", [(1000, 1000), (2500, 129)])
def test_component_kernel_matches_lapack(n, m):
    X, y, diag, Xt = _data(2, n, m)
    # L2 distances: a squared-exponential or Matern leaf on the L1 distance need not be positive definite in 2-D
    part, opart = kernels.Matern52(1.4, distance=kernels.L2Distance()), o.Matern52(1.4, distance=o.L2Distance())
    gp = GaussianProcess(kernels.ExpSquared(0.8, distance=kernels.L2Distance()) * kernels.Exp(2.0) + part, X, diag=diag)
    _check_against_oracle(gp, o.ExpSquared(0.8, distance=o.L2Distance()) * o.Exp(2.0) + opart, X, y, diag, Xt, pred=part,
                          opred=opart, include_mean=False)


@pytest.mark.parametrize("name,n,m", [("expsq_const", 2500, 1000), ("ard", 1000, 129), ("periodic", 300, 127)])
def test_against_predict(name, n, m):
    """mu is predict's bit for bit; var and predict(return_var=True)'s variance sum the same squares |L^-1 k(X, x*)|^2
    (bitwise the same forward substitution) in different orders.  Each order's rounding error is at most (N - 1) eps
    times the sum, which is at most k(x*, x*) + sqrt(eps), so they differ by at most 2 N eps (k(x*, x*) + sqrt(eps))."""
    build, dim = KERNELS[name]
    X, y, diag, Xt = _data(dim, n, m)
    gp = GaussianProcess(build(_P), X, diag=diag, mean=0.3)
    mu, var, _ = gp.predict_and_grad(y, Xt, return_var=True)
    assert np.array_equal(mu, gp.predict(y, Xt))
    mu_p, var_p = gp.predict(y, Xt, return_var=True)
    assert np.array_equal(mu, mu_p)
    kss = build(_P)(Xt[:1])[0] + np.sqrt(EPS)
    err = np.abs(var - var_p)
    print(f"{name} N={n} M={m}: max |var - predict var| = {np.max(err) / (EPS * kss):.2f} eps k**")
    assert np.all(err <= 2 * n * EPS * kss)


def test_blocks_and_permutation():
    """M = 9000 (three blocks of at most 4096): every point's outputs are bitwise those of the same point alone, or in a
    permuted call, and bitwise equal run to run"""
    build, dim = KERNELS["ard"]
    X, y, diag, Xt = _data(dim, 400, 9000)
    gp = GaussianProcess(build(_P), X, diag=diag)
    mu, var, g = gp.predict_and_grad(y, Xt, return_var=True)
    mu2, var2, g2 = gp.predict_and_grad(y, Xt, return_var=True)
    assert np.array_equal(mu, mu2) and np.array_equal(var, var2)
    assert np.array_equal(g.mean, g2.mean) and np.array_equal(g.var, g2.var)
    perm = np.random.default_rng(5).permutation(9000)
    mup, varp, gp_ = gp.predict_and_grad(y, Xt[perm], return_var=True)
    assert np.array_equal(varp, var[perm])
    assert np.array_equal(gp_.mean, g.mean[perm]) and np.array_equal(gp_.var, g.var[perm])
    for i in [0, 127, 128, 4095, 4096, 5000, 8191, 8192, 8999]:
        _, v1, g1 = gp.predict_and_grad(y, Xt[i:i + 1], return_var=True)
        assert v1[0] == var[i] and np.array_equal(g1.mean[0], g.mean[i]) and np.array_equal(g1.var[0], g.var[i]), i
    _, vo, dmo, dvo, sm, sv = predict_grad_np.predict_and_grad(build(o), X, y, diag, Xt, with_scale=True)
    assert np.all(np.abs(g.mean - dmo) <= 1e-8 * sm + 1e-300)
    assert np.all(np.abs(g.var - dvo) <= 1e-8 * sv + 1e-300)


def test_test_points_on_training_points():
    X, y, diag, Xt = _data(2, 500, 300)
    Xt[::3] = X[:100]
    k = kernels.Exp(1.1, distance=kernels.L2Distance()) + kernels.Matern32(0.9) * kernels.ExpSquared(1.5)
    ko = o.Exp(1.1, distance=o.L2Distance()) + o.Matern32(0.9) * o.ExpSquared(1.5)
    _, var, g = GaussianProcess(k, X, diag=diag).predict_and_grad(y, Xt, return_var=True)
    assert np.all(np.isfinite(var)) and np.all(np.isfinite(g.mean)) and np.all(np.isfinite(g.var))
    _, _, dmo, dvo, sm, sv = predict_grad_np.predict_and_grad(ko, X, y, diag, Xt, with_scale=True)
    assert np.all(np.abs(g.mean - dmo) <= 1e-8 * sm + 1e-300)
    assert np.all(np.abs(g.var - dvo) <= 1e-8 * sv + 1e-300)


def test_failed_factorisation_gives_nan():
    X = np.random.default_rng(1).uniform(0, 1, (200, 2))
    gp = GaussianProcess(kernels.ExpSquared(1.0) + 0.3, X, diag=-0.5)
    mu, var, g = gp.predict_and_grad(np.sin(X[:, 0]), X[:7] + 0.01, return_var=True)
    assert gp.solver.info > 0
    assert g.mean.shape == (7, 2) and g.var.shape == (7, 2) and var.shape == (7,)
    assert np.all(np.isnan(g.mean)) and np.all(np.isnan(g.var)) and np.all(np.isnan(var))


def _large_n_check():
    """N = 16384, 3-D ExpSquared: d mu and d var at a few points against Richardson-extrapolated central differences of
    the device's own predict(return_var=True)"""
    X, y, _, Xt = _data(3, 16384, 4, seed=8)
    k = 1.0 * kernels.ExpSquared(1.0)
    gp = GaussianProcess(k, X, diag=0.1)
    mu, var, g = gp.predict_and_grad(y, Xt, return_var=True)
    f = lambda Z: gp.predict(y, Z, return_var=True)
    h = 1e-3
    for i in range(Xt.shape[0]):
        for c in range(3):
            e = np.zeros((1, 3))
            e[0, c] = 1.0
            x = Xt[i:i + 1]
            (mu_p1, v_p1), (mu_m1, v_m1) = f(x + h * e), f(x - h * e)
            (mu_p2, v_p2), (mu_m2, v_m2) = f(x + 2 * h * e), f(x - 2 * h * e)
            fd_mu = (4 * (mu_p1 - mu_m1) / (2 * h) - (mu_p2 - mu_m2) / (4 * h)) / 3
            fd_var = (4 * (v_p1 - v_m1) / (2 * h) - (v_p2 - v_m2) / (4 * h)) / 3
            gm, gv = g.mean[i, c], g.var[i, c]
            assert gm == pytest.approx(fd_mu[0], rel=1e-5, abs=1e-7 * np.max(np.abs(g.mean))), (i, c)
            assert gv == pytest.approx(fd_var[0], rel=1e-5, abs=1e-7 * np.max(np.abs(g.var))), (i, c)


def test_large_n_against_central_differences():
    _large_n_check()


def test_large_n_int8_update_against_central_differences():
    """the same with the int8 fixed-point trailing update, which is not the default at N = 16384"""
    ctx = _cabi.get_context()
    before = {key: ctx.get_option(key) for key in ("ozaki_slices", "ozaki_min_n")}
    ctx.set_option("ozaki_slices", 7)
    ctx.set_option("ozaki_min_n", 0)
    try:
        _large_n_check()
    finally:
        for key, value in before.items():
            ctx.set_option(key, value)
