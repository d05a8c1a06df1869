"""oracle/predict_grad_np.py (predictive mean and variance and their gradients in the test inputs, with LAPACK and
closed-form kernel gradients) against the oracle GP's own predict and against central differences of it with respect to
single test coordinates: 1-, 2- and 3-D inputs, L1 and L2, an ARD Linear, Subspace, sums and products, a predictive
kernel that is one component of a sum, and test points that coincide with training points."""

import numpy as np
import pytest

from oracle import predict_grad_np
from oracle import tinygp_np as o

CASES = {
    "expsq_const_1d": (lambda: 1.3 * o.ExpSquared(0.9) + 0.2, 1),
    "exp_l1_matern_l2_2d": (lambda: o.Exp(1.1) + o.Matern32(0.8, distance=o.L2Distance()) * o.Matern52(1.4), 2),
    "periodic_rq_1d": (lambda: o.Cosine(2.5) + o.ExpSineSquared(1.7, gamma=0.6)
                       * o.RationalQuadratic(0.9, distance=o.L2Distance(), alpha=1.3), 1),
    "ard_linear_3d": (lambda: 1.5 * o.Linear(np.array([0.5, 1.5, 2.0]), o.ExpSquared()), 3),
    "subspace_sum_product_3d": (lambda: o.Subspace(1, o.Exp(0.7)) * o.Matern32(1.6)
                                + o.Subspace([0, 2], o.Cholesky(np.array([0.8, 1.1]), o.Matern52(1.2, distance=o.L2Distance()))),
                                3),
}


def _data(dim, n=25, m=6, seed=13):
    rng = np.random.default_rng(seed)
    X = rng.uniform(0, 3, n) if dim == 1 else rng.uniform(0, 3, (n, dim))
    y = np.sin(2 * (X if dim == 1 else X[:, 0])) + 0.3 * rng.normal(size=n)
    Xt = rng.uniform(-0.5, 3.5, m) if dim == 1 else rng.uniform(-0.5, 3.5, (m, dim))
    return X, y, rng.uniform(0.1, 0.3, n), Xt


def _check(k, X, y, diag, Xt, pred_kernel=None):
    mu, var, dmu, dvar = predict_grad_np.predict_and_grad(k, X, y, diag, Xt, mean=0.1, pred_kernel=pred_kernel)
    gp = o.GaussianProcess(k, X, diag=diag, mean=0.1)
    f = lambda Z: gp.predict(y, Z, kernel=pred_kernel, return_var=True)
    mu0, var0 = f(Xt)
    np.testing.assert_allclose(mu, mu0, rtol=1e-12, atol=1e-12)
    np.testing.assert_allclose(var, var0, rtol=1e-9, atol=1e-12)
    assert dmu.shape == Xt.shape and dvar.shape == Xt.shape
    h = 1e-6
    for idx in np.ndindex(Xt.shape):
        up, dn = Xt.copy(), Xt.copy()
        up[idx] += h
        dn[idx] -= h
        (mu_u, var_u), (mu_d, var_d) = f(up), f(dn)
        i = idx[0]
        assert dmu[idx] == pytest.approx((mu_u[i] - mu_d[i]) / (2 * h), rel=1e-6, abs=1e-7), idx
        assert dvar[idx] == pytest.approx((var_u[i] - var_d[i]) / (2 * h), rel=1e-5, abs=1e-7), idx


@pytest.mark.parametrize("name", list(CASES))
def test_matches_predict_and_central_differences(name):
    build, dim = CASES[name]
    X, y, diag, Xt = _data(dim)
    _check(build(), X, y, diag, Xt)


def test_component_kernel():
    X, y, diag, Xt = _data(2)
    part = o.Matern52(1.4)
    _check(o.ExpSquared(0.8) + part, X, y, diag, Xt, pred_kernel=part)


def test_coincident_points_are_finite():
    X, y, diag, Xt = _data(3)
    Xt[1] = X[4]
    k = o.Exp(1.1, distance=o.L2Distance()) + o.Matern32(0.9)
    out = predict_grad_np.predict_and_grad(k, X, y, diag, Xt, with_scale=True)
    assert all(np.all(np.isfinite(a)) for a in out)
