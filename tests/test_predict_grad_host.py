"""GaussianProcess.predict_and_grad through the host layer without a GPU: a stand-in for b200gp_dense_predict_grad (dense
algebra on the mock solver's factor, grad_1 k by central differences of the NumPy restatement of the kernel-program
interpreter) checks the marshalling, the (M,) and (M, D) shapes against oracle/predict_grad_np.py, a predictive kernel
that is one component of a sum, include_mean and a callable mean, that mu is predict's bit for bit, that the solver's
own factor is used (no second dense_create), NaN on a failed factorisation, and every refused case."""

from ctypes import c_void_p

import numpy as np
import pytest
import scipy.linalg as sla

from hostmock import MockLib, _addr, arr, kmat, parse_program
from oracle import predict_grad_np
from oracle import tinygp_np as o
from test_grad_host import REFUSED
from tinygp_b200 import GaussianProcess, _cabi, kernels, transforms
from tinygp_b200.gp import PredictionGrad


class PredictGradMockLib(MockLib):
    def b200gp_dense_predict_grad(self, h, prog, n_rows, Xtest, m, alpha, dmean, diag_test, var, dvar):
        self.calls.append("dense_predict_grad")
        d = self._get(h)
        n, nd = d.X.shape
        P = parse_program(prog, n_rows, nd)
        xt, a = arr(Xtest, (m, nd)).copy(), arr(alpha, (n,)).copy()
        with_var = _addr(diag_test) != 0
        if not np.all(np.isfinite(d.L)):
            arr(dmean, (m, nd))[:] = np.nan
            if with_var:
                arr(var, (m,))[:] = np.nan
                arr(dvar, (m, nd))[:] = np.nan
            return 0
        h_ = 1e-6
        G = np.empty((m, n, nd))                   # grad_1 k(x*_m, x_j)
        for c in range(nd):
            up, dn = xt.copy(), xt.copy()
            up[:, c] += h_
            dn[:, c] -= h_
            G[:, :, c] = (kmat(P, up, d.X) - kmat(P, dn, d.X)) / (2 * h_)
        arr(dmean, (m, nd))[:] = np.einsum("mjc,j->mc", G, a)
        if with_var:
            Ks = kmat(P, d.X, xt)
            A = sla.solve_triangular(d.L, Ks, lower=True)
            V = sla.cho_solve((d.L, True), Ks)
            arr(var, (m,))[:] = kmat(P, xt[:1], xt[:1])[0, 0] + arr(diag_test, (m,)) - np.sum(A * A, axis=0)
            arr(dvar, (m, nd))[:] = -2.0 * np.einsum("mjc,jm->mc", G, V)
        return 0


@pytest.fixture()
def mocklib():
    lib = PredictGradMockLib()
    ctx = _cabi.Context.__new__(_cabi.Context)
    ctx.lib, ctx.handle, ctx.device = lib, c_void_p(1), -1
    previous = _cabi._ctx
    _cabi.set_context(ctx)
    try:
        yield lib
    finally:
        _cabi.set_context(previous)


class _P:
    Exp, ExpSquared, Matern32, Matern52 = kernels.Exp, kernels.ExpSquared, kernels.Matern32, kernels.Matern52
    Cosine, RationalQuadratic, L2Distance = kernels.Cosine, kernels.RationalQuadratic, kernels.L2Distance
    Linear, Cholesky, Subspace = transforms.Linear, transforms.Cholesky, transforms.Subspace


CASES = {
    "sum_product_2d": (lambda m: 1.3 * m.ExpSquared(0.9) * m.Matern32(1.7) + m.RationalQuadratic(1.1, alpha=0.7) + 0.2, 2),
    "ard_subspace_3d": (lambda m: 1.5 * m.Linear(np.array([0.5, 1.5, 2.0]), m.ExpSquared())
                        + m.Subspace([0, 2], m.Cholesky(np.array([0.8, 1.1]), m.Matern52(1.2, distance=m.L2Distance()))), 3),
    "scalar_coords": (lambda m: m.Cholesky(0.9, m.Linear(np.array([1.4]), m.Exp(1.0))) * m.Cosine(5.0), 1),
}


def _data(dim, n=24, m=5, seed=9):
    rng = np.random.default_rng(seed)
    X = rng.uniform(0, 3, n) if dim == 1 else rng.uniform(0, 3, (n, dim))
    y = np.cos(X if dim == 1 else X[:, 0]) + 0.2 * rng.normal(size=n)
    Xt = rng.uniform(-0.3, 3.3, m) if dim == 1 else rng.uniform(-0.3, 3.3, (m, dim))
    return X, y, Xt


def _dense_calls(lib):
    return [c for c in lib.calls if c.startswith("dense")]


@pytest.mark.parametrize("name", list(CASES))
def test_matches_oracle(mocklib, name):
    build, dim = CASES[name]
    X, y, Xt = _data(dim)
    gp = GaussianProcess(build(_P), X, diag=0.15, mean=0.1)
    mu, g = gp.predict_and_grad(y, Xt)
    assert type(g) is PredictionGrad and g._fields == ("mean", "var") and g.var is None
    assert g.mean.shape == Xt.shape
    mu2, var, g2 = gp.predict_and_grad(y, Xt, return_var=True)
    assert g2.mean.shape == Xt.shape and g2.var.shape == Xt.shape and var.shape == (Xt.shape[0],)
    assert np.array_equal(mu, mu2) and np.array_equal(g.mean, g2.mean)
    mo, vo, dmo, dvo = predict_grad_np.predict_and_grad(build(o), X, y, 0.15, Xt, mean=0.1)
    np.testing.assert_allclose(mu, mo, rtol=1e-10, atol=1e-12)
    np.testing.assert_allclose(var, vo, rtol=1e-8, atol=1e-12)
    np.testing.assert_allclose(g.mean, dmo, rtol=1e-6, atol=1e-7)
    np.testing.assert_allclose(g2.var, dvo, rtol=1e-6, atol=1e-7)


def test_mean_is_predict_bitwise_and_one_factor(mocklib):
    X, y, Xt = _data(2)
    gp = GaussianProcess(kernels.Matern52(1.0) + 0.3 * kernels.ExpSquared(2.0), X, diag=0.1, mean=0.2)
    mu, var, _ = gp.predict_and_grad(y, Xt, return_var=True)
    assert _dense_calls(mocklib) == ["dense_create", "dense_predict_grad"]
    assert np.array_equal(mu, gp.predict(y, Xt))
    mu_p, var_p = gp.predict(y, Xt, return_var=True)
    assert np.array_equal(mu, mu_p)
    np.testing.assert_allclose(var, var_p, rtol=1e-12, atol=1e-14)
    mocklib.calls.clear()
    gp.predict_and_grad(y, Xt)
    assert _dense_calls(mocklib) == ["dense_predict_grad"]


def test_component_kernel_and_include_mean(mocklib):
    X, y, Xt = _data(2)
    part = kernels.Matern32(1.3)
    gp = GaussianProcess(kernels.ExpSquared(0.7) + part, X, diag=0.1, mean=0.4)
    mu, var, g = gp.predict_and_grad(y, Xt, kernel=part, include_mean=False, return_var=True)
    assert np.array_equal(mu, gp.predict(y, Xt, kernel=part, include_mean=False))
    op = o.Matern32(1.3)
    mo, vo, dmo, dvo = predict_grad_np.predict_and_grad(o.ExpSquared(0.7) + op, X, y, 0.1, Xt, mean=0.4, pred_kernel=op)
    np.testing.assert_allclose(mu, mo - 0.4, rtol=1e-10, atol=1e-12)
    np.testing.assert_allclose(var, vo, rtol=1e-8, atol=1e-12)
    np.testing.assert_allclose(g.mean, dmo, rtol=1e-6, atol=1e-7)
    np.testing.assert_allclose(g.var, dvo, rtol=1e-6, atol=1e-7)
    _, g_in = gp.predict_and_grad(y, Xt, kernel=part)
    assert np.array_equal(g_in.mean, g.mean)


def test_callable_mean_is_not_differentiated(mocklib):
    X, y, Xt = _data(1)
    k = kernels.ExpSquared(0.9)
    gp = GaussianProcess(k, X, diag=0.1, mean=lambda x: 2.0 * x)
    mu, g = gp.predict_and_grad(y, Xt)
    mu0, g0 = gp.predict_and_grad(y, Xt, include_mean=False)
    assert np.array_equal(mu, gp.predict(y, Xt)) and np.array_equal(mu - mu0, 2.0 * Xt)
    assert np.array_equal(g.mean, g0.mean)


def test_failed_factorisation_gives_nan(mocklib):
    X = np.linspace(0, 1, 20)
    Xt = np.array([0.25, 0.5, 0.75])
    gp = GaussianProcess(kernels.ExpSquared(1.0), X, diag=-0.5)
    mu, var, g = gp.predict_and_grad(np.sin(X), Xt, return_var=True)
    assert gp.solver.info > 0
    assert g.mean.shape == (3,) and g.var.shape == (3,) and var.shape == (3,)
    assert np.all(np.isnan(g.mean)) and np.all(np.isnan(g.var)) and np.all(np.isnan(var))


def test_x_test_required(mocklib):
    X, y, _ = _data(2)
    with pytest.raises(ValueError, match="X_test"):
        GaussianProcess(kernels.ExpSquared(1.0), X, diag=0.1).predict_and_grad(y, None)


@pytest.mark.parametrize("case", list(REFUSED) + ["nine_dims", "callable_transform_kernel"])
def test_refused(mocklib, case):
    if case == "nine_dims":
        X, y, Xt = _data(9, n=12)
        gp = GaussianProcess(kernels.ExpSquared(1.0), X, diag=0.1)
        match = "at most 8"
    elif case == "callable_transform_kernel":
        X, y, Xt = _data(2, n=12)
        gp = GaussianProcess(kernels.ExpSquared(1.0), X, diag=0.1)
        with pytest.raises(NotImplementedError, match="predict_and_grad"):
            gp.predict_and_grad(y, Xt, kernel=transforms.Transform(lambda x: x * 2, kernels.ExpSquared()))
        assert "dense_predict_grad" not in mocklib.calls
        return
    else:
        X, y, Xt = _data(2, n=12)
        gp = REFUSED[case](X)
        if case in ("quasisep_solver", "quasisep_dense"):
            Xt = np.sort(Xt[:, 0])
        match = "predict_and_grad"
    with pytest.raises(NotImplementedError, match=match):
        gp.predict_and_grad(y, Xt, return_var=True)
    assert "dense_predict_grad" not in mocklib.calls
