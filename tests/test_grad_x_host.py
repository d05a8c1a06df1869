"""GaussianProcess.log_probability_and_grad(y, wrt_X=True) through the host layer without a GPU: a stand-in for
b200gp_dense_log_probability_grad_x (the NumPy stand-in of the plain gradient, plus d logp / d X from central differences
of the NumPy restatement of the kernel-program interpreter) checks which entry point each call issues, the shapes of the
result for (N,) and (N, D) coordinates against oracle/grad_x_np.py, the refused cases, and that the solver's own factor
is not touched."""

from ctypes import c_void_p

import numpy as np
import pytest

from hostmock import arr, kmat, parse_program
from oracle import grad_x_np
from oracle import tinygp_np as o
from test_grad_host import REFUSED, GradMockLib
from tinygp_b200 import GaussianProcess, _cabi, kernels, transforms
from tinygp_b200.gp import LogProbabilityGrad, LogProbabilityGradX


class GradXMockLib(GradMockLib):
    def b200gp_dense_log_probability_grad_x(self, ctx, prog, n_rows, X, n, ndim, diag, resid, logp, dprog, dmetric,
                                            ddiag, alpha, dX):
        super().b200gp_dense_log_probability_grad(ctx, prog, n_rows, X, n, ndim, diag, resid, logp, dprog, dmetric, ddiag,
                                                  alpha)
        self.calls[-1] = "dense_log_probability_grad_x"
        dx = arr(dX, (n, ndim))
        a = arr(alpha, (n,)).copy()
        if np.isnan(a).any():
            dx[:] = np.nan
            return 0
        x, d = arr(X, (n, ndim)).copy(), arr(diag, (n,)).copy()
        P = parse_program(prog, n_rows, ndim)
        W = np.linalg.inv(kmat(P, x, x) + np.diag(d))
        omega = np.outer(a, a) - W
        np.fill_diagonal(omega, 0.0)
        h = 1e-6
        for i in range(n):
            for c in range(ndim):
                up, dn = x[i:i + 1].copy(), x[i:i + 1].copy()
                up[0, c] += h
                dn[0, c] -= h
                dx[i, c] = omega[i] @ ((kmat(P, up, x) - kmat(P, dn, x))[0] / (2 * h))
        return 0


@pytest.fixture()
def mocklib():
    lib = GradXMockLib()
    ctx = _cabi.Context.__new__(_cabi.Context)
    ctx.lib, ctx.handle, ctx.device = lib, c_void_p(1), -1
    previous = _cabi._ctx
    _cabi.set_context(ctx)
    try:
        yield lib
    finally:
        _cabi.set_context(previous)


def _data(dim, n=24, seed=7):
    rng = np.random.default_rng(seed)
    X = rng.uniform(0, 3, n) if dim == 1 else rng.uniform(0, 3, (n, dim))
    y = np.cos(X if dim == 1 else X[:, 0]) + 0.2 * rng.normal(size=n)
    return X, y


CASES = {
    "sum_product_2d": (lambda m: 1.3 * m.ExpSquared(0.9) * m.Matern32(1.7) + m.RationalQuadratic(1.1, alpha=0.7) + 0.2, 2),
    "ard_3d": (lambda m: 1.5 * m.Linear(np.array([0.5, 1.5, 2.0]), m.ExpSquared())
               + m.Subspace([0, 2], m.Cholesky(np.array([0.8, 1.1]), m.Matern52(1.2, distance=m.L2Distance()))), 3),
    "scalar_coords": (lambda m: m.Cholesky(0.9, m.Linear(np.array([1.4]), m.Exp(1.0))) * m.Cosine(5.0), 1),
}


class _P:
    Exp, ExpSquared, Matern32, Matern52 = kernels.Exp, kernels.ExpSquared, kernels.Matern32, kernels.Matern52
    Cosine, RationalQuadratic, L2Distance = kernels.Cosine, kernels.RationalQuadratic, kernels.L2Distance
    Linear, Cholesky, Subspace = transforms.Linear, transforms.Cholesky, transforms.Subspace


def test_default_call_is_unchanged(mocklib):
    X, y = _data(2)
    logp, g = GaussianProcess(kernels.Matern52(1.0), X, diag=0.1).log_probability_and_grad(y)
    assert type(g) is LogProbabilityGrad and g._fields == ("kernel", "diag", "mean")
    assert [c for c in mocklib.calls if c.startswith("dense")] == ["dense_log_probability_grad"]


@pytest.mark.parametrize("name", list(CASES))
def test_wrt_X_matches_oracle(mocklib, name):
    build, dim = CASES[name]
    X, y = _data(dim)
    gp = GaussianProcess(build(_P), X, diag=0.15, mean=0.1)
    lp0, g0 = gp.log_probability_and_grad(y)
    mocklib.calls.clear()
    logp, g = gp.log_probability_and_grad(y, wrt_X=True)
    assert [c for c in mocklib.calls if c.startswith("dense")] == ["dense_log_probability_grad_x"]
    assert type(g) is LogProbabilityGradX and g._fields == ("kernel", "diag", "mean", "X")
    assert logp == lp0 and g.diag == g0.diag and np.array_equal(g.mean, g0.mean)
    assert g.X.shape == X.shape
    lpo, dXo, alpha = grad_x_np.log_probability_grad_x(build(o), X, y, 0.15, mean=0.1)
    assert logp == pytest.approx(lpo, rel=1e-10)
    np.testing.assert_allclose(g.X, dXo, rtol=1e-6, atol=1e-7)
    np.testing.assert_allclose(g.mean, alpha, rtol=1e-10)


def test_non_pd_gives_nan(mocklib):
    X = np.linspace(0, 1, 20)
    logp, g = GaussianProcess(kernels.ExpSquared(1.0), X, diag=-0.5).log_probability_and_grad(np.sin(X), wrt_X=True)
    assert logp == -np.inf and np.isnan(g.kernel.scale) and np.all(np.isnan(g.X)) and g.X.shape == (20,)


def test_solver_state_untouched(mocklib):
    X, y = _data(2)
    gp = GaussianProcess(kernels.Matern52(1.0), X, diag=0.1)
    pending = gp.solver._pending
    gp.log_probability_and_grad(y, wrt_X=True)
    assert gp.solver._pending is pending and not gp.solver._h
    lp = gp.log_probability(y)                 # factors now
    h = gp.solver._h.value
    gp.log_probability_and_grad(y, wrt_X=True)
    assert gp.solver._h.value == h and gp.log_probability(y) == lp


@pytest.mark.parametrize("case", list(REFUSED) + ["nine_dims"])
def test_refused(mocklib, case):
    if case == "nine_dims":
        X, y = _data(9, n=12)
        gp = GaussianProcess(kernels.ExpSquared(1.0), X, diag=0.1)
        with pytest.raises(NotImplementedError, match="at most 8"):
            gp.log_probability_and_grad(y, wrt_X=True)
        gp.log_probability_and_grad(y)         # the plain gradient has no dimension cap
    else:
        X, y = _data(2, n=12)
        gp = REFUSED[case](X)
        with pytest.raises(NotImplementedError, match="log_probability_and_grad|gradients"):
            gp.log_probability_and_grad(y, wrt_X=True)
    assert "dense_log_probability_grad_x" not in mocklib.calls
