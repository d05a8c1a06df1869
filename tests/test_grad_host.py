"""GaussianProcess.log_probability_and_grad through the host layer without a GPU: a stand-in for
b200gp_dense_log_probability_grad (dense algebra in NumPy, slot derivatives by central differences of the NumPy
restatement of the kernel-program interpreter) checks the marshalling, the mapping of program slots back to the kernel
tree (shared nodes, ARD row scales through Linear / Cholesky / Subspace) against oracle/grad_np.py, the refused
cases, and that the solver's own factor is not touched."""

from ctypes import c_void_p

import numpy as np
import pytest
import scipy.linalg as sla

import hostmock
from hostmock import arr, kmat, out, parse_program
from oracle import grad_np
from oracle import tinygp_np as o
from tinygp_b200 import GaussianProcess, _cabi, kernels, noise, transforms
from tinygp_b200.kernels import quasisep as Q


class GradMockLib(hostmock.MockLib):
    def b200gp_dense_log_probability_grad(self, ctx, prog, n_rows, X, n, ndim, diag, resid, logp, dprog, dmetric, ddiag,
                                          alpha):
        self.calls.append("dense_log_probability_grad")
        rows = arr(prog, (n_rows, 4)).copy()
        x, d, r = arr(X, (n, ndim)).copy(), arr(diag, (n,)).copy(), arr(resid, (n,)).copy()
        P = parse_program(prog, n_rows, ndim)
        L, bad = hostmock.chol_or_nan(kmat(P, x, x) + np.diag(d))
        dp, dm = arr(dprog, (n_rows, 4)), arr(dmetric, (3, 8))
        dp[:], dm[:] = 0.0, 0.0
        if bad:
            out(logp).value = -np.inf
            dp[n_rows - P[1].shape[0]:, 2:] = np.nan
            arr(ddiag, (n,))[:] = np.nan
            arr(alpha, (n,))[:] = np.nan
            return 0
        a = sla.cho_solve((L, True), r)
        W = sla.cho_solve((L, True), np.eye(n))
        out(logp).value = -0.5 * r @ a - np.sum(np.log(np.diag(L))) - 0.5 * n * np.log(2 * np.pi)
        Wt = 0.5 * (np.outer(a, a) - W)

        def dK(mod, h):
            up, dn = rows.copy(), rows.copy()
            mod(up, h)
            mod(dn, -h)
            Pu = parse_program(c_void_p(up.ctypes.data), n_rows, ndim)
            Pd = parse_program(c_void_p(dn.ctypes.data), n_rows, ndim)
            return (kmat(Pu, x, x) - kmat(Pd, x, x)) / (2 * h)

        first = n_rows - P[1].shape[0]
        for i in range(first, n_rows):
            op = int(rows[i, 0])
            for c in ((2,) if op not in (6, 7) else (2, 3)) if op not in (16, 17) else ():
                h = 1e-6 * max(abs(rows[i, c]), 1e-3)
                dp[i, c] = np.sum(Wt * dK(lambda p, s, i=i, c=c: p.__setitem__((i, c), p[i, c] + s), h))
        start = 0
        for m, M in enumerate(P[0]):
            mr, mc = M.shape
            for rr in range(mr):
                def mod(p, s, start=start, rr=rr, mc=mc):
                    flat = p[start + 1:start + 1 + -(-mr * mc // 4)].reshape(-1)
                    flat[rr * mc:(rr + 1) * mc] *= 1.0 + s
                    p[start + 1:start + 1 + -(-mr * mc // 4)] = flat.reshape(-1, 4)
                dm[m, rr] = np.sum(Wt * dK(mod, 1e-6))
            start += 1 + -(-mr * mc // 4)
        arr(ddiag, (n,))[:] = 0.5 * (a * a - np.diag(W))
        arr(alpha, (n,))[:] = a
        return 0


@pytest.fixture()
def mocklib():
    lib = GradMockLib()
    ctx = _cabi.Context.__new__(_cabi.Context)
    ctx.lib, ctx.handle, ctx.device = lib, c_void_p(1), -1
    previous = _cabi._ctx
    _cabi.set_context(ctx)
    try:
        yield lib
    finally:
        _cabi.set_context(previous)


def _data(dim, n=30, seed=5):
    rng = np.random.default_rng(seed)
    X = rng.uniform(0, 3, n) if dim == 1 else rng.uniform(0, 3, (n, dim))
    y = np.cos(X if dim == 1 else X[:, 0]) + 0.2 * rng.normal(size=n)
    return X, y, rng


def _nodes(g, on):
    yield g, on
    for a in ("kernel1", "kernel2", "kernel"):
        if hasattr(on, a):
            yield from _nodes(getattr(g, a), getattr(on, a))


class _P:
    Exp, ExpSquared, Matern32, Matern52 = kernels.Exp, kernels.ExpSquared, kernels.Matern32, kernels.Matern52
    Cosine, ExpSineSquared, RationalQuadratic = kernels.Cosine, kernels.ExpSineSquared, kernels.RationalQuadratic
    L1Distance, L2Distance, Constant = kernels.L1Distance, kernels.L2Distance, kernels.Constant
    Linear, Cholesky, Subspace = transforms.Linear, transforms.Cholesky, transforms.Subspace


CASES = {
    "sum_product": (lambda m: 1.3 * m.ExpSquared(0.9) * m.Matern32(1.7) + m.RationalQuadratic(1.1, alpha=0.7) + 0.2, 2),
    "ard_linear": (lambda m: 1.5 * m.Linear(np.array([0.5, 1.5, 2.0]), m.ExpSquared()), 3),
    "ard_cholesky_subspace": (lambda m: m.Subspace([0, 2], m.Cholesky(np.array([0.8, 1.1]), m.Matern52(1.2, distance=m.L2Distance())))
                              + m.Subspace(1, m.Linear(0.6, m.ExpSineSquared(2.0, gamma=0.5))), 3),
    "nested_scalar_coords": (lambda m: m.Cholesky(0.9, m.Linear(np.array([1.4]), m.Exp(1.0))) * m.Cosine(5.0), 1),
}


@pytest.mark.parametrize("name", list(CASES))
@pytest.mark.parametrize("scalar_diag", [True, False])
def test_kernel_tree_gradient_matches_oracle(mocklib, name, scalar_diag):
    build, dim = CASES[name]
    X, y, rng = _data(dim)
    diag = 0.2 if scalar_diag else rng.uniform(0.1, 0.3, X.shape[0])
    k = build(_P)
    gp = GaussianProcess(k, X, diag=diag, mean=0.1)
    logp, g = gp.log_probability_and_grad(y)
    assert logp == pytest.approx(gp.log_probability(y), rel=1e-12)
    ok = build(o)
    lpo, acc, ddiag, alpha = grad_np.log_probability_grad(ok, X, y, diag, mean=0.1)
    assert logp == pytest.approx(lpo, rel=1e-10)
    seen = 0
    for gn, on in _nodes(g.kernel, ok):
        assert type(gn) is type(_find(k, on, ok))
        for (nid, field), (_, ref) in acc.items():
            if nid == id(on):
                got = getattr(gn, field)
                assert np.shape(got) == np.shape(ref)
                np.testing.assert_allclose(got, ref, rtol=1e-6, atol=1e-8)
                seen += 1
    assert seen == len(acc)
    if scalar_diag:
        assert isinstance(g.diag, float) and g.diag == pytest.approx(np.sum(ddiag), rel=1e-10)
    else:
        np.testing.assert_allclose(g.diag, ddiag, rtol=1e-10)
    np.testing.assert_allclose(g.mean, alpha, rtol=1e-10)


def _find(k, on, ok):
    for a, b in _nodes(k, ok):
        if b is on:
            return a


def test_structure_and_non_differentiable_fields(mocklib):
    X, y, _ = _data(3)
    k = 1.5 * transforms.Linear(np.array([0.5, 1.5, 2.0]), kernels.ExpSquared()) + transforms.Subspace(1, kernels.Exp(0.7))
    _, g = GaussianProcess(k, X, diag=0.1).log_probability_and_grad(y)
    lin = g.kernel.kernel1.kernel2
    assert isinstance(lin, transforms.Linear) and lin.scale.shape == (3,)
    assert isinstance(lin.kernel, kernels.ExpSquared) and isinstance(lin.kernel.scale, float) and lin.kernel.distance is None
    assert isinstance(g.kernel.kernel1.kernel1.value, float)
    sub = g.kernel.kernel2
    assert sub.axis is None and isinstance(sub.kernel.scale, float)
    assert k.kernel1.kernel2.scale.tolist() == [0.5, 1.5, 2.0]              # the model is left as it was


def test_shared_node_accumulates(mocklib):
    X, y, _ = _data(2)
    shared = kernels.ExpSquared(1.2)
    k = shared + 0.5 * shared
    _, g = GaussianProcess(k, X, diag=0.1).log_probability_and_grad(y)
    assert g.kernel.kernel1 is g.kernel.kernel2.kernel2
    os_ = o.ExpSquared(1.2)
    _, acc, _, _ = grad_np.log_probability_grad(os_ + 0.5 * os_, X, y, 0.1)
    assert g.kernel.kernel1.scale == pytest.approx(acc[(id(os_), "scale")][1], rel=1e-6)
    # two equal but distinct transforms keep their own gradients (the device gets one metric each)
    la, lb = transforms.Linear(np.array([1.0, 2.0]), kernels.Exp(1.0)), transforms.Linear(np.array([1.0, 2.0]), kernels.Matern32(1.0))
    _, g2 = GaussianProcess(la + lb, X, diag=0.1).log_probability_and_grad(y)
    oa, ob = o.Linear(np.array([1.0, 2.0]), o.Exp(1.0)), o.Linear(np.array([1.0, 2.0]), o.Matern32(1.0))
    _, acc2, _, _ = grad_np.log_probability_grad(oa + ob, X, y, 0.1)
    np.testing.assert_allclose(g2.kernel.kernel1.scale, acc2[(id(oa), "scale")][1], rtol=1e-6)
    np.testing.assert_allclose(g2.kernel.kernel2.scale, acc2[(id(ob), "scale")][1], rtol=1e-6)


def test_zero_row_scale_gives_zero(mocklib):
    X, y, _ = _data(2)
    _, g = GaussianProcess(transforms.Linear(np.array([0.0, 1.3]), kernels.ExpSquared()), X, diag=0.1).log_probability_and_grad(y)
    assert g.kernel.scale[0] == 0.0 and g.kernel.scale[1] != 0.0


def test_non_pd_gives_nan(mocklib):
    X = np.linspace(0, 1, 20)
    logp, g = GaussianProcess(kernels.ExpSquared(1.0), X, diag=-0.5).log_probability_and_grad(np.sin(X))
    assert logp == -np.inf and np.isnan(g.kernel.scale) and np.isnan(g.diag) and np.all(np.isnan(g.mean))


def test_solver_state_untouched(mocklib):
    X, y, _ = _data(2)
    gp = GaussianProcess(kernels.Matern52(1.0), X, diag=0.1)
    pending = gp.solver._pending
    gp.log_probability_and_grad(y)
    assert gp.solver._pending is pending and not gp.solver._h
    assert [c for c in mocklib.calls if c.startswith("dense")] == ["dense_log_probability_grad"]
    lp = gp.log_probability(y)                 # factors now
    h = gp.solver._h.value
    gp.log_probability_and_grad(y)
    assert gp.solver._h.value == h and gp.log_probability(y) == lp


REFUSED = {
    "quasisep_solver": lambda X: GaussianProcess(Q.Matern32(1.0), np.sort(X[:, 0]), diag=0.1),
    "noise_dense": lambda X: GaussianProcess(kernels.ExpSquared(1.0), X, noise=noise.Dense(0.1 * np.eye(X.shape[0]))),
    "noise_banded": lambda X: GaussianProcess(kernels.ExpSquared(1.0), X,
                                              noise=noise.Banded(np.full(X.shape[0], 0.1), np.full((X.shape[0], 1), 0.01))),
    "covariance": lambda X: GaussianProcess(kernels.ExpSquared(1.0), X, covariance_value=np.eye(X.shape[0]), solver=None),
    "quasisep_dense": lambda X: GaussianProcess(Q.Celerite(1.1, 0.8, 0.9, 0.1), X[:, 0], diag=0.1,
                                                solver=__import__("tinygp_b200").solvers.DirectSolver),
    "matrix_linear": lambda X: GaussianProcess(transforms.Linear(np.eye(2), kernels.ExpSquared()), X, diag=0.1),
    "matrix_cholesky": lambda X: GaussianProcess(transforms.Cholesky(np.eye(2), kernels.ExpSquared()), X, diag=0.1),
    "transform_callable": lambda X: GaussianProcess(transforms.Transform(lambda x: x * 2, kernels.ExpSquared()), X, diag=0.1),
    "over_slot_cap": lambda X: GaussianProcess(sum(kernels.RationalQuadratic(1.0 + i, alpha=1.0) for i in range(9)), X, diag=0.1),
}


@pytest.mark.parametrize("case", list(REFUSED))
def test_refused(mocklib, case):
    X, y, _ = _data(2, n=12)
    gp = REFUSED[case](X)
    with pytest.raises(NotImplementedError, match="log_probability_and_grad|gradients"):
        gp.log_probability_and_grad(y)
    assert "dense_log_probability_grad" not in mocklib.calls
