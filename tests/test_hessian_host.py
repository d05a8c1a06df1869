"""GaussianProcess.log_probability_hessian through the host layer without a GPU: a stand-in for
b200gp_dense_log_probability_hessian (the gradient stand-in of test_grad_host.py, then H over the slots from LAPACK and
central differences of the NumPy restatement of the kernel-program interpreter) checks the marshalling, the labels and
order, J^T H J for shared nodes and ARD rows, the curvature that Cholesky rows and chains of transforms add (against
finite differences of the mapped gradient), flatten, the scalar and per-point diag cases, the refused cases, and that
the solver's own factor is not touched."""

import ctypes
from ctypes import c_void_p

import numpy as np
import pytest
import scipy.linalg as sla

import hostmock
from hostmock import arr, kmat, out, parse_program
from oracle import hessian_np
from oracle import tinygp_np as o
from test_grad_host import CASES, REFUSED, GradMockLib, _P, _data
from tinygp_b200 import GaussianProcess, _cabi, kernels, transforms
from tinygp_b200.gp import LogProbabilityHessian


class HessianMockLib(GradMockLib):
    def b200gp_dense_log_probability_hessian(self, ctx, prog, n_rows, X, n, ndim, diag, resid, with_diag, logp, dprog,
                                             dmetric, ddiag, alpha, nslot, slots, hess):
        self.b200gp_dense_log_probability_grad(ctx, prog, n_rows, X, n, ndim, diag, resid, logp, dprog, dmetric, ddiag,
                                               alpha)
        self.calls[-1] = "dense_log_probability_hessian"
        rows = arr(prog, (n_rows, 4)).copy()
        x, d, r = arr(X, (n, ndim)).copy(), arr(diag, (n,)).copy(), arr(resid, (n,)).copy()
        P = parse_program(prog, n_rows, ndim)
        # slots as (program entry) or (metric block start, rows, cols, row)
        desc, where = [], []
        first = n_rows - P[1].shape[0]
        for i in range(first, n_rows):
            op = int(rows[i, 0])
            for c in ((2,) if op not in (6, 7) else (2, 3)) if op not in (16, 17) else ():
                desc.append((0, i, c))
                where.append(("p", i, c))
        start = 0
        for m, M in enumerate(P[0]):
            mr, mc = M.shape
            for rr in range(mr):
                desc.append((1, m, rr))
                where.append(("m", start, mr, mc, rr))
            start += 1 + -(-mr * mc // 4)
        S = len(desc)
        out(nslot).value = S
        (ctypes.c_int * (3 * S)).from_address(slots.value)[:] = [v for t in desc for v in t]
        steps = [1e-4 * max(abs(rows[w[1], w[2]]), 1e-2) if w[0] == "p" else 1e-4 for w in where]

        def K_at(delta):
            p = rows.copy()
            scale = {}
            for q, dv in delta.items():
                w = where[q]
                if w[0] == "p":
                    p[w[1], w[2]] += dv
                else:
                    scale[w[1:]] = scale.get(w[1:], 1.0) + dv
            for (st, mr, mc, rr), sc in scale.items():
                nd = -(-mr * mc // 4)
                flat = p[st + 1:st + 1 + nd].reshape(-1)
                flat[rr * mc:(rr + 1) * mc] *= sc
                p[st + 1:st + 1 + nd] = flat.reshape(-1, 4)
            return kmat(parse_program(c_void_p(p.ctypes.data), n_rows, ndim), x, x)

        def add(a, b, sa, sb):
            dl = {a: sa}
            dl[b] = dl.get(b, 0.0) + sb
            return K_at(dl)

        k = S + with_diag
        Hm = arr(hess, (k, k))
        L, bad = hostmock.chol_or_nan(kmat(P, x, x) + np.diag(d))
        if bad:
            Hm[:] = np.nan
            return 0
        W = sla.cho_solve((L, True), np.eye(n))
        a = W @ r
        A = np.outer(a, a) - W
        dK = [(K_at({q: steps[q]}) - K_at({q: -steps[q]})) / (2 * steps[q]) for q in range(S)]
        if with_diag:
            dK.append(np.eye(n))
        Hm[:] = 0.0
        for qa in range(S):
            for qb in range(qa, S):
                ha, hb = steps[qa], steps[qb]
                Kab = (add(qa, qb, ha, hb) - add(qa, qb, ha, -hb) - add(qa, qb, -ha, hb) + add(qa, qb, -ha, -hb)) / (4 * ha * hb)
                Hm[qa, qb] = Hm[qb, qa] = 0.5 * np.sum(A * Kab)
        V = np.stack([m @ a for m in dK], axis=1)
        WK = [W @ m for m in dK]
        F = np.array([[0.5 * np.sum(p * q.T) for q in WK] for p in WK])
        G = V.T @ W @ V
        Hm[:] = Hm - 0.5 * (G + G.T) + 0.5 * (F + F.T)
        return 0


@pytest.fixture()
def mocklib():
    lib = HessianMockLib()
    ctx = _cabi.Context.__new__(_cabi.Context)
    ctx.lib, ctx.handle, ctx.device = lib, c_void_p(1), -1
    previous = _cabi._ctx
    _cabi.set_context(ctx)
    try:
        yield lib
    finally:
        _cabi.set_context(previous)


def _against_oracle(H, labels, Ho):
    idx = {lab: i for i, lab in enumerate(labels)}
    assert sorted(idx, key=str) == sorted(H.params, key=str)
    perm = [idx[lab] for lab in H.params]
    ref = Ho[np.ix_(perm, perm)]
    np.testing.assert_allclose(H.matrix, ref, rtol=1e-5, atol=1e-6 * np.max(np.abs(ref)))


@pytest.mark.parametrize("name", list(CASES))
@pytest.mark.parametrize("scalar_diag", [True, False])
def test_matches_oracle(mocklib, name, scalar_diag):
    build, dim = CASES[name]
    X, y, rng = _data(dim)
    diag = 0.2 if scalar_diag else rng.uniform(0.1, 0.3, X.shape[0])
    gp = GaussianProcess(build(_P), X, diag=diag, mean=0.1)
    logp, g, H = gp.log_probability_hessian(y)
    assert isinstance(H, LogProbabilityHessian) and H.matrix.dtype == np.float64
    assert np.array_equal(H.matrix, H.matrix.T)
    assert (H.params[-1] == ("diag", None)) == scalar_diag
    lp2, g2 = gp.log_probability_and_grad(y)
    assert logp == lp2 and np.array_equal(H.flatten(g), H.flatten(g2)) and np.array_equal(g.mean, g2.mean)
    labels, Ho = hessian_np.hessian(build(o), X, y, diag, mean=0.1)
    _against_oracle(H, labels, Ho)


def test_params_order_shared_node_and_ard_rows(mocklib):
    X, y, _ = _data(3)
    shared = kernels.Matern32(1.1)
    k = (1.5 * transforms.Linear(np.array([0.5, 1.5, 2.0]), kernels.ExpSquared())
         + transforms.Subspace(1, transforms.Cholesky(np.array([0.7]), kernels.RationalQuadratic(0.9, alpha=1.2)))) * shared \
        + 0.5 * shared
    _, _, H = GaussianProcess(k, X, diag=0.1).log_probability_hessian(y)
    assert H.params == [("kernel1.kernel1.kernel1.kernel1.value", None),
                        ("kernel1.kernel1.kernel1.kernel2.scale", 0), ("kernel1.kernel1.kernel1.kernel2.scale", 1),
                        ("kernel1.kernel1.kernel1.kernel2.scale", 2), ("kernel1.kernel1.kernel1.kernel2.kernel.scale", None),
                        ("kernel1.kernel1.kernel2.kernel.factor", 0), ("kernel1.kernel1.kernel2.kernel.kernel.scale", None),
                        ("kernel1.kernel1.kernel2.kernel.kernel.alpha", None), ("kernel1.kernel2.scale", None),
                        ("kernel2.kernel1.value", None), ("diag", None)]
    so = o.Matern32(1.1)
    ko = (1.5 * o.Linear(np.array([0.5, 1.5, 2.0]), o.ExpSquared())
          + o.Subspace(1, o.Cholesky(np.array([0.7]), o.RationalQuadratic(0.9, alpha=1.2)))) * so + 0.5 * so
    labels, Ho = hessian_np.hessian(ko, X, y, 0.1)
    _against_oracle(H, labels, Ho)


def _flat_grad(make, X, y, theta):
    gp = GaussianProcess(make(*theta), X, diag=theta[-1])
    _, g, H = gp.log_probability_hessian(y)
    return H.flatten(g), H


@pytest.mark.parametrize("chain", ["cholesky", "cholesky_of_linear", "linear_of_cholesky"])
def test_row_scale_curvature_against_differences_of_the_mapped_gradient(mocklib, chain):
    """H over the fields = the Jacobian of the gradient over the fields, which carries d^2 lambda / d field^2 for a
    Cholesky row (lambda = f / f') and the cross terms of a chain of row scales"""
    X, y, _ = _data(2)
    makes = {
        "cholesky": lambda f0, f1, s, d: transforms.Cholesky(np.array([f0, f1]), kernels.Matern52(s, distance=kernels.L2Distance())),
        "cholesky_of_linear": lambda f0, f1, s, d: transforms.Cholesky(np.array([f0, f1]), transforms.Linear(np.array([s, 1.3]), kernels.ExpSquared())),
        "linear_of_cholesky": lambda f0, f1, s, d: transforms.Linear(np.array([f0, f1]), transforms.Cholesky(np.array([s, 0.8]), kernels.Exp(1.1))),
    }
    make = makes[chain]
    theta = np.array([0.9, 1.4, 1.2, 0.2])
    g0, H = _flat_grad(make, X, y, theta)
    # the fields in params order, as entries of theta (the fourth is the scalar diag)
    order = {"cholesky": [0, 1, 2, 3], "cholesky_of_linear": [0, 1, 2, None, None, 3],
             "linear_of_cholesky": [0, 1, 2, None, None, 3]}[chain]
    assert len(H.params) == len(order)
    for col, t in enumerate(order):
        if t is None:
            continue
        h = 1e-4 * abs(theta[t])
        up, dn = theta.copy(), theta.copy()
        up[t] += h
        dn[t] -= h
        fd = (_flat_grad(make, X, y, up)[0] - _flat_grad(make, X, y, dn)[0]) / (2 * h)
        np.testing.assert_allclose(H.matrix[:, col], fd, rtol=2e-4, atol=2e-5 * np.max(np.abs(H.matrix)), err_msg=str(H.params[col]))


def test_flatten_and_newton_step(mocklib):
    X, y, _ = _data(2)
    k = 1.3 * kernels.ExpSquared(0.9) * kernels.Matern32(1.7) + 0.2
    gp = GaussianProcess(k, X, diag=0.2)
    _, g, H = gp.log_probability_hessian(y)
    v = H.flatten(g)
    assert v.tolist() == [g.kernel.kernel1.kernel1.kernel1.value, g.kernel.kernel1.kernel1.kernel2.scale,
                          g.kernel.kernel1.kernel2.scale, g.kernel.kernel2.value, g.diag]
    assert np.all(np.isfinite(np.linalg.solve(H.matrix, v)))
    gp2 = GaussianProcess(k, X, diag=np.full(X.shape[0], 0.2))
    _, g2, H2 = gp2.log_probability_hessian(y)
    assert H2.params == H.params[:-1] and H2.matrix.shape == (4, 4)
    np.testing.assert_allclose(H2.matrix, H.matrix[:4, :4], rtol=1e-12)
    with pytest.raises(ValueError, match="per-point"):
        H.flatten(g2)
    with pytest.raises(ValueError, match="parameters"):
        H.flatten(GaussianProcess(kernels.Exp(1.0), X, diag=0.2).log_probability_and_grad(y)[1])


def test_zero_row_scale_gives_zero(mocklib):
    X, y, _ = _data(2)
    _, _, H = GaussianProcess(transforms.Linear(np.array([0.0, 1.3]), kernels.ExpSquared()), X, diag=0.1).log_probability_hessian(y)
    assert H.params[0] == ("scale", 0)
    assert np.all(H.matrix[0] == 0.0) and np.all(H.matrix[:, 0] == 0.0) and H.matrix[1, 1] != 0.0


def test_non_pd_gives_nan(mocklib):
    X = np.linspace(0, 1, 20)
    logp, g, H = GaussianProcess(kernels.ExpSquared(1.0) + 0.3, X, diag=-0.5).log_probability_hessian(np.sin(X))
    assert logp == -np.inf and np.isnan(g.diag) and np.all(np.isnan(g.mean))
    assert H.matrix.shape == (3, 3) and np.all(np.isnan(H.matrix))


def test_solver_state_untouched(mocklib):
    X, y, _ = _data(2)
    gp = GaussianProcess(kernels.Matern52(1.0), X, diag=0.1)
    pending = gp.solver._pending
    gp.log_probability_hessian(y)
    assert gp.solver._pending is pending and not gp.solver._h
    assert [c for c in mocklib.calls if c.startswith("dense")] == ["dense_log_probability_hessian"]
    lp = gp.log_probability(y)                 # factors now
    h = gp.solver._h.value
    gp.log_probability_hessian(y)
    assert gp.solver._h.value == h and gp.log_probability(y) == lp


@pytest.mark.parametrize("case", list(REFUSED))
def test_refused(mocklib, case):
    X, y, _ = _data(2, n=12)
    gp = REFUSED[case](X)
    with pytest.raises(NotImplementedError, match="log_probability_hessian"):
        gp.log_probability_hessian(y)
    assert "dense_log_probability_hessian" not in mocklib.calls
