"""GaussianProcess.fisher_information through the host layer without a GPU: a stand-in for b200gp_dense_fisher
(W from LAPACK, slot derivatives by central differences of the NumPy restatement of the kernel-program interpreter)
checks the marshalling, the parameter labels and order, the map of program slots back to the kernel's fields on both
sides (shared nodes, ARD rows through Linear / Cholesky / Subspace) against oracle/fisher_np.py, flatten, the scalar and
per-point diag cases, the refused cases, and that the solver's own factor is not touched."""

import ctypes
from ctypes import c_void_p

import numpy as np
import pytest
import scipy.linalg as sla

import hostmock
from hostmock import arr, kmat, out, parse_program
from oracle import fisher_np
from oracle import tinygp_np as o
from test_grad_host import CASES, REFUSED, GradMockLib, _P, _data
from tinygp_b200 import GaussianProcess, _cabi, kernels, transforms
from tinygp_b200.gp import FisherInformation, LogProbabilityGradX


class FisherMockLib(GradMockLib):
    def b200gp_dense_fisher(self, ctx, prog, n_rows, X, n, ndim, diag, with_diag, nslot, slots, fisher):
        self.calls.append("dense_fisher")
        rows = arr(prog, (n_rows, 4)).copy()
        x, d = arr(X, (n, ndim)).copy(), arr(diag, (n,)).copy()
        P = parse_program(prog, n_rows, ndim)
        K = kmat(P, x, x) + np.diag(d)

        def dK(mod, h):
            up, dn = rows.copy(), rows.copy()
            mod(up, h)
            mod(dn, -h)
            return (kmat(parse_program(c_void_p(up.ctypes.data), n_rows, ndim), x, x)
                    - kmat(parse_program(c_void_p(dn.ctypes.data), n_rows, ndim), x, x)) / (2 * h)

        desc, mats = [], []
        first = n_rows - P[1].shape[0]
        for i in range(first, n_rows):
            op = int(rows[i, 0])
            for c in ((2,) if op not in (6, 7) else (2, 3)) if op not in (16, 17) else ():
                h = 1e-6 * max(abs(rows[i, c]), 1e-3)
                desc.append((0, i, c))
                mats.append(dK(lambda p, s, i=i, c=c: p.__setitem__((i, c), p[i, c] + s), h))
        start = 0
        for m, M in enumerate(P[0]):
            mr, mc = M.shape
            for rr in range(mr):
                def mod(p, s, start=start, rr=rr, mc=mc, mr=mr):
                    flat = p[start + 1:start + 1 + -(-mr * mc // 4)].reshape(-1)
                    flat[rr * mc:(rr + 1) * mc] *= 1.0 + s
                    p[start + 1:start + 1 + -(-mr * mc // 4)] = flat.reshape(-1, 4)
                desc.append((1, m, rr))
                mats.append(dK(mod, 1e-6))
            start += 1 + -(-mr * mc // 4)
        out(nslot).value = len(desc)
        (ctypes.c_int * (3 * len(desc))).from_address(slots.value)[:] = [v for t in desc for v in t]
        if with_diag:
            mats.append(np.eye(n))
        k = len(mats)
        F = arr(fisher, (k, k))
        L, bad = hostmock.chol_or_nan(K)
        if bad:
            F[:] = np.nan
            return 0
        A = [sla.cho_solve((L, True), m) for m in mats]
        F[:] = [[0.5 * np.sum(a * b.T) for b in A] for a in A]
        F[:] = 0.5 * (F + F.T)
        return 0


@pytest.fixture()
def mocklib():
    lib = FisherMockLib()
    ctx = _cabi.Context.__new__(_cabi.Context)
    ctx.lib, ctx.handle, ctx.device = lib, c_void_p(1), -1
    previous = _cabi._ctx
    _cabi.set_context(ctx)
    try:
        yield lib
    finally:
        _cabi.set_context(previous)


def _against_oracle(F, labels, Fo):
    idx = {lab: i for i, lab in enumerate(labels)}
    assert sorted(idx, key=str) == sorted(F.params, key=str)
    perm = [idx[lab] for lab in F.params]
    ref = Fo[np.ix_(perm, perm)]
    np.testing.assert_allclose(F.matrix, ref, rtol=1e-5, atol=1e-7 * np.max(np.abs(ref)))


@pytest.mark.parametrize("name", list(CASES))
@pytest.mark.parametrize("scalar_diag", [True, False])
def test_matches_oracle(mocklib, name, scalar_diag):
    build, dim = CASES[name]
    X, _, rng = _data(dim)
    diag = 0.2 if scalar_diag else rng.uniform(0.1, 0.3, X.shape[0])
    F = GaussianProcess(build(_P), X, diag=diag, mean=0.1).fisher_information()
    assert isinstance(F, FisherInformation) and F.matrix.dtype == np.float64
    assert np.array_equal(F.matrix, F.matrix.T)
    assert (F.params[-1] == ("diag", None)) == scalar_diag
    labels, Fo = fisher_np.fisher(build(o), X, diag)
    _against_oracle(F, labels, Fo)


def test_params_order_and_labels(mocklib):
    X, _, _ = _data(3)
    shared = kernels.Matern32(1.1)
    k = (1.5 * transforms.Linear(np.array([0.5, 1.5, 2.0]), kernels.ExpSquared())
         + transforms.Subspace(1, transforms.Cholesky(np.array([0.7]), kernels.RationalQuadratic(0.9, alpha=1.2)))) * shared \
        + 0.5 * shared
    F = GaussianProcess(k, X, diag=0.1).fisher_information()
    assert F.params == [("kernel1.kernel1.kernel1.kernel1.value", None),
                        ("kernel1.kernel1.kernel1.kernel2.scale", 0), ("kernel1.kernel1.kernel1.kernel2.scale", 1),
                        ("kernel1.kernel1.kernel1.kernel2.scale", 2), ("kernel1.kernel1.kernel1.kernel2.kernel.scale", None),
                        ("kernel1.kernel1.kernel2.kernel.factor", 0), ("kernel1.kernel1.kernel2.kernel.kernel.scale", None),
                        ("kernel1.kernel1.kernel2.kernel.kernel.alpha", None), ("kernel1.kernel2.scale", None),
                        ("kernel2.kernel1.value", None), ("diag", None)]
    so = o.Matern32(1.1)
    ko = (1.5 * o.Linear(np.array([0.5, 1.5, 2.0]), o.ExpSquared())
          + o.Subspace(1, o.Cholesky(np.array([0.7]), o.RationalQuadratic(0.9, alpha=1.2)))) * so + 0.5 * so
    labels, Fo = fisher_np.fisher(ko, X, 0.1)
    _against_oracle(F, labels, Fo)
    # the shared Matern32 occurs twice in the program: its row and column are the sums over both occurrences
    assert F.matrix.shape == (11, 11)


def test_flatten_and_scoring_step(mocklib):
    X, y, _ = _data(2)
    k = 1.3 * kernels.ExpSquared(0.9) * kernels.Matern32(1.7) + 0.2
    gp = GaussianProcess(k, X, diag=0.2)
    F = gp.fisher_information()
    _, g = gp.log_probability_and_grad(y)
    v = F.flatten(g)
    assert v.shape == (len(F.params),)
    assert v.tolist() == [g.kernel.kernel1.kernel1.kernel1.value, g.kernel.kernel1.kernel1.kernel2.scale,
                          g.kernel.kernel1.kernel2.scale, g.kernel.kernel2.value, g.diag]
    step = np.linalg.solve(F.matrix, v)
    assert np.all(np.isfinite(step))
    np.testing.assert_array_equal(F.flatten(LogProbabilityGradX(*g, X=np.zeros_like(X))), v)
    # a per-point diag: no diag parameter, and a gradient of another model does not flatten
    gp2 = GaussianProcess(k, X, diag=np.full(X.shape[0], 0.2))
    F2 = gp2.fisher_information()
    assert F2.params == F.params[:-1]
    np.testing.assert_array_equal(F2.flatten(gp2.log_probability_and_grad(y)[1]), F2.flatten(g))
    with pytest.raises(ValueError, match="per-point"):
        F.flatten(gp2.log_probability_and_grad(y)[1])
    with pytest.raises(ValueError, match="parameters"):
        F.flatten(GaussianProcess(kernels.Exp(1.0), X, diag=0.2).log_probability_and_grad(y)[1])


def test_ard_rows_map_back_through_each_transform(mocklib):
    """a metric row owned by two nested transforms: F_user = J^T F_slot J with d lambda / d s = 1 / s and -1 / f"""
    X, _, _ = _data(1)
    k = transforms.Cholesky(0.9, transforms.Linear(np.array([1.4]), kernels.Exp(1.0))) * kernels.Cosine(5.0)
    F = GaussianProcess(k, X, diag=0.2).fisher_information()
    assert F.params == [("kernel1.factor", None), ("kernel1.kernel.scale", 0), ("kernel1.kernel.kernel.scale", None),
                        ("kernel2.scale", None), ("diag", None)]
    labels, Fo = fisher_np.fisher(o.Cholesky(0.9, o.Linear(np.array([1.4]), o.Exp(1.0))) * o.Cosine(5.0), X, 0.2)
    _against_oracle(F, labels, Fo)


def test_zero_row_scale_gives_zero(mocklib):
    X, _, _ = _data(2)
    F = GaussianProcess(transforms.Linear(np.array([0.0, 1.3]), kernels.ExpSquared()), X, diag=0.1).fisher_information()
    assert F.params[0] == ("scale", 0)
    assert np.all(F.matrix[0] == 0.0) and np.all(F.matrix[:, 0] == 0.0) and F.matrix[1, 1] > 0.0


def test_non_pd_gives_nan(mocklib):
    X = np.linspace(0, 1, 20)
    F = GaussianProcess(kernels.ExpSquared(1.0) + 0.3, X, diag=-0.5).fisher_information()
    assert F.matrix.shape == (3, 3) and np.all(np.isnan(F.matrix))


def test_solver_state_untouched(mocklib):
    X, y, _ = _data(2)
    gp = GaussianProcess(kernels.Matern52(1.0), X, diag=0.1)
    pending = gp.solver._pending
    gp.fisher_information()
    assert gp.solver._pending is pending and not gp.solver._h
    assert [c for c in mocklib.calls if c.startswith("dense")] == ["dense_fisher"]
    lp = gp.log_probability(y)                 # factors now
    h = gp.solver._h.value
    gp.fisher_information()
    assert gp.solver._h.value == h and gp.log_probability(y) == lp


@pytest.mark.parametrize("case", list(REFUSED))
def test_refused(mocklib, case):
    X, _, _ = _data(2, n=12)
    gp = REFUSED[case](X)
    with pytest.raises(NotImplementedError, match="fisher_information"):
        gp.fisher_information()
    assert "dense_fisher" not in mocklib.calls
