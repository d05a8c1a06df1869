"""GaussianProcess.log_probability_hessian on the GPU: parity with the LAPACK / complex-step Hessian of
oracle/hessian_np.py on the native fp64 and the int8-update factorisations, bitwise symmetry and reproducibility, the
logp / gradient / alpha of log_probability_and_grad and the F of fisher_information bit for bit, non positive-definite
input, and central differences of the device gradient at n = 16384."""

import ctypes

import numpy as np
import pytest

from oracle import hessian_np
from oracle import tinygp_np as o
from test_fisher_gpu import CASES, _P, _data
from tinygp_b200 import GaussianProcess, _cabi, kernels

pytestmark = pytest.mark.gpu

_ORACLE = {}


def _check(name, n, scalar_diag=True):
    build, dim = CASES[name]
    X, dvec = _data(dim, n)
    y = np.cos(X if dim == 1 else X[:, 0]) + 0.3 * np.random.default_rng(n).normal(size=n)
    diag = 0.2 if scalar_diag else dvec
    gp = GaussianProcess(build(_P), X, diag=diag, mean=0.1)
    logp, g, H = gp.log_probability_hessian(y)
    key = (name, n, scalar_diag)
    if key not in _ORACLE:
        _ORACLE[key] = hessian_np.hessian(build(o), X, y, diag, mean=0.1)
    labels, Ho = _ORACLE[key]
    idx = {lab: i for i, lab in enumerate(labels)}
    assert sorted(idx, key=str) == sorted(H.params, key=str)
    perm = [idx[lab] for lab in H.params]
    ref = Ho[np.ix_(perm, perm)]
    err = np.max(np.abs(H.matrix - ref)) / np.max(np.abs(ref))
    assert err <= 1e-8, (name, n, err)
    assert np.array_equal(H.matrix, H.matrix.T)
    lp2, g2 = gp.log_probability_and_grad(y)
    assert logp == lp2 and np.array_equal(H.flatten(g), H.flatten(g2)) and np.array_equal(g.mean, g2.mean)


@pytest.mark.parametrize("n", [300, 1000, 2500])
@pytest.mark.parametrize("name", list(CASES))
def test_hessian_matches_oracle(name, n):
    _check(name, n)


@pytest.mark.parametrize("n", [300, 1000, 2500])
@pytest.mark.parametrize("name", ["expsq_const", "ard", "periodic"])
def test_hessian_matches_oracle_int8_update(name, n):
    ctx = _cabi.get_context()
    ctx.set_option("ozaki_min_n", 0)
    ctx.set_option("nb", 256)
    try:
        _check(name, n)
    finally:
        ctx.reset_options()


@pytest.mark.parametrize("name", ["exp_matern", "ard"])
def test_hessian_per_point_diag(name):
    _check(name, 1000, scalar_diag=False)


def test_bitwise_symmetric_reproducible_and_equal_to_gradient_and_fisher():
    X, d = _data(3, 1500)
    y = np.sin(X[:, 0])
    gp = GaussianProcess(CASES["ard"][0](_P), X, diag=0.2)
    before = gp.log_probability(y)
    lp1, g1, H1 = gp.log_probability_hessian(y)
    lp2, g2, H2 = gp.log_probability_hessian(y)
    assert np.array_equal(H1.matrix, H1.matrix.T)
    assert np.array_equal(H1.matrix, H2.matrix) and H1.params == H2.params and lp1 == lp2
    lpg, gg = gp.log_probability_and_grad(y)
    assert lp1 == lpg and np.array_equal(H1.flatten(g1), H1.flatten(gg)) and np.array_equal(g1.mean, gg.mean)
    assert gp.log_probability(y) == before
    # the F part, through the diagnostics entry, against b200gp_dense_fisher on the same input
    prog, x, slots = gp.solver._grad_slots("test")
    ctx = _cabi.get_context()
    k = len(slots) + 1
    hess, terms = np.empty(k * k), np.empty(3 * k * k)
    ctx.check(ctx.lib.b200gp_dense_hessian_terms_test(ctx.handle, _cabi.ptr(prog), prog.shape[0], _cabi.ptr(x),
                                                      x.shape[0], x.shape[1], _cabi.ptr(gp.solver._diag),
                                                      _cabi.ptr(np.ascontiguousarray(y)), 1, _cabi.ptr(hess),
                                                      _cabi.ptr(terms)))
    ns, origin, F = ctypes.c_int(), np.zeros(48, dtype=np.int32), np.empty(k * k)
    ctx.check(ctx.lib.b200gp_dense_fisher(ctx.handle, _cabi.ptr(prog), prog.shape[0], _cabi.ptr(x), x.shape[0],
                                          x.shape[1], _cabi.ptr(gp.solver._diag), 1, ctypes.byref(ns), _cabi.ptr(origin),
                                          _cabi.ptr(F)))
    S2, G, Fh = terms.reshape(3, k, k)
    assert np.array_equal(Fh, F.reshape(k, k))
    assert np.array_equal(hess.reshape(k, k), (S2 - G) + Fh)
    # the noise diagonal: no second-derivative term
    assert np.all(S2[-1] == 0.0) and np.all(S2[:, -1] == 0.0)


def test_non_pd_gives_nan():
    X = np.linspace(0, 1, 200)
    logp, g, H = GaussianProcess(kernels.ExpSquared(1.0) + 0.3, X, diag=-0.5).log_probability_hessian(np.sin(X))
    assert logp == -np.inf and np.all(np.isnan(g.mean))
    assert H.matrix.shape == (3, 3) and np.all(np.isnan(H.matrix))


def test_central_differences_of_the_device_gradient_at_16384():
    """H against (g(theta + h e_b) - g(theta - h e_b)) / 2h of the device gradient, at two steps: the error of the
    differences is estimated from their change between the steps (truncation ~ h^2) and the rounding of the gradient"""
    n = 16384
    rng = np.random.default_rng(21)
    X = rng.uniform(0, 40, (n, 2))
    y = np.sin(X[:, 0]) + 0.3 * rng.normal(size=n)
    theta = np.array([1.2, 1.5, 0.8, 2.0, 0.3])

    def make(t):
        k = t[0] * kernels.ExpSquared(t[1]) + t[2] * kernels.Matern32(t[3], distance=kernels.L2Distance())
        return GaussianProcess(k, X, diag=t[4])

    _, g, H = make(theta).log_probability_hessian(y)
    assert H.params == [("kernel1.kernel1.value", None), ("kernel1.kernel2.scale", None),
                        ("kernel2.kernel1.value", None), ("kernel2.kernel2.scale", None), ("diag", None)]
    grad = lambda t: H.flatten(make(t).log_probability_and_grad(y)[1])
    for b in range(len(theta)):
        cols = []
        for rel in (1e-3, 5e-4):
            h = rel * theta[b]
            up, dn = theta.copy(), theta.copy()
            up[b] += h
            dn[b] -= h
            cols.append((grad(up) - grad(dn)) / (2 * h))
        fd = cols[1]
        err = np.abs(cols[0] - cols[1]) + 1e-6 * np.max(np.abs(H.matrix))
        print(b, np.max(np.abs(H.matrix[:, b] - fd) / err))
        assert np.all(np.abs(H.matrix[:, b] - fd) <= 3 * err), (b, H.matrix[:, b], fd, err)
