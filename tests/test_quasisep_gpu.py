"""Parity of the CUDA QuasisepSolver path against the oracle (run with -m gpu on an H100)."""

from ctypes import byref, c_int, c_void_p

import numpy as np
import pytest

from oracle import tinygp_np as o
from tinygp_b200 import GaussianProcess, _cabi, noise, solvers
from tinygp_b200.kernels import quasisep as Q
from util import LOGP_RTOL, rel, to_oracle

pytestmark = pytest.mark.gpu

QS = {
    "m32": lambda: Q.Matern32(1.5),                                   # test_solver.py:30
    "m52+exp": lambda: 1.5 * Q.Matern52(1.5) + 0.3 * Q.Exp(1.5),      # test_solver.py:31
    "sho+m32": lambda: Q.SHO(1.5, 3.0, 1.8) + Q.Matern32(1.5, 0.9),   # BASELINE config 4
    "sho_over": lambda: Q.SHO(1.5, 0.3),
    "sho_crit": lambda: Q.SHO(1.5, 0.5, 1.3),
    "celerite": lambda: Q.Celerite(1.1, 0.8, 0.9, 0.1),
    "cos+exp": lambda: Q.Cosine(2.5) + Q.Exp(0.7, 1.3),
    "j6": lambda: Q.SHO(1.5, 3.0, 1.8) + Q.Matern32(1.5, 0.9) + 0.5 * Q.SHO(0.4, 1.2),
    "exp": lambda: Q.Exp(2.0, 0.8),
    "prod_sho_m32": lambda: Q.SHO(1.5, 3.0, 1.8) * Q.Matern32(1.5, 0.9),          # quasisep.py:298-331 (J = 4)
    "prod3_plus_m52": lambda: 0.7 * (Q.Exp(2.0, 1.1) * Q.Celerite(1.1, 0.1, 0.3, 1.5)) + Q.Matern52(2.5, 1.3),   # J = 2 + 3
}


def _data(n, seed=84930):
    rng = np.random.default_rng(seed)
    X = np.sort(rng.uniform(-3, 3, n))
    return X, np.sin(X), rng


@pytest.mark.parametrize("qs_kernel", [1, 0])      # 1: layout-specialised kernels (default), 0: generic J x J kernels
@pytest.mark.parametrize("name", sorted(QS))
@pytest.mark.parametrize("n", [1, 50, 333])
def test_factor_and_ops_parity(name, n, qs_kernel, ctx):
    ctx.set_option("qs_kernel", qs_kernel)           # restored by the autouse fixture of conftest.py
    X, y, rng = _data(n)
    k = QS[name]()
    ko = to_oracle(k)
    diag = rng.uniform(0.05, 0.2, n)
    s = solvers.QuasisepSolver(k, X, noise.Diagonal(diag))
    so = o.QuasisepSolver(ko, X, o.Diagonal(diag))
    # generators (kernels/quasisep.py:102-116)
    for got, want in zip(s.generators(), (so.d, so.p, so.q, so.a)):
        np.testing.assert_allclose(got, want, rtol=1e-12, atol=1e-14)
    c, w = s.factor_arrays()
    np.testing.assert_allclose(c, so.c, rtol=1e-10, atol=1e-12)
    np.testing.assert_allclose(w, so.w, rtol=1e-9, atol=1e-11)
    assert rel(s.normalization(), so.normalization()) < 1e-11
    np.testing.assert_allclose(s.variance(), so.variance(), rtol=1e-14)
    Y = rng.normal(size=(n, 3))
    np.testing.assert_allclose(s.solve_triangular(y), so.solve_triangular(y), rtol=1e-9, atol=1e-11)
    np.testing.assert_allclose(s.solve_triangular(Y), so.solve_triangular(Y), rtol=1e-9, atol=1e-11)
    np.testing.assert_allclose(s.solve_triangular(Y, transpose=True), so.solve_triangular(Y, transpose=True),
                               rtol=1e-9, atol=1e-11)
    np.testing.assert_allclose(s.dot_triangular(Y), so.dot_triangular(Y), rtol=1e-10, atol=1e-12)
    if n <= 60:
        np.testing.assert_allclose(s.covariance(), so.covariance(), rtol=1e-10, atol=1e-12)
        # Quasisep == Direct on the covariance (test_solver.py:34-47)
        np.testing.assert_allclose(s.covariance(), k(X, X) + np.diag(diag), rtol=5e-7, atol=5e-7)


@pytest.mark.parametrize("qs_kernel,qs_tree", [(1, 0), (1, 1), (0, 0)])
@pytest.mark.parametrize("name", sorted(QS))
def test_logp_quasisep_equals_oracle_and_dense(name, qs_kernel, qs_tree, ctx):
    ctx.set_option("qs_kernel", qs_kernel)
    ctx.set_option("qs_tree", qs_tree)
    # test_solver.py:59-79: QuasisepSolver vs DirectSolver log-probability
    X, y, _ = _data(700)
    k = QS[name]()
    gp = GaussianProcess(k, X, diag=0.1)
    lp = gp.log_probability(y)
    lpo = o.GaussianProcess(to_oracle(k), X, diag=0.1).log_probability(y)
    assert rel(lp, lpo) < LOGP_RTOL, (lp, lpo)
    K = k(X, X) + 0.1 * np.eye(len(X))
    Lc = np.linalg.cholesky(K)
    lpd = -0.5 * np.sum(np.linalg.solve(Lc, y) ** 2) - np.sum(np.log(np.diag(Lc))) - 0.5 * len(X) * np.log(2 * np.pi)
    assert rel(lp, lpd) < 1e-7
    # parallel flag is accepted and gives the same numbers (test_solver.py:62-68)
    lp2 = GaussianProcess(k, X, diag=0.1, parallel=True, assume_sorted=True).log_probability(y)
    assert lp2 == lp


def test_unsorted_raises_and_ties_allowed(ctx):
    # test_solver.py:127-143 ; _check_sorted is a bit-exact boolean
    X, y, _ = _data(500)
    with pytest.raises(ValueError, match="sorted"):
        GaussianProcess(Q.Matern32(1.0), X[::-1].copy(), diag=0.1)
    Xs = X.copy()
    Xs[250], Xs[251] = Xs[251], Xs[250]
    with pytest.raises(ValueError, match="sorted"):
        GaussianProcess(Q.Matern32(1.0), Xs, diag=0.1)
    GaussianProcess(Q.Matern32(1.0), Xs, diag=0.1, assume_sorted=True)   # unchecked
    Xt = X.copy()
    Xt[10] = Xt[9]
    GaussianProcess(Q.Matern32(1.0), Xt, diag=0.1).log_probability(y)    # ties allowed
    flag = c_int(-1)
    for arr, want in ((X, 0), (Xs, 1), (Xt, 0), (np.array([1.0]), 0), (np.array([2.0, 1.0]), 1)):
        a = _cabi.f64(arr)
        ctx.check(ctx.lib.b200gp_qs_check_sorted(ctx.handle, _cabi.ptr(a), a.shape[0], byref(flag)))
        assert flag.value == want == int(np.any(np.diff(arr) < 0.0))


def test_searchsorted_bit_exact(ctx):
    # kernels/quasisep.py:121 : searchsorted(X2, X1, side="right") - 1
    rng = np.random.default_rng(3)
    a = np.sort(rng.uniform(0, 10, 10_000))
    a[100:105] = a[100]                       # repeated values
    v = np.concatenate([rng.uniform(-1, 11, 5000), a[::7], [a[0], a[-1], -5.0, 50.0]])
    out = np.empty(v.shape[0], dtype=np.int64)
    ctx.check(ctx.lib.b200gp_searchsorted_right_m1(ctx.handle, _cabi.ptr(a), a.shape[0], _cabi.ptr(v), v.shape[0],
                                                   c_void_p(out.ctypes.data)))
    assert np.array_equal(out, np.searchsorted(a, v, side="right") - 1)


def test_non_pd_gives_minus_inf():
    X = np.linspace(0, 1, 300)
    gp = GaussianProcess(Q.Matern32(1.0), X, diag=-0.5)
    assert gp.solver.info > 0
    assert gp.log_probability(np.ones(300)) == -np.inf


def test_large_n_against_c_oracle_and_properties():
    """N = 1e6 (many chunks, several tree levels): vs the C oracle, plus size-independent round trips."""
    from oracle import cref
    rng = np.random.default_rng(49384)
    n = 1_000_000
    t = np.sort(rng.uniform(0, 1e5, n))
    y = np.sin(t) + 0.1 * rng.normal(size=n)
    k = Q.SHO(1.5, 3.0, 1.8) + Q.Matern32(1.5, 0.9)
    gp = GaussianProcess(k, t, diag=0.1, assume_sorted=True)
    lp = gp.log_probability(y)
    d, p, q, a = o.qs_generators_fast(to_oracle(k), t)
    lpo = cref.qs_log_probability(d + 0.1, p, q, a, y)
    assert rel(lp, lpo) < LOGP_RTOL, (lp, lpo)
    s = gp.solver
    z = rng.normal(size=n)
    np.testing.assert_allclose(s.dot_triangular(s.solve_triangular(z)), z, rtol=1e-8, atol=1e-9)
    a1 = s.solve_triangular(s.solve_triangular(y), transpose=True)
    np.testing.assert_allclose(s.matmul(a1), y, rtol=1e-7, atol=1e-8)     # K K^-1 y == y


# ------------------------------------------------------------------------------------------------
# row f2: dense evaluation and the GeneralQSM product on the device (kernels/quasisep.py:118-163)
# ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", sorted(QS))
def test_dense_evaluation_on_device(name):
    """k(X1, X2) of a quasiseparable kernel: closed form in the CUDA build kernel vs the oracle's
    state-space evaluate (h Pinf T h)."""
    k, ko = QS[name](), to_oracle(QS[name]())
    rng = np.random.default_rng(5)
    X1, X2 = rng.uniform(-3, 3, 90), rng.uniform(-3, 3, 60)
    X2[:5] = X1[:5]                                  # tau = 0 pairs
    np.testing.assert_allclose(k(X1, X2), ko(X1, X2), rtol=1e-11, atol=1e-13)
    np.testing.assert_allclose(k(X1), ko(X1), rtol=1e-12)
    with pytest.raises(ValueError):
        k(np.zeros((4, 2)), np.zeros((4, 2)))


@pytest.mark.parametrize("name", sorted(QS))
@pytest.mark.parametrize("n,m", [(1, 3), (60, 45), (300, 40)])
def test_general_matmul_parity(name, n, m):
    """Quasisep.matmul(X1, X2, y) (general.py:66-106) vs the dense product; test points unsorted, outside the
    training range on both sides, and coinciding with training points.  (Sizes are bounded by the oracle, whose
    dense evaluate is a Python loop per pair; n = 300 spans 5 scan chunks, the large test below the tree.)"""
    k, ko = QS[name](), to_oracle(QS[name]())
    rng = np.random.default_rng(n + m)
    X2 = np.sort(rng.uniform(-3, 3, n))
    X1 = rng.uniform(-4, 4, m)
    X1[0], X1[1], X1[2] = X2[0], X2[-1], X2[n // 2]
    if n > 10:
        X2[7] = X2[6]                                # a repeated training coordinate
    y = rng.normal(size=n)
    Kd = ko(X1, X2)
    np.testing.assert_allclose(k.matmul(X1, X2, y), Kd @ y, rtol=1e-9, atol=1e-10)
    Y = rng.normal(size=(n, 3))
    np.testing.assert_allclose(k.matmul(X1, X2, Y), Kd @ Y, rtol=1e-9, atol=1e-10)
    if n <= 60:
        np.testing.assert_allclose(k.matmul(X2, y), ko(X2, X2) @ y, rtol=1e-9, atol=1e-10)   # symmetric form


def test_general_matmul_large_consistency():
    """N = 3e5 training points, M = 1e5 test points: rows at training coordinates equal the symmetric product
    (core.py:499-505) minus the noise term, and far-away test points decouple."""
    n, m = 300_000, 100_000
    rng = np.random.default_rng(9)
    X = np.sort(rng.uniform(0, 3e4, n))
    y = np.sin(X) + 0.1 * rng.normal(size=n)
    k = Q.SHO(1.5, 3.0, 1.8) + Q.Matern32(1.5, 0.9)
    diag = np.full(n, 0.1)
    gp = GaussianProcess(k, X, diag=diag)
    sym = gp.solver.matmul(y) - diag * y
    pick = rng.integers(0, n, m)
    got = k.matmul(X[pick], X, y)
    np.testing.assert_allclose(got, sym[pick], rtol=1e-9, atol=1e-9)
    far = k.matmul(np.array([-1e5, 1e6]), X, y)     # exp(-tau) underflows: no coupling (Matern/SHO decay)
    assert np.all(np.abs(far) < 1e-300)
