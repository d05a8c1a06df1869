"""Parity of the CUDA DirectSolver path against the oracle (run with -m gpu on an H100).
Everything goes through the C-ABI (ctypes) exactly as a user of the plugin surface would."""

import numpy as np
import pytest
import scipy.linalg

from oracle import tinygp_np as o
from tinygp_b200 import GaussianProcess, kernels, noise, solvers
from util import LOGP_RTOL, assert_close, rel, to_oracle

pytestmark = pytest.mark.gpu

KERNELS = {
    "expsq": lambda: kernels.ExpSquared(1.5),
    "exp": lambda: kernels.Exp(0.7),
    "m32": lambda: kernels.Matern32(1.5),
    "m32_l2": lambda: kernels.Matern32(1.5, kernels.L2Distance()),
    "m52": lambda: kernels.Matern52(2.5),
    "cos": lambda: kernels.Cosine(2.3),
    "ess": lambda: kernels.ExpSineSquared(2.3, gamma=1.3),
    "rq": lambda: kernels.RationalQuadratic(1.2, alpha=1.7),
    "rq_l2": lambda: kernels.RationalQuadratic(1.2, kernels.L2Distance(), alpha=1.7),
    "expsq_l1": lambda: kernels.ExpSquared(1.5, kernels.L1Distance()),
    "combo": lambda: 1.8 * kernels.ExpSquared(0.9) + kernels.Matern32(3.0) * kernels.Constant(0.4) + 0.1,
    "c3": lambda: 1.5 * kernels.Matern52(2.0) + 0.7 * kernels.RationalQuadratic(1.5, alpha=1.5),
    # BASELINE config 3 with Euclidean metrics (the L1 defaults are not positive definite for D > 1)
    "c3_l2": lambda: (1.5 * kernels.Matern52(2.0, kernels.L2Distance())
                      + 0.7 * kernels.RationalQuadratic(1.5, kernels.L2Distance(), alpha=1.5)),
    "combo_l2": lambda: (1.8 * kernels.ExpSquared(0.9)
                         + kernels.Matern32(3.0, kernels.L2Distance()) * kernels.Constant(0.4) + 0.1),
}


@pytest.mark.parametrize("build_fast", [1, 0])     # 1: sum-of-products normal form (default), 0: program interpreter
@pytest.mark.parametrize("name", sorted(KERNELS))
@pytest.mark.parametrize("ndim", [1, 3])
def test_kernel_matrix_parity(name, ndim, build_fast, ctx):
    ctx.set_option("build_fast", build_fast)          # restored by conftest's autouse fixture
    rng = np.random.default_rng(1234 + ndim)
    X1 = rng.uniform(-3, 3, (137, ndim)) if ndim > 1 else rng.uniform(-3, 3, 137)
    X2 = rng.uniform(-3, 3, (61, ndim)) if ndim > 1 else rng.uniform(-3, 3, 61)
    k = KERNELS[name]()
    ko = to_oracle(k)
    np.testing.assert_allclose(k(X1, X2), ko(X1, X2), rtol=1e-13, atol=1e-15)
    np.testing.assert_allclose(k(X1, X1), ko(X1, X1), rtol=1e-13, atol=1e-15)
    np.testing.assert_allclose(k(X1), ko(X1), rtol=1e-15)
    y = rng.normal(size=61)
    np.testing.assert_allclose(k.matmul(X1, X2, y), ko(X1, X2) @ y, rtol=1e-11, atol=1e-12)
    # the diagonal of a stationary kernel is exact (explicit differences, distance.py:58-59)
    if name not in ("combo", "c3", "c3_l2", "combo_l2"):
        assert np.all(np.diag(k(X1, X1)) == np.diag(ko(X1, X1)))


def test_scalar_evaluate_and_edge_shapes():
    k = kernels.Matern52(1.3)
    assert np.isclose(k.evaluate(0.3, 1.1), to_oracle(k)(np.array([0.3]), np.array([1.1]))[0, 0], rtol=1e-14)
    one = k(np.array([0.5]), np.array([0.5, 0.7]))
    assert one.shape == (1, 2) and one[0, 0] == 1.0
    with pytest.raises(ValueError):
        k(np.zeros((3, 2)), np.zeros((3, 3)))
    with pytest.raises(Exception):
        k(np.zeros((0,)), np.zeros((3,)))


@pytest.mark.parametrize("potf2", [2, 1])
@pytest.mark.parametrize("n", [1, 50, 128, 300, 1100])
def test_factor_parity(n, ctx, potf2):
    ctx.set_option("potf2_version", potf2)
    rng = np.random.default_rng(n)
    X = rng.uniform(0, 6, (n, 2))
    k = 1.3 * kernels.ExpSquared(0.8)
    diag = rng.uniform(0.05, 0.2, n)
    for nb in (128, 512):
        ctx.set_option("nb", nb)
        ctx.set_option("ozaki_slices", 0)      # the native fp64 DMMA path is the one under test here
        s = solvers.DirectSolver(k, X, noise.Diagonal(diag))
        so = o.DirectSolver(to_oracle(k), X, o.Diagonal(diag))
        assert s.info == 0
        np.testing.assert_allclose(s.scale_tril, so.scale_tril, rtol=1e-10, atol=1e-12)
        assert rel(s.normalization(), so.normalization()) < 1e-12
        assert_close(s.variance(), so.variance(), 1e-14, 1e-14)
        np.testing.assert_allclose(s.covariance(), so.covariance(), rtol=1e-13, atol=1e-15)
    ctx.set_option("nb", 1024)
    ctx.reset_options()       # library defaults (NOT a literal: the default plane count is 7)
    ctx.set_option("potf2_version", 2)


@pytest.mark.parametrize("n,ndim,name", [(256, 1, "expsq"), (777, 3, "c3_l2"), (2048, 3, "expsq"),
                                         (1500, 2, "combo_l2"), (640, 1, "c3"), (900, 1, "combo")])
def test_log_probability_parity(n, ndim, name):
    rng = np.random.default_rng(84930)
    if ndim == 1:
        X = np.sort(rng.uniform(-3, 3, n))  # BASELINE config 1 (test_solver.py:19-24)
        y = np.sin(X)
    else:
        X = rng.uniform(0, 8, (n, ndim))
        y = np.sin(X[:, 0]) + 0.1 * rng.normal(size=n)
    k = KERNELS[name]()
    lp = GaussianProcess(k, X, diag=0.1).log_probability(y)
    lpo = o.GaussianProcess(to_oracle(k), X, diag=0.1).log_probability(y)
    assert rel(lp, lpo) < LOGP_RTOL, (lp, lpo)
    # mean handling (gp.py:81-88)
    lp = GaussianProcess(k, X, diag=0.1, mean=0.3).log_probability(y)
    lpo = o.GaussianProcess(to_oracle(k), X, diag=0.1, mean=0.3).log_probability(y)
    assert rel(lp, lpo) < LOGP_RTOL


def test_fused_log_probability_entry_point(ctx):
    from ctypes import byref, c_double
    from tinygp_b200 import _cabi
    rng = np.random.default_rng(5)
    n = 900
    X = np.ascontiguousarray(rng.uniform(0, 8, (n, 3)))
    y = np.sin(X[:, 0])
    diag = np.full(n, 0.1)
    k = kernels.ExpSquared(1.0)
    prog = k.program()
    lp = c_double()
    ctx.check(ctx.lib.b200gp_dense_log_probability(ctx.handle, _cabi.ptr(prog), prog.shape[0], _cabi.ptr(X), n, 3,
                                                   _cabi.ptr(diag), _cabi.ptr(y), byref(lp)))
    lpo = o.GaussianProcess(to_oracle(k), X, diag=0.1).log_probability(y)
    assert rel(lp.value, lpo) < LOGP_RTOL


def test_solves_and_products():
    rng = np.random.default_rng(7)
    n = 700
    X = rng.uniform(0, 8, (n, 3))
    k = kernels.Matern32(2.0, kernels.L2Distance())
    s = solvers.DirectSolver(k, X, noise.Diagonal(np.full(n, 0.1)))
    L = np.linalg.cholesky(to_oracle(k)(X, X) + 0.1 * np.eye(n))
    y = rng.normal(size=n)
    Y = rng.normal(size=(n, 5))
    np.testing.assert_allclose(s.solve_triangular(y), scipy.linalg.solve_triangular(L, y, lower=True),
                               rtol=1e-9, atol=1e-11)
    np.testing.assert_allclose(s.solve_triangular(y, transpose=True),
                               scipy.linalg.solve_triangular(L, y, lower=True, trans=1), rtol=1e-9, atol=1e-11)
    np.testing.assert_allclose(s.solve_triangular(Y), scipy.linalg.solve_triangular(L, Y, lower=True),
                               rtol=1e-9, atol=1e-11)
    np.testing.assert_allclose(s.solve_triangular(Y, transpose=True),
                               scipy.linalg.solve_triangular(L, Y, lower=True, trans=1), rtol=1e-9, atol=1e-11)
    np.testing.assert_allclose(s.dot_triangular(y), L @ y, rtol=1e-11, atol=1e-12)
    Z = rng.normal(size=(n, 3, 2))
    np.testing.assert_allclose(s.dot_triangular(Z), np.einsum("ij,j...->i...", L, Z), rtol=1e-11, atol=1e-12)
    # tests/test_kernels/test_kernels.py:72-83
    Kinv_y = s.solve_triangular(s.solve_triangular(y), transpose=True)
    np.testing.assert_allclose(Kinv_y, np.linalg.solve(L @ L.T, y), rtol=1e-8, atol=1e-10)


@pytest.mark.parametrize("n,m", [(300, 40), (500, 200)])
def test_condition_and_predict(n, m):
    rng = np.random.default_rng(11)
    X = rng.uniform(0, 6, (n, 2))
    Xt = rng.uniform(0, 6, (m, 2))
    y = np.sin(X[:, 0]) + 0.1 * rng.normal(size=n)
    k = 1.5 * kernels.Matern52(2.0, kernels.L2Distance())
    gp = GaussianProcess(k, X, diag=0.1, mean=0.2)
    gpo = o.GaussianProcess(to_oracle(k), X, diag=0.1, mean=0.2)
    lp, cond = gp.condition(y, Xt, diag=0.05)
    lpo, condo = gpo.condition(y, Xt, diag=0.05)
    assert rel(lp, lpo) < LOGP_RTOL
    assert_close(cond.loc, condo.loc)
    assert_close(cond.covariance, condo.covariance)
    assert_close(cond.variance, condo.variance)
    # conditioned GP is itself a working GP (second M x M Cholesky, gp.py:208-221)
    yt = rng.normal(size=m)
    assert rel(cond.log_probability(yt), condo.log_probability(yt)) < 1e-7
    # predict at the inputs (noise shortcut) and with return_var / return_cov
    assert_close(gp.predict(y), gpo.predict(y))
    mu, var = gp.predict(y, Xt, return_var=True)
    muo, varo = gpo.predict(y, Xt, return_var=True)
    assert_close(mu, muo)
    assert_close(var, varo)
    mu, cov = gp.predict(y, return_cov=True, include_mean=False)
    muo, covo = gpo.predict(y, return_cov=True, include_mean=False)
    assert_close(mu, muo)
    assert_close(cov, covo)
    with pytest.raises(ValueError):
        gp.condition(y, np.zeros((4, 3)))


def test_non_pd_gives_minus_inf():
    X = np.zeros((200, 1))
    gp = GaussianProcess(kernels.ExpSquared(1.0), X, diag=-2.0)
    assert gp.solver.info > 0
    assert gp.log_probability(np.ones(200)) == -np.inf
    # default jitter (gp.py:388-393) on distinct points is fine
    X = np.linspace(0, 100, 200)
    gp = GaussianProcess(kernels.Exp(1.0), X)
    gpo = o.GaussianProcess(o.Exp(1.0), X)
    assert rel(gp.log_probability(np.sin(X)), gpo.log_probability(np.sin(X))) < 1e-7


def test_reference_default_l1_metric_is_indefinite_in_3d():
    """Matern/RationalQuadratic default to the L1 metric (stationary.py:56); for D > 1 that matrix is
    not positive definite.  Reference behaviour: NaN factor -> log_probability = -inf (gp.py:316)."""
    rng = np.random.default_rng(7)
    X = rng.uniform(0, 8, (700, 3))
    y = np.sin(X[:, 0])
    k = kernels.Matern32(2.0)
    gp = GaussianProcess(k, X, diag=0.1)
    gpo = o.GaussianProcess(to_oracle(k), X, diag=0.1)
    assert gpo.log_probability(y) == -np.inf
    assert gp.solver.info > 0 and gp.log_probability(y) == -np.inf


def test_sampling_statistics():
    # tests/test_gp.py:24-38 (statistical parity only: the RNG stream differs from JAX's)
    rng = np.random.default_rng(1058390)
    X = np.sort(rng.uniform(-3, 3, 30))
    gp = GaussianProcess(kernels.Matern32(1.5), X, diag=0.01, mean=0.5)
    y = gp.sample(123, shape=(50_000,))
    assert y.shape == (50_000, 30)
    assert np.allclose(np.mean(y, axis=0), 0.5, atol=0.02)
    assert np.allclose(np.cov(y, rowvar=False), gp.covariance, atol=0.03)
    assert gp.sample(1).shape == (30,)


@pytest.mark.parametrize("slices", [8, 0])
def test_large_n_properties(ctx, slices):
    """N = 8192: parity against the oracle (LAPACK dpotrf, ~3 s) plus size-independent identities, for the int8
    fixed-point trailing update (8 digit planes, forced on with ozaki_min_n = 0) and for the native fp64 DMMA path
    (the default)."""
    ctx.set_option("ozaki_slices", slices)
    if slices:
        ctx.set_option("ozaki_min_n", 0)
    rng = np.random.default_rng(49382)
    n = 8192
    X = rng.uniform(0, 10, (n, 3))
    y = np.sin(X[:, 0]) + 0.1 * rng.normal(size=n)
    k = 1.0 * kernels.ExpSquared(1.0)
    gp = GaussianProcess(k, X, diag=0.1)
    lp = gp.log_probability(y)
    lpo = o.GaussianProcess(to_oracle(k), X, diag=0.1).log_probability(y)
    assert rel(lp, lpo) < LOGP_RTOL, (lp, lpo)
    # L (L^T (L^-T (L^-1 y))) == y   and   |L z|^2 == z^T K z
    a = gp.solver.solve_triangular(gp.solver.solve_triangular(y), transpose=True)
    back = gp.solver.dot_triangular(gp.solver.solve_triangular(y))
    np.testing.assert_allclose(back, y, rtol=1e-9, atol=1e-10)
    # K (K^-1 y) == y with K applied by the matrix-free kernel matvec
    np.testing.assert_allclose(k.matmul(X, X, a) + 0.1 * a, y, rtol=1e-8, atol=1e-9)
    assert rel(y @ a, np.sum(gp.solver.solve_triangular(y) ** 2)) < 1e-10
    ctx.reset_options()


def test_batched_hyperparameter_grid(ctx):
    """BASELINE config 5 in miniature: B kernels over one (X, y); each entry equals its own log_probability."""
    from ctypes import c_void_p
    from tinygp_b200 import _cabi
    rng = np.random.default_rng(49385)
    n = 900
    X = np.ascontiguousarray(rng.uniform(0, 8, (n, 3)))
    y = np.sin(X[:, 0]) + 0.1 * rng.normal(size=n)
    diag = np.full(n, 0.1)
    grid = [(s, a) for s in (0.5, 1.0, 2.0) for a in (0.3, 1.0, 4.0)]
    ks = [a * kernels.ExpSquared(scale=s) for s, a in grid]
    progs = np.ascontiguousarray(np.stack([k.program() for k in ks]))
    out = np.empty(len(ks))
    for nb in (128, 512, 4096):
        ctx.set_option("nb_batched", nb)
        ctx.check(ctx.lib.b200gp_dense_log_probability_batched(
            ctx.handle, _cabi.ptr(progs), progs.shape[1], len(ks), _cabi.ptr(X), n, 3, _cabi.ptr(diag), _cabi.ptr(y),
            _cabi.ptr(out)))
        for k, got in zip(ks, out):
            want = o.GaussianProcess(to_oracle(k), X, diag=0.1).log_probability(y)
            assert rel(got, want) < LOGP_RTOL, (got, want)
    ctx.set_option("nb_batched", 4096)       # the library default
    # a non-PD member of the batch gives -inf without disturbing the others
    bad = np.ascontiguousarray(np.stack([ks[0].program(), (-1.0 * kernels.ExpSquared(1.0)).program()]))
    out2 = np.empty(2)
    ctx.check(ctx.lib.b200gp_dense_log_probability_batched(
        ctx.handle, _cabi.ptr(bad), bad.shape[1], 2, _cabi.ptr(X), n, 3, _cabi.ptr(diag), _cabi.ptr(y), _cabi.ptr(out2)))
    assert out2[1] == -np.inf and rel(out2[0], out[0]) < 1e-12
    # a batch whose members are NOT one common single-leaf kernel: the interpreter builds it (lower triangle only)
    L2 = kernels.L2Distance()
    mixed = [1.3 * kernels.ExpSquared(0.8), 0.7 * kernels.Matern32(1.5, L2), 1.1 * kernels.Matern52(2.0, L2)]
    pm = np.ascontiguousarray(np.stack([k.program() for k in mixed]))
    out3 = np.empty(3)
    ctx.check(ctx.lib.b200gp_dense_log_probability_batched(
        ctx.handle, _cabi.ptr(pm), pm.shape[1], 3, _cabi.ptr(X), n, 3, _cabi.ptr(diag), _cabi.ptr(y), _cabi.ptr(out3)))
    for k, got in zip(mixed, out3):
        want = o.GaussianProcess(to_oracle(k), X, diag=0.1).log_probability(y)
        assert rel(got, want) < LOGP_RTOL, (got, want)
    # larger problems (interior build tiles, several panels): Matern-5/2 grid on the specialised batched build
    n2 = 2304
    X2 = np.ascontiguousarray(rng.uniform(0, 10, (n2, 2)))
    y2 = np.cos(X2[:, 1]) + 0.1 * rng.normal(size=n2)
    d2 = np.full(n2, 0.05)
    ks2 = [a * kernels.Matern52(s, L2) for s, a in ((0.7, 0.5), (1.5, 2.0))]
    p2 = np.ascontiguousarray(np.stack([k.program() for k in ks2]))
    out4 = np.empty(2)
    ctx.check(ctx.lib.b200gp_dense_log_probability_batched(
        ctx.handle, _cabi.ptr(p2), p2.shape[1], 2, _cabi.ptr(X2), n2, 2, _cabi.ptr(d2), _cabi.ptr(y2), _cabi.ptr(out4)))
    for k, got in zip(ks2, out4):
        want = o.GaussianProcess(to_oracle(k), X2, diag=0.05).log_probability(y2)
        assert rel(got, want) < LOGP_RTOL, (got, want)
