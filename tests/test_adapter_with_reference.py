"""The plugin boundary, literally: the UNMODIFIED reference `tinygp.GaussianProcess` (from /root/reference, over the
NumPy stand-ins for jax/equinox in tests/golden/jaxshim) driven with `solver=tinygp_b200.adapter.DirectSolver /
QuasisepSolver`.  tinygp's own gp.py makes every call (constructor with `covariance=`, the six Solver methods, the
Conditioned kernel calling back into `solve_triangular`); the tinygp_b200 host layer answers, here over the mock C-ABI
(tests/hostmock.py) because this container has no GPU and the GPU box has no reference checkout.  Results must equal
what the reference computes with its own solvers."""

import os
import sys
from ctypes import c_void_p

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
sys.path.insert(0, os.path.join(HERE, "golden"))

import refimport  # noqa: E402

if not refimport.available():
    pytest.skip("the reference checkout (/root/reference) is not present on this machine", allow_module_level=True)

import hostmock  # noqa: E402
from tinygp_b200 import _cabi, adapter  # noqa: E402


@pytest.fixture()
def tinygp(monkeypatch):
    saved = list(sys.path)
    mods = set(sys.modules)
    tg = refimport.install()
    lib = hostmock.MockLib()
    ctx = _cabi.Context.__new__(_cabi.Context)
    ctx.lib, ctx.handle, ctx.device = lib, c_void_p(1), -1
    previous = _cabi._ctx
    _cabi.set_context(ctx)
    try:
        yield tg
    finally:
        _cabi.set_context(previous)
        sys.path[:] = saved
        for m in set(sys.modules) - mods:          # do not leak the stand-in `jax` into other test modules
            if m.split(".")[0] in ("jax", "equinox", "tinygp"):
                del sys.modules[m]


def _close(a, b, tol=1e-9):
    a, b = np.asarray(a, dtype=np.float64), np.asarray(b, dtype=np.float64)
    assert a.shape == b.shape and np.all(np.isfinite(b)), "the reference itself must be finite for this comparison"
    assert np.max(np.abs(a - b)) <= tol * max(1.0, np.max(np.abs(b))), (np.max(np.abs(a - b)))


DENSE = [
    "1.7 * kernels.ExpSquared(0.9)",
    "kernels.Matern32(1.3, distance=kernels.L2Distance()) + 0.3 * kernels.RationalQuadratic(scale=1.5, alpha=0.8)",
    "kernels.Exp(1.3) * kernels.ExpSquared(3.0) + 0.05",
    "transforms.Subspace(0, kernels.ExpSquared(1.2)) + 0.5 * transforms.Linear(np.array([0.7, 1.4]), kernels.Matern52(0.9))",
]


@pytest.mark.parametrize("expr", DENSE)
def test_reference_gaussian_process_with_b200_direct_solver(tinygp, expr):
    from tinygp import GaussianProcess, kernels, transforms
    rng = np.random.default_rng(3)
    X, Xt = rng.uniform(0, 4, (40, 2)), rng.uniform(0, 4, (6, 2))
    y = np.sin(X[:, 0]) + 0.1 * rng.normal(size=40)
    k = eval(expr, {"kernels": kernels, "transforms": transforms, "np": np})
    ref = GaussianProcess(k, X, diag=0.07, mean=0.2)
    ours = GaussianProcess(k, X, diag=0.07, mean=0.2, solver=adapter.DirectSolver)
    assert isinstance(ours.solver, adapter.DirectSolver)
    _close(ours.log_probability(y), ref.log_probability(y))
    _close(ours.variance, ref.variance)
    _close(ours.covariance, ref.covariance)
    lp_o, cond_o = ours.condition(y, Xt, diag=1e-3)
    lp_r, cond_r = ref.condition(y, Xt, diag=1e-3)
    _close(lp_o, lp_r)
    _close(cond_o.loc, cond_r.loc)
    _close(cond_o.variance, cond_r.variance)          # tinygp's Conditioned kernel calls back into our solve_triangular
    _close(cond_o.covariance, cond_r.covariance)
    _close(cond_o.log_probability(np.cos(Xt[:, 0])), cond_r.log_probability(np.cos(Xt[:, 0])))
    mu_o, var_o = ours.predict(y, return_var=True)
    mu_r, var_r = ref.predict(y, return_var=True)
    _close(mu_o, mu_r)
    _close(var_o, var_r)
    import jax
    _close(ours.sample(jax.random.PRNGKey(4), shape=(3,)), ref.sample(jax.random.PRNGKey(4), shape=(3,)))


QS = [
    "quasisep.SHO(omega=1.5, quality=3.0, sigma=1.8) + quasisep.Matern32(scale=1.5, sigma=0.9)",
    "2.0 * quasisep.Matern52(1.2) + quasisep.Celerite(1.1, 0.1, 0.3, 1.5)",
    "quasisep.Cosine(scale=3.0, sigma=0.7) + quasisep.Exp(scale=2.0, sigma=0.5)",
]


@pytest.mark.parametrize("expr", QS)
def test_reference_gaussian_process_with_b200_quasisep_solver(tinygp, expr):
    from tinygp import GaussianProcess
    from tinygp.kernels import quasisep
    rng = np.random.default_rng(5)
    t = np.sort(rng.uniform(0, 12, 60))
    tt = rng.uniform(-1, 13, 5)
    y = np.sin(t) + 0.1 * rng.normal(size=60)
    k = eval(expr, {"quasisep": quasisep})
    ref = GaussianProcess(k, t, diag=0.07)
    ours = GaussianProcess(k, t, diag=0.07, solver=adapter.QuasisepSolver, parallel=True)
    _close(ours.log_probability(y), ref.log_probability(y))
    _close(ours.variance, ref.variance)
    lp_o, cond_o = ours.condition(y, tt, diag=1e-3)
    lp_r, cond_r = ref.condition(y, tt, diag=1e-3)
    _close(lp_o, lp_r)
    _close(cond_o.loc, cond_r.loc)
    _close(cond_o.variance, cond_r.variance)
    _close(cond_o.covariance, cond_r.covariance)
    with pytest.raises(ValueError, match="Input coordinates must be sorted"):
        GaussianProcess(k, t[::-1].copy(), diag=0.07, solver=adapter.QuasisepSolver)


def test_unsupported_objects_are_refused_loudly(tinygp):
    from tinygp import GaussianProcess, kernels, noise
    X = np.linspace(0, 1, 5)
    with pytest.raises(NotImplementedError, match="unsupported by the B200"):
        GaussianProcess(kernels.DotProduct(), X, diag=0.1, solver=adapter.DirectSolver)


def test_reference_gaussian_process_with_banded_and_dense_noise(tinygp):
    """the reference's own noise.Banded / noise.Dense objects (noise.py:98-240) through the adapter's solvers"""
    from tinygp import GaussianProcess, kernels, noise
    from tinygp.kernels import quasisep
    rng = np.random.default_rng(8)
    t = np.sort(rng.uniform(0, 12, 50))
    tt, y = rng.uniform(-1, 13, 5), np.sin(t)
    banded = noise.Banded(diag=rng.uniform(0.1, 0.2, 50), off_diags=0.02 * rng.normal(size=(50, 2)))
    dense = noise.Dense(value=np.asarray(banded + np.zeros((50, 50))))
    kq = quasisep.Matern32(scale=1.5, sigma=1.8) + quasisep.Exp(scale=0.7)
    from tinygp.solvers import DirectSolver, QuasisepSolver
    for k, nz, theirs, solver in ((kq, banded, QuasisepSolver, adapter.QuasisepSolver),
                                  (kq, banded, DirectSolver, adapter.DirectSolver),
                                  (kernels.Matern52(1.1), dense, DirectSolver, adapter.DirectSolver)):
        ref, ours = GaussianProcess(k, t, noise=nz, solver=theirs), GaussianProcess(k, t, noise=nz, solver=solver)
        _close(ours.log_probability(y), ref.log_probability(y))
        _close(ours.covariance, ref.covariance)
        (lp_o, cond_o), (lp_r, cond_r) = ours.condition(y, tt, diag=1e-3), ref.condition(y, tt, diag=1e-3)
        _close(lp_o, lp_r)
        _close(cond_o.loc, cond_r.loc)
        _close(cond_o.covariance, cond_r.covariance)
