"""oracle/grad_np.py (the closed-form log-likelihood gradient the device gradient is checked against) agrees with central
finite differences of the oracle's own log_probability."""

import numpy as np
import pytest

from oracle import grad_np
from oracle import tinygp_np as o

L2 = o.L2Distance
L1 = o.L1Distance


def _cases():
    return {
        "const_expsq_l2": (lambda: o.Constant(1.3) * o.ExpSquared(0.9) + o.Constant(0.2), 2),
        "exp_matern": (lambda: o.Exp(1.1) + o.Matern32(0.8, distance=L2()) * o.Matern52(1.4), 2),
        "periodic": (lambda: o.Cosine(2.5) + o.ExpSineSquared(1.7, gamma=0.6) * o.RationalQuadratic(0.9, distance=L2(), alpha=1.3), 1),
        "l1_squared": (lambda: o.RationalQuadratic(1.2, alpha=0.8) + 0.5 * o.ExpSquared(1.4, distance=L1()), 3),
        "l2_distance": (lambda: o.Exp(0.9, distance=L2()) * o.Cosine(3.0, distance=L2())
                        + o.ExpSineSquared(2.0, distance=L2(), gamma=1.1), 1),
        "linear_cholesky": (lambda: o.Linear(1.3, o.Matern32(1.0)) + o.Cholesky(np.array([0.7, 1.2]), o.ExpSquared(1.0)), 2),
        "ard_subspace": (lambda: 1.5 * o.Linear(np.array([0.5, 1.5, 2.0]), o.ExpSquared())
                         + o.Subspace(1, o.Exp(0.7)) + o.Subspace([0, 2], o.Linear(np.array([0.8, 1.1]), o.Matern52(1.2))), 3),
        "nested_cholesky": (lambda: o.Cholesky(0.9, o.Linear(np.array([1.4, 0.6]), o.RationalQuadratic(1.0, alpha=2.0))), 2),
        "scalar_coords": (lambda: o.ExpSineSquared(1.3, gamma=0.9) * o.ExpSquared(2.0) + o.Linear(0.7, o.Matern32(1.0)), 1),
    }


def _logp(kernel, X, y, diag):
    return o.GaussianProcess(kernel, X, diag=diag).log_probability(y)


def _data(dim, n=40, seed=0):
    rng = np.random.default_rng(seed)
    X = rng.uniform(0, 3, n) if dim == 1 else rng.uniform(0, 3, (n, dim))
    y = np.sin(2 * (X if dim == 1 else X[:, 0])) + 0.3 * rng.normal(size=n)
    return X, y, rng


def _fd(f, get, set_, h):
    v = get()
    set_(v + h)
    up = f()
    set_(v - h)
    dn = f()
    set_(v)
    return (up - dn) / (2 * h)


@pytest.mark.parametrize("name", list(_cases()))
@pytest.mark.parametrize("diag_kind", ["scalar", "per_point"])
def test_oracle_gradient_matches_finite_differences(name, diag_kind):
    build, dim = _cases()[name]
    X, y, rng = _data(dim)
    diag = 0.3 if diag_kind == "scalar" else rng.uniform(0.1, 0.5, X.shape[0])
    k = build()
    logp, grads, ddiag, alpha = grad_np.log_probability_grad(k, X, y, diag)
    assert logp == pytest.approx(_logp(k, X, y, diag), rel=1e-12)
    assert grads
    f = lambda: _logp(k, X, y, diag)
    for (_, field), (node, g) in grads.items():
        val = getattr(node, field)
        if np.ndim(val) == 0:
            h = 1e-5 * max(abs(float(val)), 1e-2)
            ref = _fd(f, lambda: getattr(node, field), lambda v: setattr(node, field, v), h)
            assert g == pytest.approx(ref, rel=1e-6, abs=1e-7), (field, g, ref)
        else:
            for i in range(val.shape[0]):
                h = 1e-5 * max(abs(float(val[i])), 1e-2)
                ref = _fd(f, lambda: float(val[i]), lambda v: val.__setitem__(i, v), h)
                assert g[i] == pytest.approx(ref, rel=1e-6, abs=1e-7), (field, i, g[i], ref)
    # noise and mean
    d = np.broadcast_to(np.asarray(diag, dtype=np.float64), y.shape).copy()
    for i in (0, 7, 31):
        h = 1e-6
        dd = d.copy()
        dd[i] += h
        up = _logp(k, X, y, dd)
        dd[i] -= 2 * h
        dn = _logp(k, X, y, dd)
        assert ddiag[i] == pytest.approx((up - dn) / (2 * h), rel=1e-6, abs=1e-8)
    yy = y.copy()
    yy[3] -= 1e-6
    up = _logp(k, X, yy, diag)
    yy[3] += 2e-6
    dn = _logp(k, X, yy, diag)
    assert alpha[3] == pytest.approx((up - dn) / 2e-6, rel=1e-6, abs=1e-8)      # d logp / d mean = -d logp / d y


def test_oracle_gradient_non_pd():
    X = np.zeros((5, 1))
    logp, grads, ddiag, alpha = grad_np.log_probability_grad(o.ExpSquared(1.0), X, np.ones(5), -1.0)
    assert logp == -np.inf and np.all(np.isnan(ddiag)) and np.all(np.isnan(alpha))
