"""oracle/grad_x_np.py (d logp / d X with LAPACK and closed-form kernel gradients) against central differences of the
oracle's own log_probability with respect to single coordinates: several kernels, 1-D and 3-D, L1 and L2, ARD
transforms, products and sums; coincident points give a finite gradient."""

import numpy as np
import pytest

from oracle import grad_x_np
from oracle import tinygp_np as o

CASES = {
    "expsq_const_3d": (lambda: 1.3 * o.ExpSquared(0.9) + 0.2, 3),
    "exp_l1_matern_l2_2d": (lambda: o.Exp(1.1) + o.Matern32(0.8, distance=o.L2Distance()) * o.Matern52(1.4), 2),
    "periodic_1d": (lambda: o.Cosine(2.5) + o.ExpSineSquared(1.7, gamma=0.6)
                    * o.RationalQuadratic(0.9, distance=o.L2Distance(), alpha=1.3), 1),
    "rq_l1_expsq_l1_1d": (lambda: o.RationalQuadratic(1.2, alpha=0.8) + 0.5 * o.ExpSquared(1.4, distance=o.L1Distance()), 1),
    "exp_l2_3d": (lambda: 0.7 * o.Exp(1.3, distance=o.L2Distance()), 3),
    "ard_3d": (lambda: 1.5 * o.Linear(np.array([0.5, 1.5, 2.0]), o.ExpSquared())
               + o.Subspace(1, o.Exp(0.7))
               + o.Subspace([0, 2], o.Cholesky(np.array([0.8, 1.1]), o.Matern52(1.2, distance=o.L2Distance()))), 3),
    "scalar_transforms_1d": (lambda: o.Cholesky(0.9, o.Linear(0.7, o.Matern32(1.0))) * o.ExpSineSquared(3.0, gamma=0.4), 1),
}


def _data(dim, n=25, seed=11):
    rng = np.random.default_rng(seed)
    X = rng.uniform(0, 3, n) if dim == 1 else rng.uniform(0, 3, (n, dim))
    y = np.sin(2 * (X if dim == 1 else X[:, 0])) + 0.3 * rng.normal(size=n)
    return X, y, rng.uniform(0.1, 0.3, n)


@pytest.mark.parametrize("name", list(CASES))
def test_matches_central_differences(name):
    build, dim = CASES[name]
    X, y, diag = _data(dim)
    k = build()
    logp, dX, alpha = grad_x_np.log_probability_grad_x(k, X, y, diag, mean=0.1)
    f = lambda Xp: o.GaussianProcess(k, Xp, diag=diag, mean=0.1).log_probability(y)
    assert logp == pytest.approx(f(X), rel=1e-12)
    assert dX.shape == X.shape
    h = 1e-6
    for idx in [(0,), (7,), (24,)] if dim == 1 else [(0, 0), (7, dim - 1), (24, dim // 2), (13, 0)]:
        up, dn = X.copy(), X.copy()
        up[idx] += h
        dn[idx] -= h
        fd = (f(up) - f(dn)) / (2 * h)
        assert dX[idx] == pytest.approx(fd, rel=1e-6, abs=1e-7), (idx, dX[idx], fd)


def test_translation_invariance_and_duplicates():
    X, y, diag = _data(3)
    X[5] = X[3]                                      # a duplicate point: the pair contributes 0
    k = o.Exp(1.1, distance=o.L2Distance()) + o.Matern32(0.9)
    _, dX, _, scale = grad_x_np.log_probability_grad_x(k, X, y, diag, with_scale=True)
    assert np.all(np.isfinite(dX)) and np.all(np.isfinite(scale))
    assert np.linalg.norm(dX.sum(axis=0)) <= 1e-12 * np.sum(np.linalg.norm(dX, axis=1))
