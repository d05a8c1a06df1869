"""oracle/hessian_np.py, the observed Hessian of the log-likelihood, checked two independent ways: against central
differences of oracle/grad_np.py's closed-form gradient, and through the identity E_y[H] = -F by Monte Carlo against
oracle/fisher_np.py."""

import numpy as np
import pytest

from oracle import fisher_np, grad_np, hessian_np
from oracle import tinygp_np as o

CASES = {
    "sum_product": (lambda: 1.3 * o.ExpSquared(0.9) * o.Matern32(1.7) + o.RationalQuadratic(1.1, alpha=0.7) + 0.2, 2),
    "periodic_l1": (lambda: o.Cosine(2.5) + o.ExpSineSquared(1.7, gamma=0.6) * o.Exp(0.9, distance=o.L1Distance()), 1),
    "ard": (lambda: 1.5 * o.Linear(np.array([0.5, 1.5, 2.0]), o.ExpSquared())
            + o.Subspace([0, 2], o.Cholesky(np.array([0.8, 1.1]), o.Matern52(1.2, distance=o.L2Distance()))), 3),
    "nested_l1": (lambda: o.Cholesky(0.9, o.Linear(np.array([1.4]), o.RationalQuadratic(1.0, alpha=2.0)))
                  * o.Exp(1.3, distance=o.L1Distance()), 1),
}


def _data(dim, n=25, seed=2):
    rng = np.random.default_rng(seed)
    X = rng.uniform(0, 3, n) if dim == 1 else rng.uniform(0, 3, (n, dim))
    y = np.cos(X if dim == 1 else X[:, 0]) + 0.3 * rng.normal(size=n)
    return X, y


def _grad_vector(kernel, X, y, diag, plist):
    _, acc, ddiag, _ = grad_np.log_probability_grad(kernel, X, y, diag)
    g = []
    for _, node, field, idx in plist:
        v = acc.get((id(node), field), [None, 0.0])[1]
        g.append(float(v if idx is None else np.asarray(v)[idx]))
    return np.array(g + [np.sum(ddiag)])


@pytest.mark.parametrize("name", list(CASES))
def test_matches_central_differences_of_the_gradient(name):
    make, dim = CASES[name]
    X, y = _data(dim)
    k, diag = make(), 0.3
    labels, Hm = hessian_np.hessian(k, X, y, diag)
    plist = fisher_np.params(k)
    assert labels == [p[0] for p in plist] + [("diag", None)]
    assert np.array_equal(Hm, Hm.T)
    cols = []
    for b in range(len(labels)):
        h = 1e-5
        gs = []
        for s in (h, -h):
            if b < len(plist):
                _, node, field, idx = plist[b]
                old = getattr(node, field)
                new = np.array(old, dtype=np.float64)
                if idx is None:
                    new = new + s
                else:
                    new[idx] += s
                setattr(node, field, new if np.ndim(old) else np.float64(new))
                try:
                    gs.append(_grad_vector(k, X, y, diag, plist))
                finally:
                    setattr(node, field, old)
            else:
                gs.append(_grad_vector(k, X, y, diag + s, plist))
        cols.append((gs[0] - gs[1]) / (2 * h))
    fd = np.array(cols).T
    np.testing.assert_allclose(Hm, fd, rtol=1e-5, atol=1e-6 * np.max(np.abs(Hm)))


def test_expected_hessian_is_minus_fisher():
    """E_y[H] = -F for y ~ N(0, K): only the alpha alpha^T parts of H depend on y, with E[alpha alpha^T] = W"""
    k = 1.2 * o.ExpSquared(0.8) + 0.5 * o.Matern32(1.5)
    X, _ = _data(1, n=12, seed=4)
    diag = 0.2
    _, F = fisher_np.fisher(k, X, diag)
    K = fisher_np.kernel_matrix(k, X) + diag * np.eye(X.shape[0])
    L = np.linalg.cholesky(K)
    rng = np.random.default_rng(9)
    draws = [hessian_np.hessian(k, X, L @ rng.standard_normal(X.shape[0]), diag)[1] for _ in range(1500)]
    mean = np.mean(draws, axis=0)
    sem = np.std(draws, axis=0) / np.sqrt(len(draws))
    assert np.all(np.abs(mean + F) <= 5 * sem + 1e-12), (mean, -F, sem)


def test_non_pd_gives_nan():
    X = np.linspace(0, 1, 10)
    labels, Hm = hessian_np.hessian(o.ExpSquared(1.0) + 0.3, X, np.sin(X), -0.5)
    assert Hm.shape == (3, 3) and np.all(np.isnan(Hm))
