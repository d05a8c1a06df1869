"""The Fisher-information oracle (oracle/fisher_np.py) against two independent restatements: the closed-form
derivative contraction of oracle/grad_np.py with the weight 1/2 W dK_b W, and the covariance of the score over draws of
y (the information identity F = Cov_y(grad logp)), by Monte Carlo."""

import numpy as np
import pytest

from oracle import fisher_np, grad_np
from oracle import tinygp_np as o

CASES = {
    "sum_product": (lambda: 1.3 * o.ExpSquared(0.9) * o.Matern32(1.7) + o.RationalQuadratic(1.1, alpha=0.7) + 0.2, 2),
    "ard_linear_l1": (lambda: 1.5 * o.Linear(np.array([0.5, 1.5, 2.0]), o.Matern52(1.1, distance=o.L1Distance())), 3),
    "cholesky_subspace": (lambda: o.Subspace([0, 2], o.Cholesky(np.array([0.8, 1.1]), o.Matern52(1.2, distance=o.L2Distance())))
                          + o.Subspace(1, o.Linear(0.6, o.ExpSineSquared(2.0, gamma=0.5))), 3),
    "nested_periodic": (lambda: o.Cholesky(0.9, o.Linear(np.array([1.4]), o.Exp(1.0))) * o.Cosine(5.0), 1),
}


def _data(dim, n, seed=2):
    rng = np.random.default_rng(seed)
    X = rng.uniform(0, 3, n) if dim == 1 else rng.uniform(0, 3, (n, dim))
    return X, rng


@pytest.mark.parametrize("name", list(CASES))
def test_matches_closed_form_contraction(name):
    build, dim = CASES[name]
    X, _ = _data(dim, 40)
    k = build()
    labels, F = fisher_np.fisher(k, X, 0.2)
    assert labels[-1] == ("diag", None) and np.array_equal(F, F.T)
    _, dK = fisher_np.derivatives(k, X)
    W = fisher_np.inverse(k, X, 0.2)
    D = X[:, None, None] - X[None, :, None] if X.ndim == 1 else X[:, None, :] - X[None, :, :]
    ents = fisher_np.params(k)
    for b, dKb in enumerate(dK):
        acc = {}
        grad_np._walk(k, D, 0.5 * W @ dKb @ W, acc, False)
        col = [acc[(id(node), field)][1] if idx is None else acc[(id(node), field)][1][idx] for _, node, field, idx in ents]
        col.append(0.5 * np.trace(W @ dKb @ W))
        np.testing.assert_allclose(F[:, b], col, rtol=1e-9, atol=1e-11 * np.max(np.abs(F)))


def test_derivatives_match_central_differences():
    k = 0.7 * o.Linear(np.array([0.5, 1.5]), o.RationalQuadratic(1.1, alpha=0.9)) + o.ExpSineSquared(1.3, gamma=0.4)
    X, _ = _data(2, 12)
    _, dK = fisher_np.derivatives(k, X, False)
    for (label, node, field, idx), d in zip(fisher_np.params(k), dK):
        old = np.array(getattr(node, field), dtype=np.float64)
        h = 1e-6 * max(1.0, abs(float(old if idx is None else old[idx])))
        mats = []
        for s in (h, -h):
            new = old.copy()
            if idx is None:
                new = new + s
            else:
                new[idx] += s
            setattr(node, field, float(new) if idx is None else new)
            mats.append(fisher_np.kernel_matrix(k, X))
        setattr(node, field, float(old) if idx is None else old)
        np.testing.assert_allclose(d, (mats[0] - mats[1]) / (2 * h), rtol=1e-6, atol=1e-8, err_msg=str(label))


def test_information_identity_by_monte_carlo():
    """F = Cov_y(grad logp) for y ~ N(0, K): every entry within 5 standard errors over 4000 draws at n = 60"""
    k = 1.2 * o.Matern32(0.8) + 0.3 * o.ExpSquared(2.0)
    X, rng = _data(1, 60, seed=7)
    labels, F = fisher_np.fisher(k, X, 0.15)
    lab2, g = fisher_np.score_samples(k, X, 0.15, 4000, rng)
    assert labels == lab2
    prod = g[:, :, None] * g[:, None, :]          # E[grad] = 0: the covariance is the mean of the products
    est, se = prod.mean(axis=0), prod.std(axis=0, ddof=1) / np.sqrt(g.shape[0])
    assert np.all(np.abs(est - F) <= 5 * se), (est, F, se)


def test_non_pd_gives_nan():
    _, F = fisher_np.fisher(o.ExpSquared(1.0), np.linspace(0, 1, 10), -0.5)
    assert np.all(np.isnan(F))


def test_labels_follow_the_tree():
    s = o.ExpSquared(1.0)
    k = o.Sum(o.Product(o.Constant(2.0), s), o.Linear(np.array([1.0, 2.0]), s))
    labels = [lab for lab, *_ in fisher_np.params(k)]
    assert labels == [("kernel1.kernel1.value", None), ("kernel1.kernel2.scale", None), ("kernel2.scale", 0),
                      ("kernel2.scale", 1)]
