"""GaussianProcess.fisher_information on the GPU: parity with the LAPACK / complex-step Fisher information of
oracle/fisher_np.py on the native fp64 and the int8-update factorisations, bitwise symmetry and reproducibility, non
positive-definite input, and an exact identity at n = 32768."""

import numpy as np
import pytest

from oracle import fisher_np
from oracle import tinygp_np as o
from tinygp_b200 import GaussianProcess, _cabi, kernels, transforms

pytestmark = pytest.mark.gpu

CASES = {   # the kernel families of test_grad_gpu.py
    "expsq_const": (lambda m: 1.3 * m.ExpSquared(0.9) + 0.2, 3),
    "exp_matern": (lambda m: m.Exp(1.1) + m.Matern32(0.8, distance=m.L2Distance()) * m.Matern52(1.4), 2),
    "periodic": (lambda m: m.Cosine(2.5) + m.ExpSineSquared(1.7, gamma=0.6) * m.RationalQuadratic(0.9, distance=m.L2Distance(), alpha=1.3), 1),
    "rq_l1": (lambda m: m.RationalQuadratic(1.2, alpha=0.8) + 0.5 * m.ExpSquared(1.4, distance=m.L1Distance()), 1),
    "ard": (lambda m: 1.5 * m.Linear(np.array([0.5, 1.5, 2.0]), m.ExpSquared())
            + m.Subspace(1, m.Exp(0.7)) + m.Subspace([0, 2], m.Cholesky(np.array([0.8, 1.1]), m.Matern52(1.2, distance=m.L2Distance()))), 3),
    "linear0d": (lambda m: m.Cholesky(0.9, m.Linear(0.7, m.Matern32(1.0))) * m.ExpSineSquared(3.0, gamma=0.4), 1),
}


class _P:
    Exp, ExpSquared, Matern32, Matern52 = kernels.Exp, kernels.ExpSquared, kernels.Matern32, kernels.Matern52
    Cosine, ExpSineSquared, RationalQuadratic = kernels.Cosine, kernels.ExpSineSquared, kernels.RationalQuadratic
    L1Distance, L2Distance = kernels.L1Distance, kernels.L2Distance
    Linear, Cholesky, Subspace = transforms.Linear, transforms.Cholesky, transforms.Subspace


def _data(dim, n, seed=3):
    rng = np.random.default_rng(seed)
    side = 3.0 * (n / 300.0) ** (1.0 / dim)
    X = rng.uniform(0, side, n) if dim == 1 else rng.uniform(0, side, (n, dim))
    return X, rng.uniform(0.1, 0.3, n)


_ORACLE = {}


def _check(name, n, scalar_diag=True):
    build, dim = CASES[name]
    X, dvec = _data(dim, n)
    diag = 0.2 if scalar_diag else dvec
    F = GaussianProcess(build(_P), X, diag=diag).fisher_information()
    key = (name, n, scalar_diag)
    if key not in _ORACLE:
        _ORACLE[key] = fisher_np.fisher(build(o), X, diag)
    labels, Fo = _ORACLE[key]
    idx = {lab: i for i, lab in enumerate(labels)}
    assert sorted(idx, key=str) == sorted(F.params, key=str)
    perm = [idx[lab] for lab in F.params]
    ref = Fo[np.ix_(perm, perm)]
    err = np.max(np.abs(F.matrix - ref)) / np.max(np.abs(ref))
    assert err <= 1e-9, (name, n, err)
    assert np.array_equal(F.matrix, F.matrix.T)


@pytest.mark.parametrize("n", [300, 1000, 2500])
@pytest.mark.parametrize("name", list(CASES))
def test_fisher_matches_oracle(name, n):
    _check(name, n)


@pytest.mark.parametrize("n", [300, 1000, 2500])
@pytest.mark.parametrize("name", ["expsq_const", "ard", "periodic"])
def test_fisher_matches_oracle_int8_update(name, n):
    ctx = _cabi.get_context()
    ctx.set_option("ozaki_min_n", 0)
    ctx.set_option("nb", 256)
    try:
        _check(name, n)
    finally:
        ctx.reset_options()


@pytest.mark.parametrize("name", ["exp_matern", "ard"])
def test_fisher_per_point_diag(name):
    _check(name, 1000, scalar_diag=False)


def test_bitwise_symmetric_reproducible_and_solver_untouched():
    X, d = _data(3, 1500)
    gp = GaussianProcess(CASES["ard"][0](_P), X, diag=d)
    y = np.sin(X[:, 0])
    before = gp.log_probability(y)
    F1 = gp.fisher_information()
    F2 = gp.fisher_information()
    assert np.array_equal(F1.matrix, F1.matrix.T)
    assert np.array_equal(F1.matrix, F2.matrix) and F1.params == F2.params
    assert gp.log_probability(y) == before


def test_non_pd_gives_nan():
    X = np.linspace(0, 1, 200)
    F = GaussianProcess(kernels.ExpSquared(1.0) + 0.3, X, diag=-0.5).fisher_information()
    assert F.matrix.shape == (3, 3) and np.all(np.isnan(F.matrix))


def test_scale_identity_at_32768():
    """c * k with a scalar diag d: c dK/dc + d dK/dd = K, so v^T F v = 1/2 tr(W K W K) = n / 2 for v = (c, d)"""
    n, c, d = 32768, 1.3, 0.5
    X = np.random.default_rng(11).uniform(0, 100, n)
    F = GaussianProcess(c * kernels.ExpSquared(0.05), X, diag=d).fisher_information()
    assert F.params == [("kernel1.value", None), ("kernel2.scale", None), ("diag", None)]
    v = np.array([c, 0.0, d])
    got = v @ F.matrix @ v
    print(f"n={n}: v^T F v = {got!r}, n / 2 = {n / 2}")
    assert got == pytest.approx(n / 2, rel=1e-10)
