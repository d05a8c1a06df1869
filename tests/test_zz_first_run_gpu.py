"""GPU cases for the newer device code paths.  This file sorts late so that a surprise here cannot hide the other results
under `pytest -x`:
  * QuasisepSolver conditioning on the device (`b200gp_qs_condition`), diag((K + N)^-1) and the O(N) conditioned variance
    (GramBack backward scan; its source passes on the CPU in tests/test_device_code_on_host.py);
  * the K-range split of the int8 update, the build-ahead option, the warp-shuffle tree option;
The reference-golden / restated-reference cases that depend on this code follow in test_zzy_*, the changed and new int8
kernel variants in test_zzz_*."""

import numpy as np
import pytest

from oracle import tinygp_np as o
from tinygp_b200 import GaussianProcess
from tinygp_b200.kernels import quasisep as Q
from util import LOGP_RTOL, rel, to_oracle

pytestmark = pytest.mark.gpu

KERNELS = {
    "sho+m32": Q.SHO(1.5, 3.0, 1.8) + Q.Matern32(1.5, 0.9),
    "m52": Q.Matern52(2.5, 1.3),
    "exp": Q.Exp(1.7, 0.8),
    "sum3": 2.0 * Q.Matern32(1.2) + Q.SHO(0.8, 4.0, 0.6) + 0.5 * Q.Exp(5.0),
}


def _data(n, seed=3):
    rng = np.random.default_rng(seed)
    t = np.sort(rng.uniform(0, n / 8.0, n))
    return t, np.sin(t) + 0.1 * rng.normal(size=n), rng.uniform(0.05, 0.2, n)


@pytest.mark.parametrize("n", [1, 63, 700, 4099])
@pytest.mark.parametrize("name", list(KERNELS))
def test_inverse_diagonal_parity(name, n):
    t, y, noise = _data(n)
    gp = GaussianProcess(KERNELS[name], t, diag=noise)
    got = gp.solver.inverse_diagonal()
    so = o.QuasisepSolver(to_oracle(KERNELS[name]), t, o.Diagonal(noise))
    if n <= 700:
        want = np.diag(np.linalg.inv(so.covariance()))
    else:
        idx = np.unique(np.r_[0, 1, n // 2, n - 2, n - 1, np.random.default_rng(1).integers(0, n, 12)])
        E = np.zeros((n, idx.size)); E[idx, np.arange(idx.size)] = 1.0
        want = so.solve_triangular(so.solve_triangular(E), transpose=True)[idx, np.arange(idx.size)]
        got = got[idx]
    np.testing.assert_allclose(got, want, rtol=1e-9, atol=0)


@pytest.mark.parametrize("name", list(KERNELS))
def test_predict_variance_at_the_inputs_is_the_reference_qsm_branch(name):
    """gp.predict(y, return_var=True): solver.py:124-129 read by :84-85, here by one backward scan"""
    t, y, noise = _data(200)
    mu, var = GaussianProcess(KERNELS[name], t, diag=noise).predict(y, return_var=True)
    muo, varo = o.GaussianProcess(to_oracle(KERNELS[name]), t, diag=noise).predict(y, return_var=True)
    np.testing.assert_allclose(mu, muo, rtol=5e-7, atol=5e-7)
    np.testing.assert_allclose(var, varo, rtol=1e-8, atol=1e-12)


def test_large_series_smoothing_variance_is_linear_time():
    """N = 2e6: no N x N matrix anywhere; the variance lies between 0 and the prior variance + jitter and equals
    the dense value on a window far from the ends (the process decorrelates over a few time scales)."""
    n = 2_000_000
    t, y, noise = _data(n, seed=5)
    k = KERNELS["sho+m32"]
    gp = GaussianProcess(k, t, diag=noise)
    mu, var = gp.predict(y, return_var=True)
    assert mu.shape == var.shape == (n,) and np.all(np.isfinite(var))
    prior = 1.8 ** 2 + 0.9 ** 2
    assert var.min() > 0.0 and var.max() < prior + 1e-6
    # a 3000-point window (~375 time units >> every time scale of the kernel) treated as its own GP -- the small-N path,
    # whose parity with the oracle is the test above -- must agree with the full series away from the window's ends
    lo, hi = n // 2 - 1500, n // 2 + 1500
    muw, varw = GaussianProcess(k, t[lo:hi], diag=noise[lo:hi]).predict(y[lo:hi], return_var=True)
    mid = slice(1000, 2000)
    np.testing.assert_allclose(var[lo:hi][mid], varw[mid], rtol=1e-6, atol=1e-10)
    np.testing.assert_allclose(mu[lo:hi][mid], muw[mid], rtol=1e-6, atol=1e-8)


def _data_sorted(n, seed=84930):
    rng = np.random.default_rng(seed)
    X = np.sort(rng.uniform(-3, 3, n))
    return X, np.sin(X), rng


def test_condition_dense_branch():
    # solver.py:131-139 via gp.condition with X_test
    X, y, rng = _data_sorted(120)
    Xt = np.sort(rng.uniform(-3, 3, 30))
    k = Q.SHO(1.5, 3.0, 1.8) + Q.Matern32(1.5, 0.9)
    lp, cond = GaussianProcess(k, X, diag=0.1).condition(y, Xt)
    ko = to_oracle(k)
    lpo, condo = o.GaussianProcess(ko, X, diag=0.1).condition(y, Xt)
    assert rel(lp, lpo) < LOGP_RTOL
    np.testing.assert_allclose(cond.loc, condo.loc, rtol=5e-7, atol=5e-7)
    np.testing.assert_allclose(cond.covariance, condo.covariance, rtol=5e-7, atol=5e-7)


def test_predict_at_test_points_parity():
    """gp.predict(y, X_test) through QuasisepSolver: mean by the O(n + m) general product (gp.py:357), variance by
    the dense branch (solver.py:131-139) with the kernel evaluated on the device."""
    X, y, rng = _data_sorted(200)
    Xt = rng.uniform(-3.5, 3.5, 60)                  # unsorted, partly extrapolating
    k = Q.SHO(1.5, 3.0, 1.8) + Q.Matern32(1.5, 0.9)
    mu, var = GaussianProcess(k, X, diag=0.1).predict(y, Xt, return_var=True)
    muo, varo = o.GaussianProcess(to_oracle(k), X, diag=0.1).predict(y, Xt, return_var=True)
    np.testing.assert_allclose(mu, muo, rtol=5e-7, atol=5e-7)
    np.testing.assert_allclose(var, varo, rtol=5e-7, atol=5e-7)


def test_int8_update_splits_k_ranges_beyond_the_int32_bound(ctx):
    """|accumulator| <= S * 4096 * K must stay below 2^31: K = 75264 > 74880 (S = 7) is run as two exact segments.
    Two rows carry +64 in every digit -- the worst case the bound is about -- so a single unsplit launch WOULD wrap
    (7 * 4096 * 75264 > 2^31 - 1); the result must still equal the integer-exact reference."""
    from tinygp_b200 import _cabi
    S, rows, K = 7, 256, 75264
    rng = np.random.default_rng(11)
    planes = rng.integers(-64, 65, size=(S, rows, K), dtype=np.int8)
    planes[:, :2, :] = 64                        # rows 0 and 1: every digit of every plane is +64
    rs = np.ones(rows)
    C = rng.normal(size=(rows, rows))
    got = C.copy()
    pl = np.ascontiguousarray(planes)
    ctx.check(ctx.lib.b200gp_i8_update_test(ctx.handle, _cabi.ptr(pl), S, rows, K, _cabi.ptr(rs), _cabi.ptr(got)))
    want = C.copy()
    P = planes.astype(np.float64)                # integer sums < 2^53: the BLAS products below are exact
    for s in range(S):
        for t in range(S - s):
            want -= 2.0 ** -(12 + 7 * (s + t)) * (P[s] @ P[t].T)
    assert sum(float(P[s][0] @ P[6 - s][1]) for s in range(7)) > 2 ** 31 - 1   # the last digit group, unsplit, wraps
    np.testing.assert_allclose(got, want, rtol=0, atol=1e-12 * max(1.0, np.abs(want).max()))


@pytest.mark.parametrize("n", [3000, 2600])         # nb = 512: six full panels; five and a last one of 128 columns
def test_build_ahead_option_gives_the_same_factorisation(ctx, n):
    """option build_ahead (block column J+1 is generated on a side stream under the int8 update of column J): a pure
    reordering of independent work, so the result must be bit-identical to the serial order"""
    from tinygp_b200 import kernels
    rng = np.random.default_rng(17)
    X = rng.uniform(0, 20.0 * (n / 65536.0) ** (1 / 3), (n, 3))
    y = np.sin(X[:, 0]) + 0.1 * rng.normal(size=n)
    k = 1.3 * kernels.ExpSquared(0.8)
    ctx.set_option("nb", 512)
    ctx.set_option("ozaki_min_n", 0)
    ctx.set_option("ozaki_slices", 7)
    out = []
    try:
        ctx.set_option("ozaki_subpanel", 0)      # one fp64 panel per block column: 4 diagonal tiles per look-ahead chain
        for ahead in (0, 1):
            ctx.set_option("build_ahead", ahead)
            out.append(GaussianProcess(k, X, diag=0.1).log_probability(y))
    finally:
        ctx.reset_options()
    assert out[0] == out[1], out
    lpo = o.GaussianProcess(to_oracle(k), X, diag=0.1).log_probability(y)
    assert rel(out[0], lpo) < LOGP_RTOL


@pytest.mark.parametrize("n", [40, 700, 40000])
@pytest.mark.parametrize("name", ["sho+m32", "m52", "sum3"])
def test_warp_shuffle_tree_option(ctx, name, n):
    """option qs_tree = 1: the chunk composites are scanned by warp-shuffle (Hillis-Steele, fan-in 32) kernels instead
    of the thread-sequential fan-in-16 tree; factor, solves, log-probability and the inverse diagonal must keep parity"""
    t, y, noise = _data(n, seed=n)
    k = KERNELS[name]
    so = o.QuasisepSolver(to_oracle(k), t, o.Diagonal(noise))
    ctx.set_option("qs_tree", 1)
    ctx.set_option("qs_chunk", 4 if n <= 700 else 64)        # small chunks -> several tree levels at small n
    try:
        gp = GaussianProcess(k, t, diag=noise)
        c, w = gp.solver.factor_arrays()
        lp = gp.log_probability(y)
        a = gp.solver.solve_triangular(y)
        at = gp.solver.solve_triangular(a, transpose=True)
        inv = gp.solver.inverse_diagonal()
    finally:
        ctx.set_option("qs_tree", 0)
        ctx.set_option("qs_chunk", 64)
    np.testing.assert_allclose(c, so.c, rtol=1e-10, atol=0)
    np.testing.assert_allclose(w, so.w, rtol=1e-9, atol=1e-12)
    ao = so.solve_triangular(y)
    np.testing.assert_allclose(a, ao, rtol=1e-8, atol=1e-11)
    np.testing.assert_allclose(at, so.solve_triangular(ao, transpose=True), rtol=1e-8, atol=1e-11)
    lpo = -0.5 * ao @ ao - so.normalization()
    assert rel(lp, lpo) < LOGP_RTOL
    idx = np.unique(np.r_[0, n // 2, n - 1])
    E = np.zeros((n, idx.size)); E[idx, np.arange(idx.size)] = 1.0
    want = so.solve_triangular(so.solve_triangular(E), transpose=True)[idx, np.arange(idx.size)]
    np.testing.assert_allclose(inv[idx], want, rtol=1e-9, atol=0)
