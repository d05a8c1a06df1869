"""The int8 fixed-point (Ozaki-style) trailing update on the wgmma tensor cores: exactness of the integer products, digit
cutting, and parity of the full factorisation against the oracle (run with -m gpu on an H100)."""

import numpy as np
import pytest

from oracle import tinygp_np as o
from tinygp_b200 import GaussianProcess, _cabi, kernels, noise, solvers
from util import LOGP_RTOL, rel, to_oracle

pytestmark = pytest.mark.gpu


def _ref_update(C, planes, rs, S):
    out = C.copy()
    P = planes.astype(np.float64)
    for s in range(S):
        for t in range(S - s):
            out -= 2.0 ** -(12 + 7 * (s + t)) * (rs[:, None] * rs[None, :]) * (P[s] @ P[t].T)
    return out


@pytest.mark.parametrize("layout", [0, 1])
@pytest.mark.parametrize("pairing", [0])      # paired-group kernels: tests/test_zz_first_run_gpu.py (changed after the last GPU run)
@pytest.mark.parametrize("cluster", [1, 2, 11, 21, 12, 22, 41, 42])
@pytest.mark.parametrize("rows,K,S", [(256, 128, 1), (256, 512, 3), (512, 1024, 8), (768, 384, 7), (512, 2048, 2)])
def test_i8_update_kernel_is_exact(ctx, rows, K, S, cluster, pairing, layout):
    """pairing: 0 = one digit group per pass (default), 1 = two groups per pass sharing their operand stages,
    2 = the paired loop structure with single groups (diagnostic).  layout: 0 = plane-major digit planes,
    1 = chunk-major (all planes of a 128-byte K chunk adjacent; one 4-D tensor map)."""
    if (pairing or layout) and cluster in (1, 2):
        pytest.skip("the wide variant has neither switch; the paired default launch is tested in test_zzz_*")
    ctx.set_option("ozaki_cluster", cluster)
    ctx.set_option("ozaki_pairing", pairing)
    ctx.set_option("ozaki_layout", layout)
    rng = np.random.default_rng(rows + K + S)
    planes = rng.integers(-64, 65, size=(S, rows, K), dtype=np.int8)
    rs = 2.0 ** rng.integers(-2, 3, size=rows).astype(np.float64)
    C = rng.normal(size=(rows, rows))
    got = np.ascontiguousarray(C.copy())
    pl = np.ascontiguousarray(planes)
    ctx.check(ctx.lib.b200gp_i8_update_test(ctx.handle, _cabi.ptr(pl), S, rows, K, _cabi.ptr(rs), _cabi.ptr(got)))
    ctx.reset_options()
    want = _ref_update(C, planes, rs, S)
    # integer dot products are exact; the only rounding is one fp64 fma per group
    np.testing.assert_allclose(got, want, rtol=0, atol=1e-13 * max(1.0, np.abs(want).max()))


@pytest.mark.parametrize("lookahead,subpanel", [(1, 256), (0, 256), (0, 0), (0, 512)])
@pytest.mark.parametrize("slices", [8, 7, 6])
@pytest.mark.parametrize("n,nb", [(1024, 256), (3000, 512), (6144, 1024)])
def test_ozaki_factor_parity(ctx, n, nb, slices, lookahead, subpanel):
    """subpanel: fp64 panel width inside a block column (two-level blocking; 0 = one fp64 panel per block column)"""
    rng = np.random.default_rng(n)
    X = rng.uniform(0, 20.0 * (n / 65536.0) ** (1 / 3), (n, 3))
    y = np.sin(X[:, 0]) + 0.1 * rng.normal(size=n)
    k = 1.3 * kernels.ExpSquared(0.8)
    diag = rng.uniform(0.05, 0.2, n)
    ctx.set_option("nb", nb)
    ctx.set_option("ozaki_slices", slices)
    ctx.set_option("ozaki_min_n", 0)
    ctx.set_option("ozaki_lookahead", lookahead)
    ctx.set_option("ozaki_subpanel", subpanel)
    try:
        s = solvers.DirectSolver(k, X, noise.Diagonal(diag))
        lp = GaussianProcess(k, X, diag=diag).log_probability(y)
    finally:
        ctx.set_option("ozaki_lookahead", 0)
        ctx.reset_options()
        ctx.set_option("ozaki_min_n", 8192)
        ctx.set_option("nb", 1024)
    so = o.DirectSolver(to_oracle(k), X, o.Diagonal(diag))
    lpo = o.GaussianProcess(to_oracle(k), X, diag=diag).log_probability(y)
    assert s.info == 0
    tol = {8: 1e-10, 7: 1e-10, 6: 1e-9}[slices]
    np.testing.assert_allclose(s.scale_tril, so.scale_tril, rtol=tol, atol=tol)
    assert rel(s.normalization(), so.normalization()) < (1e-9 if slices == 6 else 1e-10)
    assert rel(lp, lpo) < LOGP_RTOL, (lp, lpo)


@pytest.mark.parametrize("layout,pairing", [(1, 0)])
def test_ozaki_layout_and_pairing_variants(ctx, layout, pairing):
    """the whole factorisation with the optional digit-plane layout / group pairing switched on"""
    n = 3000
    rng = np.random.default_rng(7)
    X = rng.uniform(0, 20.0 * (n / 65536.0) ** (1 / 3), (n, 3))
    y = np.sin(X[:, 0]) + 0.1 * rng.normal(size=n)
    k = 1.3 * kernels.ExpSquared(0.8)
    ctx.set_option("nb", 512)
    ctx.set_option("ozaki_min_n", 0)
    ctx.set_option("ozaki_cluster", 21)
    ctx.set_option("ozaki_layout", layout)
    ctx.set_option("ozaki_pairing", pairing)
    try:
        lp = GaussianProcess(k, X, diag=0.1).log_probability(y)
    finally:
        ctx.reset_options()
    lpo = o.GaussianProcess(to_oracle(k), X, diag=0.1).log_probability(y)
    assert rel(lp, lpo) < LOGP_RTOL, (lp, lpo)


def test_ozaki_non_pd_and_large_scales(ctx):
    """Row scales span orders of magnitude (heteroscedastic diag); an indefinite matrix still yields -inf."""
    rng = np.random.default_rng(2)
    n = 2048
    X = rng.uniform(0, 6, (n, 2))
    y = rng.normal(size=n)
    diag = 10.0 ** rng.uniform(-2, 3, n)
    k = 50.0 * kernels.ExpSquared(1.1)
    ctx.set_option("nb", 256)
    ctx.set_option("ozaki_slices", 8)
    ctx.set_option("ozaki_min_n", 0)
    try:
        lp = GaussianProcess(k, X, diag=diag).log_probability(y)
        bad = GaussianProcess(kernels.Matern32(2.0), rng.uniform(0, 8, (n, 3)), diag=0.1)   # L1 in 3-D: indefinite
        lpbad = bad.log_probability(y)
    finally:
        ctx.reset_options()
        ctx.set_option("ozaki_min_n", 8192)
        ctx.set_option("nb", 1024)
    lpo = o.GaussianProcess(to_oracle(k), X, diag=diag).log_probability(y)
    assert rel(lp, lpo) < LOGP_RTOL
    assert bad.solver.info > 0 and lpbad == -np.inf


def test_sharded_step_api_single_rank():
    """The multi-GPU step API (update_rows / pack / unpack / panel / finish) with world_size 1."""
    from tinygp_b200 import multigpu
    rng = np.random.default_rng(77)
    n = 3000
    X = rng.uniform(0, 7, (n, 3))
    y = np.sin(X[:, 0]) + 0.1 * rng.normal(size=n)
    k = 1.3 * kernels.ExpSquared(0.8)
    ctx = _cabi.get_context()
    ctx.set_option("nb", 512)
    try:
        lpo = o.GaussianProcess(to_oracle(k), X, diag=0.1).log_probability(y)
        for slices in (8, 7):
            for streaming in (True, False):
                lp = multigpu.log_probability_sharded(k, X, np.full(n, 0.1), y, slices=slices, streaming=streaming)
                assert rel(lp, lpo) < LOGP_RTOL, (lp, lpo, slices, streaming)
    finally:
        ctx.set_option("nb", 1024)
