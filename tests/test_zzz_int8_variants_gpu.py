"""int8 update kernel variants: the paired-group kernels `i8_update_kernel<CM, CN, true, 1>` for every cluster shape, the
default 2 x 1 cluster launch (ozaki_cluster = 2) with and without pairing, and its split-K segments.  Last file of the
`-m gpu` suite on purpose: if a kernel faulted, the CUDA context of the test process would be unusable for whatever came
after it."""

import numpy as np
import pytest

from oracle import tinygp_np as o
from tinygp_b200 import GaussianProcess
from util import LOGP_RTOL, rel, to_oracle

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("layout", [0, 1])
@pytest.mark.parametrize("pairing", [1, 2])
@pytest.mark.parametrize("cluster", [11, 21, 12, 22, 41, 42])
@pytest.mark.parametrize("rows,K,S", [(256, 128, 1), (256, 512, 3), (512, 1024, 8), (768, 384, 7), (512, 2048, 2)])
def test_paired_group_kernels_are_exact(ctx, rows, K, S, cluster, pairing, layout):
    """i8_update_kernel<CM, CN, true, 1>: two digit groups per pass (pairing 1) and its single-group diagnostic (2); for an
    odd plane count the unpaired group is group 0."""
    from test_ozaki_gpu import _ref_update
    from tinygp_b200 import _cabi
    ctx.set_option("ozaki_cluster", cluster)
    ctx.set_option("ozaki_pairing", pairing)
    ctx.set_option("ozaki_layout", layout)
    rng = np.random.default_rng(rows + K + S)
    planes = rng.integers(-64, 65, size=(S, rows, K), dtype=np.int8)
    rs = 2.0 ** rng.integers(-2, 3, size=rows).astype(np.float64)
    C = rng.normal(size=(rows, rows))
    got = C.copy()
    pl = np.ascontiguousarray(planes)
    try:
        ctx.check(ctx.lib.b200gp_i8_update_test(ctx.handle, _cabi.ptr(pl), S, rows, K, _cabi.ptr(rs), _cabi.ptr(got)))
    finally:
        ctx.reset_options()
    want = _ref_update(C, planes, rs, S)
    np.testing.assert_allclose(got, want, rtol=0, atol=1e-13 * max(1.0, np.abs(want).max()))


@pytest.mark.parametrize("layout,pairing", [(1, 1), (0, 1), (0, 2)])
def test_factorisation_with_paired_groups(ctx, layout, pairing):
    from tinygp_b200 import kernels
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


@pytest.mark.parametrize("pairing", [1, 2])
@pytest.mark.parametrize("rows,K,S", [(256, 128, 1), (256, 512, 3), (512, 1024, 8), (768, 384, 7), (512, 2048, 2),
                                      (1024, 4096, 7)])
def test_paired_cta_pair_kernel_is_exact(ctx, rows, K, S, pairing):
    """the default launch shape (ozaki_cluster = 2: 2 x 1 cluster, B slices multicast) with two digit groups per pass (same
    exactness harness as tests/test_ozaki_gpu.py::test_i8_update_kernel_is_exact)"""
    from tinygp_b200 import _cabi
    ctx.set_option("ozaki_cluster", 2)
    ctx.set_option("ozaki_pairing", pairing)
    rng = np.random.default_rng(rows + K + S)
    planes = rng.integers(-64, 65, size=(S, rows, K), dtype=np.int8)
    rs = 2.0 ** rng.integers(-2, 3, size=rows).astype(np.float64)
    C = rng.normal(size=(rows, rows))
    got = C.copy()
    pl = np.ascontiguousarray(planes)
    try:
        ctx.check(ctx.lib.b200gp_i8_update_test(ctx.handle, _cabi.ptr(pl), S, rows, K, _cabi.ptr(rs), _cabi.ptr(got)))
    finally:
        ctx.reset_options()
    want = C.copy()
    P = planes.astype(np.float64)
    for s in range(S):
        for t in range(S - s):
            want -= 2.0 ** -(12 + 7 * (s + t)) * (rs[:, None] * rs[None, :]) * (P[s] @ P[t].T)
    np.testing.assert_allclose(got, want, rtol=0, atol=1e-13 * max(1.0, np.abs(want).max()))


@pytest.mark.parametrize("force", [2, 3, 5])
@pytest.mark.parametrize("rows,K,S", [(512, 1024, 7), (768, 1920, 7), (1024, 4096, 8), (256, 640, 3)])
def test_split_k_segments_are_exact(ctx, rows, K, S, force):
    """default launch shape with the K range cut into segments inside one launch (segment 0 updates C, the others their own
    zero-filled scratch tiles, added afterwards in a fixed order): same integer sums, one more fp64 addition per segment"""
    from tinygp_b200 import _cabi
    ctx.set_option("ozaki_cluster", 2)
    ctx.set_option("ozaki_pairing", 1)
    ctx.set_option("ozaki_splitk_force", force)
    rng = np.random.default_rng(rows + K + S + force)
    planes = rng.integers(-64, 65, size=(S, rows, K), dtype=np.int8)
    rs = 2.0 ** rng.integers(-2, 3, size=rows).astype(np.float64)
    C = rng.normal(size=(rows, rows))
    got = C.copy()
    pl = np.ascontiguousarray(planes)
    try:
        ctx.check(ctx.lib.b200gp_i8_update_test(ctx.handle, _cabi.ptr(pl), S, rows, K, _cabi.ptr(rs), _cabi.ptr(got)))
    finally:
        ctx.reset_options()
    want = C.copy()
    P = planes.astype(np.float64)
    for s in range(S):
        for t in range(S - s):
            want -= 2.0 ** -(12 + 7 * (s + t)) * (rs[:, None] * rs[None, :]) * (P[s] @ P[t].T)
    np.testing.assert_allclose(got, want, rtol=0, atol=1e-13 * max(1.0, np.abs(want).max()))


@pytest.mark.parametrize("force", [0, 3])
def test_factorisation_with_split_k(ctx, force):
    """whole factorisation with the split-K policy on (default) and with three forced segments in every update launch"""
    from tinygp_b200 import kernels
    n = 6144
    rng = np.random.default_rng(11)
    X = rng.uniform(0, 20.0 * (n / 65536.0) ** (1 / 3), (n, 3))
    y = np.sin(X[:, 0]) + 0.1 * rng.normal(size=n)
    k = 1.3 * kernels.ExpSquared(0.8)
    ctx.set_option("nb", 512)
    ctx.set_option("ozaki_min_n", 0)
    ctx.set_option("ozaki_splitk_force", force)
    try:
        lp = GaussianProcess(k, X, diag=0.1).log_probability(y)
    finally:
        ctx.reset_options()
    lpo = o.GaussianProcess(to_oracle(k), X, diag=0.1).log_probability(y)
    assert rel(lp, lpo) < LOGP_RTOL, (lp, lpo)


@pytest.mark.parametrize("slices", [0, 7])
def test_panel_with_eight_diagonal_tiles_matches_oracle(ctx, slices):
    """right-looking order inside the diagonal block of the panel factorisation, 8 tiles per chain at nb = 1024: parity
    with the oracle on the native fp64 path (slices 0) and on the int8 update (7 planes)"""
    from tinygp_b200 import kernels
    n = 6144
    rng = np.random.default_rng(23)
    X = rng.uniform(0, 20.0 * (n / 65536.0) ** (1 / 3), (n, 3))
    y = np.sin(X[:, 0]) + 0.1 * rng.normal(size=n)
    k = 1.3 * kernels.ExpSquared(0.8)
    ctx.set_option("nb", 1024)
    ctx.set_option("ozaki_min_n", 0 if slices else 1 << 40)
    try:
        lp = GaussianProcess(k, X, diag=0.1).log_probability(y)
    finally:
        ctx.reset_options()
    lpo = o.GaussianProcess(to_oracle(k), X, diag=0.1).log_probability(y)
    assert rel(lp, lpo) < LOGP_RTOL, (lp, lpo)
