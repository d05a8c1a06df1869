"""The fp64 GEMM mainloop (the DMMA warp tile of tinygp_b200/csrc/dmma.cuh) on the GPU against NumPy / LAPACK: the
plain NT product behind b200gp_gram_downdate, factorisations whose trailing updates use every epilogue mode (beta 1,
and beta 2, the generated first update) and the panel GEMMs, and the batched entry point."""

import numpy as np
import pytest
import scipy.linalg

from oracle import tinygp_np as o
from tinygp_b200 import _cabi, kernels, noise, solvers
from util import LOGP_RTOL, rel, to_oracle

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("k", [128, 1024, 640])
@pytest.mark.parametrize("m", [300, 512])
def test_gram_downdate_matches_numpy(ctx, m, k):
    rng = np.random.default_rng(m + k)
    At = rng.normal(size=(m, k))
    C0 = rng.normal(size=(m, m))
    C = np.ascontiguousarray(C0.copy())
    ctx.check(ctx.lib.b200gp_gram_downdate(ctx.handle, _cabi.ptr(At), m, k, _cabi.ptr(C)))
    want = C0 - At @ At.T
    np.testing.assert_allclose(C, want, rtol=0, atol=1e-12 * np.abs(At).max() ** 2 * k)


@pytest.mark.parametrize("nb", [128, 512, 1024])
def test_factor_against_lapack(ctx, nb):
    rng = np.random.default_rng(nb)
    n = 2500           # several blocks of every nb, and a ragged last tile
    X = rng.uniform(0, 10, (n, 3))
    k = 1.3 * kernels.Matern52(1.5, kernels.L2Distance())
    diag = rng.uniform(0.05, 0.2, n)
    ctx.set_option("nb", nb)
    ctx.set_option("ozaki_slices", 0)       # the native fp64 path
    s = solvers.DirectSolver(k, X, noise.Diagonal(diag))
    assert s.info == 0
    want = scipy.linalg.cholesky(to_oracle(k)(X, X) + np.diag(diag), lower=True)
    np.testing.assert_allclose(s.scale_tril, want, rtol=1e-10, atol=1e-12)


def test_batched_grid(ctx):
    rng = np.random.default_rng(7)
    n = 1300
    X = np.ascontiguousarray(rng.uniform(0, 8, (n, 2)))
    y = np.sin(X[:, 0]) + 0.1 * rng.normal(size=n)
    diag = np.full(n, 0.1)
    ks = [a * kernels.ExpSquared(s) for s in (0.6, 1.7) for a in (0.5, 2.0)]
    progs = np.ascontiguousarray(np.stack([kk.program() for kk in ks]))
    out = np.empty(len(ks))
    ctx.set_option("nb_batched", 256)
    ctx.check(ctx.lib.b200gp_dense_log_probability_batched(
        ctx.handle, _cabi.ptr(progs), progs.shape[1], len(ks), _cabi.ptr(X), n, 2, _cabi.ptr(diag), _cabi.ptr(y),
        _cabi.ptr(out)))
    for kk, got in zip(ks, out):
        want = o.GaussianProcess(to_oracle(kk), X, diag=0.1).log_probability(y)
        assert rel(got, want) < LOGP_RTOL, (got, want)
