"""One factorisation sharded over TWO GPUs (NCCL, one process per GPU): BASELINE config 3's path at a size the oracle
can check; skipped when fewer than two CUDA devices are visible.  The split panel step of the sharded path
(b200gp_mg_panel_factor / b200gp_mg_panel_finish) is also driven with one rank, which needs one GPU only."""

import os
import socket

import numpy as np
import pytest

pytestmark = pytest.mark.gpu


def _free_port():
    with socket.socket() as s:
        s.bind(("127.0.0.1", 0))
        return s.getsockname()[1]


def _worker(rank, world, port, n, nb, streaming, split, q, mg_splitk=0):
    import torch
    import torch.distributed as dist
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    os.environ["LOCAL_RANK"] = str(rank)
    torch.cuda.set_device(rank)
    from tinygp_b200 import kernels, multigpu
    ctx = multigpu.make_context(rank)
    dist.init_process_group("nccl", rank=rank, world_size=world, device_id=torch.device("cuda", rank))
    try:
        ctx.set_option("nb", nb)
        ctx.set_option("mg_splitk", mg_splitk)
        rng = np.random.default_rng(49383)
        side = 25.0 * (n / 131072.0) ** (1.0 / 3.0)
        X = np.ascontiguousarray(rng.uniform(0.0, side, (n, 3)))
        y = np.sin(X[:, 0]) + 0.1 * rng.normal(size=n)
        diag = np.full(n, 0.1)
        L2 = kernels.L2Distance()
        k = 1.5 * kernels.Matern52(2.0, L2) + 0.7 * kernels.RationalQuadratic(1.5, L2, alpha=1.5)
        stats = {}
        lp = multigpu.log_probability_sharded(k, X, diag, y, slices=7, streaming=streaming, ctx=ctx, stats=stats,
                                                split_panel=split)
        q.put((rank, lp, stats.get("exchange", "")))
    finally:
        dist.destroy_process_group()


@pytest.mark.parametrize("streaming,split,mg_splitk", [(True, True, 1), (True, True, 0), (True, False, 0), (False, False, 0)])
def test_sharded_two_ranks_matches_oracle_and_single_rank(streaming, split, mg_splitk):
    import torch
    if torch.cuda.device_count() < 2:
        pytest.skip("needs two GPUs")
    import torch.multiprocessing as mp
    from oracle import tinygp_np as o
    from tinygp_b200 import kernels, multigpu
    n, nb, world = 5000, 512, 2
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = _free_port()
    procs = [ctx.Process(target=_worker, args=(r, world, port, n, nb, streaming, split, q, mg_splitk)) for r in range(world)]
    for p in procs:
        p.start()
    res = sorted(q.get(timeout=600) for _ in range(world))
    for p in procs:
        p.join(timeout=120)
        assert p.exitcode == 0
    rng = np.random.default_rng(49383)
    side = 25.0 * (n / 131072.0) ** (1.0 / 3.0)
    X = np.ascontiguousarray(rng.uniform(0.0, side, (n, 3)))
    y = np.sin(X[:, 0]) + 0.1 * rng.normal(size=n)
    ko = o.Constant(1.5) * o.Matern52(2.0, o.L2Distance()) + o.Constant(0.7) * o.RationalQuadratic(1.5, o.L2Distance(), alpha=1.5)
    lpo = o.GaussianProcess(ko, X, diag=0.1).log_probability(y)
    assert res[0][1] == res[1][1]                                  # every rank holds the same value
    assert abs(res[0][1] - lpo) <= 1e-8 * abs(lpo), (res, lpo)
    if streaming:
        assert "in-place" in res[0][2]
        assert ("broadcast" in res[0][2]) == split
    # the same library, one rank: bit-identical when every tile keeps one K range (integer products are exact and the panel
    # work is replicated); with the tail split-K on (option mg_splitk) the last bits depend on how many tiles a rank has
    from tinygp_b200 import _cabi
    c = _cabi.get_context()
    c.set_option("nb", nb)
    c.set_option("mg_splitk", mg_splitk)
    L2 = kernels.L2Distance()
    k = 1.5 * kernels.Matern52(2.0, L2) + 0.7 * kernels.RationalQuadratic(1.5, L2, alpha=1.5)
    lp1 = multigpu.log_probability_sharded(k, X, np.full(n, 0.1), y, slices=7, streaming=streaming)
    if mg_splitk == 0:
        assert lp1 == res[0][1], (lp1, res)
    else:
        assert abs(lp1 - res[0][1]) <= 1e-12 * abs(lp1), (lp1, res)


@pytest.mark.parametrize("n,last", [(1100, 128), (1536, 512)])
def test_split_panel_step_on_one_rank(ctx, n, last):
    """b200gp_mg_panel_factor (diagonal block + this rank's rows below it) then b200gp_mg_panel_finish, with world = 1:
    bit-identical to the one-call panel step b200gp_mg_panel, and parity with the oracle.  nb = 512: n = 1100 ends with a
    128-column panel, n = 1536 has three full ones."""
    from ctypes import byref, c_double, c_int, c_int64, c_void_p
    from oracle import tinygp_np as o
    from tinygp_b200 import _cabi, kernels, multigpu
    from util import LOGP_RTOL, rel, to_oracle
    rng = np.random.default_rng(n)
    X = np.ascontiguousarray(rng.uniform(0, 20.0 * (n / 65536.0) ** (1 / 3), (n, 3)))
    y = np.sin(X[:, 0]) + 0.1 * rng.normal(size=n)
    diag = np.full(n, 0.1)
    k = 1.3 * kernels.ExpSquared(0.8)
    ctx.set_option("nb", 512)
    prog, x = k.lower_for(X)
    d, r = _cabi.f64(diag), _cabi.f64(y)
    lib = ctx.lib
    mg = c_void_p()
    ctx.check(lib.b200gp_mg_create(ctx.handle, _cabi.ptr(prog), prog.shape[0], _cabi.ptr(x), n, x.shape[1], _cabi.ptr(d),
                                   _cabi.ptr(r), 7, 0, byref(mg)))
    try:
        np_, nb, ncol = c_int64(), c_int64(), c_int()
        ctx.check(lib.b200gp_mg_geometry(mg, byref(np_), byref(nb), byref(ncol)))
        np_, nb, ncol = np_.value, nb.value, ncol.value
        assert nb == 512 and ncol == 3 and np_ - 2 * nb == last
        for J in range(ncol):
            r0, r1 = multigpu.my_rows(np_, J * nb, 1, 0)
            ctx.check(lib.b200gp_mg_update_rows(mg, J, r0, r1))
            ctx.check(lib.b200gp_mg_panel_factor(mg, J, r0, r1))
            ctx.check(lib.b200gp_mg_panel_finish(mg, J))
        lp = c_double()
        ctx.check(lib.b200gp_mg_finish(mg, byref(lp)))
    finally:
        lib.b200gp_mg_free(mg)
    want = multigpu.log_probability_sharded(k, X, diag, y, slices=7, streaming=False, ctx=ctx)
    assert lp.value == want, (lp.value, want)
    lpo = o.GaussianProcess(to_oracle(k), X, diag=0.1).log_probability(y)
    assert rel(lp.value, lpo) < LOGP_RTOL, (lp.value, lpo)
