"""The N > 1 host logic (problem sharding, max-over-ranks timing, result gather) on CPU with gloo, world_size 2.
The data path itself has no collective (replicas)."""

import os

import pytest
import socket

import numpy as np
import torch.distributed as dist
import torch.multiprocessing as mp

from tinygp_b200 import parallel


def _free_port():
    with socket.socket() as s:
        s.bind(("127.0.0.1", 0))
        return s.getsockname()[1]


def _worker(rank, world, port, nprob, q):
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    try:
        idx = parallel.shard_indices(nprob, rank, world)
        # stand-in for the per-problem log-probabilities computed by this rank's GPU
        vals = np.sin(idx.astype(np.float64)) - 3.0 * idx
        full = parallel.gather_results(idx, vals, nprob)
        tmax = parallel.max_over_ranks(10.0 + rank)
        q.put((rank, idx.tolist(), full.tolist(), tmax))
    finally:
        dist.destroy_process_group()


def test_sharding_is_a_partition():
    for nprob, world in [(1024, 8), (7, 2), (3, 4), (1, 1)]:
        seen = np.concatenate([parallel.shard_indices(nprob, r, world) for r in range(world)])
        assert sorted(seen.tolist()) == list(range(nprob))


def test_world_size_2_gloo():
    world, nprob = 2, 11
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = _free_port()
    procs = [ctx.Process(target=_worker, args=(r, world, port, nprob, q)) for r in range(world)]
    for p in procs:
        p.start()
    res = [q.get(timeout=120) for _ in range(world)]
    for p in procs:
        p.join(timeout=60)
        assert p.exitcode == 0
    want = np.sin(np.arange(nprob, dtype=np.float64)) - 3.0 * np.arange(nprob)
    for rank, idx, full, tmax in res:
        assert idx == list(range(rank, nprob, world))
        np.testing.assert_allclose(full, want, rtol=0, atol=0)
        assert tmax == 11.0          # max over ranks of (10 + rank)


def test_row_chunks_partition_every_block_column():
    from tinygp_b200 import multigpu
    for np_, nb, world in [(65536, 1024, 8), (131072, 1024, 8), (3072, 256, 2), (1280, 256, 4), (256, 256, 2)]:
        for c0 in range(0, np_, nb):
            ch = multigpu.row_chunk(np_, c0, world)
            assert ch % multigpu.ALIGN == 0
            cover = []
            for r in range(world):
                r0, r1 = multigpu.my_rows(np_, c0, world, r)
                assert c0 <= r0 <= r1 <= np_ and r0 % 128 == 0 and (r1 - r0) <= ch
                cover.append((r0, r1))
            # contiguous, disjoint, complete
            assert cover[0][0] == c0
            for (a0, a1), (b0, b1) in zip(cover, cover[1:]):
                assert a1 == b0 or (a1 == np_ and b0 == np_)
            assert max(r1 for _, r1 in cover) == np_


def _inplace_worker(rank, world, port, np_, nb, q):
    import torch
    from tinygp_b200 import multigpu
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    try:
        col = torch.full(((np_ + world * multigpu.ALIGN) * nb,), -1.0, dtype=torch.float64)
        ok = True
        for c0 in range(0, np_, nb):
            r0, r1 = multigpu.my_rows(np_, c0, world, rank)
            rows = torch.arange(r0, r1, dtype=torch.float64)
            col[r0 * nb:r1 * nb] = (rows[:, None] * 1000.0 + c0 + torch.arange(nb, dtype=torch.float64)[None, :]).reshape(-1)
            o0, o1, i0, i1 = multigpu.inplace_slices(np_, nb, c0, world, rank)
            ch = multigpu.row_chunk(np_, c0, world)
            assert i0 == o0 + rank * ch * nb and i1 - i0 == ch * nb and o1 - o0 == world * ch * nb
            out = col[o0:o1]
            dist.all_gather_into_tensor(out, col[i0:i1].clone())    # gloo has no in-place path: same geometry, copied input
            allrows = torch.arange(c0, np_, dtype=torch.float64)
            want = (allrows[:, None] * 1000.0 + c0 + torch.arange(nb, dtype=torch.float64)[None, :]).reshape(-1)
            ok = ok and bool(torch.equal(col[c0 * nb:np_ * nb], want))
        q.put((rank, ok))
    finally:
        dist.destroy_process_group()


def test_inplace_slices_stay_inside_the_column_buffer():
    """the in-place all-gather's output covers `world` equal chunks from row c0 on and may reach past np: never past the
    world * ALIGN spare rows the column buffer has, for every block column of the bench sizes on 2 / 4 / 8 ranks"""
    from tinygp_b200 import multigpu
    for np_, nb in [(131072, 1024), (65536, 1024), (65664, 1024), (5120, 512), (1280, 256)]:
        for world in (2, 4, 8):
            limit = (np_ + world * multigpu.ALIGN) * nb
            for c0 in range(0, np_, nb):
                ch = multigpu.row_chunk(np_, c0, world)
                prev_hi = None
                for rank in range(world):
                    o0, o1, i0, i1 = multigpu.inplace_slices(np_, nb, c0, world, rank)
                    assert o0 == c0 * nb and o1 - o0 == world * ch * nb and o1 <= limit
                    assert i0 == o0 + rank * ch * nb and i1 - i0 == ch * nb and o0 <= i0 < i1 <= o1
                    assert prev_hi is None or i0 == prev_hi
                    prev_hi = i1
                    r0, r1 = multigpu.my_rows(np_, c0, world, rank)
                    assert r0 * nb >= i0 or r0 == np_                 # a rank's rows start inside its own chunk ...
                    assert r1 * nb <= i1 or r1 == np_                 # ... and end inside it


@pytest.mark.parametrize("world", [2, 4])
def test_inplace_block_column_allgather_geometry(world):
    """the sharded path's exchange (multigpu.inplace_slices): every rank ends up with every row of the block column"""
    np_, nb = 1280, 256
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = _free_port()
    procs = [ctx.Process(target=_inplace_worker, args=(r, world, port, np_, nb, q)) for r in range(world)]
    for p in procs:
        p.start()
    res = [q.get(timeout=120) for _ in range(world)]
    for p in procs:
        p.join(timeout=60)
        assert p.exitcode == 0
    assert all(ok for _, ok in res)
