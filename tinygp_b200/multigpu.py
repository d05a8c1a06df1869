"""One dense ``log_probability`` sharded over several GPUs (one process per GPU, ``torch.distributed``).

The int8 tensor-core trailing update of block column J is split by ROWS over the ranks; one
``all_gather_into_tensor`` per block column (NCCL over NVLink, rows x nb x 8 bytes) gives every rank the whole
updated column, and every rank then factors the panel and cuts its digits redundantly (cheap, deterministic),
so there is no panel broadcast.  See ``include/b200gp.h`` (b200gp_mg_*).
"""

from __future__ import annotations

from ctypes import byref, c_double, c_int, c_int64, c_void_p

from tinygp_b200 import _cabi

ALIGN = 256  # row chunks are whole 256-row tile pairs


def row_chunk(np_: int, c0: int, world: int) -> int:
    """Rows per rank for the column block starting at c0 (equal chunks, ALIGN-aligned, last ones may be short)."""
    rows = np_ - c0
    return max(ALIGN, -(-rows // (ALIGN * world)) * ALIGN)


def my_rows(np_: int, c0: int, world: int, rank: int) -> tuple[int, int]:
    ch = row_chunk(np_, c0, world)
    r0 = min(np_, c0 + rank * ch)
    return r0, min(np_, r0 + ch)


def inplace_slices(np_: int, nb: int, c0: int, world: int, rank: int) -> tuple[int, int, int, int]:
    """Element ranges (out_lo, out_hi, in_lo, in_hi) of the contiguous rolling block column (row r at r * nb) for the
    in-place all-gather of block column c0: the output covers `world` equal chunks starting at row c0 and the input is this
    rank's chunk INSIDE it (NCCL's in-place condition: in_lo == out_lo + rank * chunk).  The last chunks may reach past
    np (the buffer has world * ALIGN spare rows)."""
    ch = row_chunk(np_, c0, world)
    out_lo = c0 * nb
    in_lo = (c0 + rank * ch) * nb
    return out_lo, (c0 + world * ch) * nb, in_lo, in_lo + ch * nb


def make_context(local_rank: int = 0) -> _cabi.Context:
    """A library context on torch's current CUDA stream (so NCCL collectives order with our kernels).
    The legacy default stream has handle 0, which the C-ABI reads as "make a private stream", so a dedicated
    torch stream is created and made current for this process."""
    import torch

    torch.cuda.set_device(local_rank)
    stream = torch.cuda.Stream(device=local_rank)
    torch.cuda.set_stream(stream)
    ctx = _cabi.Context(device=local_rank, stream=stream.cuda_stream)
    ctx.torch_stream = stream          # keep it alive
    ctx.on_torch_stream = True
    _cabi.set_context(ctx)
    return ctx


def log_probability_sharded(kernel, X, diag, resid, *, slices: int = 8, streaming: bool | None = None,
                            ctx: _cabi.Context | None = None, X_dev=None, diag_dev=None, resid_dev=None,
                            stats: dict | None = None, split_panel: bool = True) -> float:
    """log N(resid | 0, k(X,X) + diag) with the factorisation sharded over the default process group.
    `*_dev` may be given as CUDA tensors (device-resident inputs, bench `value` leg).  `streaming=True` keeps no
    np x np fp64 matrix (forward solve and log-det are folded into the panel steps)."""
    import torch
    import torch.distributed as dist

    world = dist.get_world_size() if (dist.is_available() and dist.is_initialized()) else 1
    rank = dist.get_rank() if world > 1 else 0
    ctx = ctx or _cabi.get_context()
    if world > 1 and not getattr(ctx, "on_torch_stream", False):
        raise _cabi.B200Error("sharded runs need a context created by multigpu.make_context()")
    lib = ctx.lib
    if X_dev is None:
        prog, x = kernel.lower_for(X)
        n, ndim = x.shape
        d, r = _cabi.f64(diag), _cabi.f64(resid)      # converted copies must outlive b200gp_mg_create
        xp, dp, rp = _cabi.ptr(x), _cabi.ptr(d), _cabi.ptr(r)
        keep = (x, d, r)
    else:
        prog = kernel.program()   # device-resident coordinates: no host-side transforms
        n, ndim = X_dev.shape
        xp, dp, rp = X_dev.data_ptr(), diag_dev.data_ptr(), resid_dev.data_ptr()
        keep = ()
    if streaming is None:   # stream only when matrix + digit planes would not fit comfortably in HBM
        npad = -(-n // 128) * 128
        streaming = npad * npad * (8.0 + slices) > 150e9
    mg = c_void_p()
    ctx.check(lib.b200gp_mg_create(ctx.handle, _cabi.ptr(prog), prog.shape[0], xp, n, ndim, dp, rp, int(slices),
                                   int(bool(streaming)), byref(mg)))
    try:
        np_, nb, ncol = c_int64(), c_int64(), c_int()
        ctx.check(lib.b200gp_mg_geometry(mg, byref(np_), byref(nb), byref(ncol)))
        np_, nb, ncol = np_.value, nb.value, ncol.value
        inplace = bool(streaming) and world > 1
        if inplace:
            # the rolling block column lives in a torch tensor: rank chunks are contiguous row ranges of it, so the
            # collective runs IN PLACE (input = this rank's slice of the output) -- no pack / unpack copies
            col_rows = np_ + world * ALIGN
            colbuf = torch.empty(col_rows * nb, dtype=torch.float64, device="cuda")
            ctx.check(lib.b200gp_mg_use_colbuf(mg, colbuf.data_ptr(), col_rows))
        elif world > 1:
            chmax = row_chunk(np_, 0, world)
            mine_buf = torch.empty(chmax * nb, dtype=torch.float64, device="cuda")
            full_buf = torch.empty(world * chmax * nb, dtype=torch.float64, device="cuda")
        for J in range(ncol):
            c0 = J * nb
            ch = row_chunk(np_, c0, world)
            r0, r1 = my_rows(np_, c0, world, rank)
            ctx.check(lib.b200gp_mg_update_rows(mg, J, r0, r1))
            if inplace:
                o0, o1, i0, i1 = inplace_slices(np_, nb, c0, world, rank)
                out = colbuf[o0:o1]
                kbj = min(nb, np_ - c0)
                if split_panel and ch >= kbj:
                    # sharded triangular solve: the diagonal block's rows (all inside rank 0's chunk) go to everyone, each
                    # rank factors the block and solves ITS rows, and the finished column is all-gathered in place
                    dist.broadcast(colbuf[c0 * nb:(c0 + kbj) * nb], src=0)
                    ctx.check(lib.b200gp_mg_panel_factor(mg, J, r0, r1))
                    dist.all_gather_into_tensor(out, colbuf[i0:i1])
                    ctx.check(lib.b200gp_mg_panel_finish(mg, J))
                    if stats is not None:
                        stats["bytes"] = stats.get("bytes", 0) + int(out.numel() * 8) + int(kbj * nb * 8)
                        stats["exchange"] = ("NCCL broadcast of the diagonal block + in-place all_gather_into_tensor of the "
                                             "factored block column (row-sharded update AND triangular solve)")
                    continue
                dist.all_gather_into_tensor(out, colbuf[i0:i1])
                if stats is not None:
                    stats["bytes"] = stats.get("bytes", 0) + int(out.numel() * 8)
                    stats.setdefault("exchange", "in-place dist.all_gather_into_tensor (NCCL) on the contiguous block column, one per block column")
            elif world > 1:
                mine = mine_buf[: ch * nb]
                full = full_buf[: world * ch * nb]
                ctx.check(lib.b200gp_mg_pack(mg, J, r0, r1, mine.data_ptr()))
                dist.all_gather_into_tensor(full, mine)
                if stats is not None:
                    stats["bytes"] = stats.get("bytes", 0) + int(full.numel() * 8)
                    stats["exchange"] = "pack -> dist.all_gather_into_tensor (NCCL) -> unpack, one per block column"
                for r in range(world):
                    if r == rank:
                        continue
                    q0 = min(np_, c0 + r * ch)
                    q1 = min(np_, q0 + ch)
                    if q1 > q0:
                        ctx.check(lib.b200gp_mg_unpack(mg, J, q0, q1, full.data_ptr() + r * ch * nb * 8))
            ctx.check(lib.b200gp_mg_panel(mg, J))
        lp = c_double()
        ctx.check(lib.b200gp_mg_finish(mg, byref(lp)))
        del keep
        return lp.value
    finally:
        lib.b200gp_mg_free(mg)
