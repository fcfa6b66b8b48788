"""Functional collectives on contiguous tensors (the NCCL/gloo baseline backend and correctness oracle).

Every comm-bound op in the framework has two interchangeable backends behind one autograd Function:
this module (`torch.distributed`: NCCL on the GPU, gloo on the CPU plumbing tier, also the multi-node path) and
`colossalai_b200.parallel.fused` (sm_90a kernels over NVLink peer memory).  Parity: the raw collective call
sites inventoried in SURVEY §2.12 (`shardformer/layer/_operation.py:1187-1282`).
"""
from __future__ import annotations

from typing import List, Optional, Sequence

import threading
from contextlib import contextmanager

import torch
import torch.distributed as dist
from torch.distributed import ProcessGroup

__all__ = [
    "group_size", "group_rank", "group_key", "all_reduce", "all_gather", "reduce_scatter", "all_to_all_single",
    "all_to_all_uneven", "broadcast", "split_along", "send_recv_ring",
]


def group_size(group: Optional[ProcessGroup]) -> int:
    if not dist.is_initialized():
        return 1
    return dist.get_world_size(group)


def group_rank(group: Optional[ProcessGroup]) -> int:
    if not dist.is_initialized():
        return 0
    return dist.get_rank(group)


def group_key(group: Optional[ProcessGroup]):
    """Identity of a process group for caches that outlive a call (workspaces, symmetric buffers).  `id(group)` can be
    reused by a NEW group once the old one is destroyed and collected - a cache keyed by it would then hand the new
    group a workspace mapped for other ranks; torch's `group_name` is a process-wide unique string that is never reused.
    `None` is the default (world) group."""
    if group is None and dist.is_initialized():
        group = dist.group.WORLD
    name = getattr(group, "group_name", None)
    return ("pg", name) if name else ("id", id(group))


# ---- fp8 communication switch (reference: the `fp8_communication` flag threaded through every parallel layer).
# Layers enter `fp8_communication(True)` around their forward; the autograd functions remember the flag for backward.
_FP8_STATE = threading.local()


def fp8_enabled() -> bool:
    return getattr(_FP8_STATE, "on", False)


@contextmanager
def fp8_communication(enabled: bool = True):
    prev = fp8_enabled()
    _FP8_STATE.on = bool(enabled)
    try:
        yield
    finally:
        _FP8_STATE.on = prev


def _fp8_ok(x: torch.Tensor) -> bool:
    return fp8_enabled() and x.is_floating_point() and x.dtype in (torch.float16, torch.bfloat16, torch.float32)


def all_reduce(x: torch.Tensor, group: Optional[ProcessGroup] = None, op=dist.ReduceOp.SUM,
               async_op: bool = False):
    if group_size(group) == 1:
        return None if async_op else x
    if _fp8_ok(x) and op == dist.ReduceOp.SUM and not async_op:
        from ..quantization.fp8 import all_reduce_fp8

        all_reduce_fp8(x, "e4m3", group=group)
        return x
    work = dist.all_reduce(x, op=op, group=group, async_op=async_op)
    return work if async_op else x


def all_gather(x: torch.Tensor, dim: int = 0, group: Optional[ProcessGroup] = None) -> torch.Tensor:
    """Concatenate every rank's `x` along `dim`."""
    ws = group_size(group)
    if ws == 1:
        return x
    dim = dim % x.dim()
    x = x.contiguous()
    out = torch.empty((ws,) + tuple(x.shape), dtype=x.dtype, device=x.device)
    if _fp8_ok(x):
        from ..quantization.fp8 import all_gather_fp8

        all_gather_fp8(list(out.unbind(0)), x, group=group, fp8_format="e4m3")
    else:
        dist.all_gather_into_tensor(out.view(-1), x.view(-1), group=group)
    if dim == 0:
        return out.view((ws * x.shape[0],) + tuple(x.shape[1:]))
    # [ws, d0, ..., ddim, ...] -> [d0, ..., ws*ddim, ...]
    out = out.movedim(0, dim)  # [..., ws, ddim, ...]
    shape = list(x.shape)
    shape[dim] *= ws
    return out.reshape(shape)


def reduce_scatter(x: torch.Tensor, dim: int = 0, group: Optional[ProcessGroup] = None) -> torch.Tensor:
    """Sum over ranks, then keep this rank's 1/ws slice along `dim`."""
    ws = group_size(group)
    if ws == 1:
        return x
    dim = dim % x.dim()
    assert x.shape[dim] % ws == 0, f"reduce_scatter: dim {dim} of {tuple(x.shape)} not divisible by {ws}"
    if dim != 0:
        shape = list(x.shape)
        shape[dim] //= ws
        x = x.reshape(shape[:dim] + [ws, shape[dim]] + shape[dim + 1:]).movedim(dim, 0)
        out_shape = shape
    else:
        out_shape = [x.shape[0] // ws] + list(x.shape[1:])
    x = x.contiguous()
    out = torch.empty(out_shape, dtype=x.dtype, device=x.device)
    if _fp8_ok(x):
        from ..quantization.fp8 import reduce_scatter_fp8

        reduce_scatter_fp8(out, list(x.view((ws,) + tuple(out_shape)).unbind(0)), group=group, fp8_format="e5m2")
    else:
        dist.reduce_scatter_tensor(out.view(-1), x.view(-1), group=group)
    return out


def all_to_all_single(x: torch.Tensor, scatter_dim: int, gather_dim: int,
                      group: Optional[ProcessGroup] = None) -> torch.Tensor:
    """Split `x` into ws pieces along `scatter_dim`, exchange, concatenate received pieces along `gather_dim`
    (DeepSpeed-Ulysses layout switch)."""
    ws = group_size(group)
    if ws == 1:
        return x
    scatter_dim, gather_dim = scatter_dim % x.dim(), gather_dim % x.dim()
    assert x.shape[scatter_dim] % ws == 0
    pieces = [p.contiguous() for p in x.chunk(ws, dim=scatter_dim)]
    send = torch.stack(pieces, 0)
    recv = torch.empty_like(send)
    dist.all_to_all_single(recv.view(-1), send.view(-1), group=group)
    return torch.cat(list(recv.unbind(0)), dim=gather_dim)


def all_to_all_uneven(x: torch.Tensor, in_splits: Sequence[int], out_splits: Sequence[int],
                      group: Optional[ProcessGroup] = None) -> torch.Tensor:
    """Row-wise uneven all-to-all (`x` is [rows, ...]; splits are row counts per peer)."""
    ws = group_size(group)
    if ws == 1:
        return x
    x = x.contiguous()
    out = torch.empty((int(sum(out_splits)),) + tuple(x.shape[1:]), dtype=x.dtype, device=x.device)
    dist.all_to_all_single(out, x, list(map(int, out_splits)), list(map(int, in_splits)), group=group)
    return out


def broadcast(x: torch.Tensor, src: int, group: Optional[ProcessGroup] = None) -> torch.Tensor:
    if group_size(group) > 1:
        dist.broadcast(x, src=src, group=group)
    return x


def split_along(x: torch.Tensor, dim: int, group: Optional[ProcessGroup] = None) -> torch.Tensor:
    ws = group_size(group)
    if ws == 1:
        return x
    assert x.shape[dim] % ws == 0, f"split_along: dim {dim} of {tuple(x.shape)} not divisible by {ws}"
    return x.chunk(ws, dim=dim)[group_rank(group)].contiguous()


def send_recv_ring(send: torch.Tensor, recv: torch.Tensor, group: Optional[ProcessGroup] = None,
                   reverse: bool = False) -> List:
    """One ring hop: send to next rank, receive from previous (or reversed).  Returns work handles."""
    ws, r = group_size(group), group_rank(group)
    ranks = dist.get_process_group_ranks(group) if group is not None else list(range(ws))
    nxt, prv = ranks[(r + 1) % ws], ranks[(r - 1) % ws]
    if reverse:
        nxt, prv = prv, nxt
    ops = [dist.P2POp(dist.isend, send, nxt, group), dist.P2POp(dist.irecv, recv, prv, group)]
    if r % 2 == 1:
        ops.reverse()
    return dist.batch_isend_irecv(ops)
