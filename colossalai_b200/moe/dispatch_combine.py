"""Expert-parallel dispatch -> grouped experts -> combine.

Parity: reference EP blocks (`shardformer/modeling/mixtral.py:123-208`): sort tokens by expert, exchange sizes,
uneven all-to-all, local experts, all-to-all back, un-sort, weighted sum.  Baseline (`nccl`) backend below keeps
that algorithm (dropless) but exchanges sizes as ONE device tensor and grouped-GEMMs the local experts.  The
`fused` backend (parallel/fused.py, kernel/csrc/moe.cu) removes the host sync by writing rows straight into
per-expert symmetric receive buffers over NVLink.
"""
from __future__ import annotations

from typing import Optional

import torch
import torch.distributed as dist

from ..parallel import comm
from ._operation import AllToAllUneven

__all__ = ["moe_forward", "set_moe_backend", "get_moe_backend"]

import os

_BACKEND = os.environ.get("CB200_MOE_BACKEND", "auto")     # auto | nccl | fused


def set_moe_backend(name: str) -> None:
    global _BACKEND
    assert name in ("auto", "nccl", "fused")
    _BACKEND = name


def get_moe_backend() -> str:
    return _BACKEND


def _use_fused(x: torch.Tensor, num_experts: int, ep_group) -> bool:
    if _BACKEND == "nccl" or not x.is_cuda or x.dtype not in (torch.bfloat16, torch.float16) or x.shape[1] % 8:
        return False
    from . import fused_ep

    ok = fused_ep.available(ep_group)
    if _BACKEND == "fused" and not ok:
        raise RuntimeError("CB200_MOE_BACKEND=fused but the fused expert-parallel kernels are unavailable")
    # single-rank groups gain nothing from the symmetric-buffer path unless explicitly requested
    return ok and ((ep_group is not None and comm.group_size(ep_group) > 1) or _BACKEND == "fused")


def _aligned_rows(x: torch.Tensor) -> bool:
    """Lay the expert-grouped rows out with every expert's range padded to 128 rows (zero rows): the native grouped
    weight-gradient GEMM then needs no re-layout pass (moe/grouped_gemm.py)."""
    return (x.is_cuda and x.dtype in (torch.bfloat16, torch.float16)
            and os.environ.get("CB200_GROUPED_GEMM", "native") == "native"
            and torch.cuda.get_device_capability(x.device)[0] == 9)


def _padded_counts(counts: torch.Tensor) -> torch.Tensor:
    from .grouped_gemm import ALIGN

    pc = (counts + ALIGN - 1) // ALIGN * ALIGN
    pc.cb200_aligned = True
    return pc


def moe_forward(x: torch.Tensor, topk_w: torch.Tensor, topk_idx: torch.Tensor, experts, num_experts: int,
                ep_group: Optional[dist.ProcessGroup]) -> torch.Tensor:
    """x [T, H]; topk_w [T, k] fp32; topk_idx [T, k] -> [T, H]."""
    if _use_fused(x, num_experts, ep_group):
        from . import fused_ep

        return fused_ep.moe_forward_fused(x, topk_w, topk_idx, experts, num_experts, ep_group)
    T, H = x.shape
    k = topk_idx.shape[1]
    ep = comm.group_size(ep_group) if ep_group is not None else 1     # None = no expert parallelism (NOT the world)
    n_local = num_experts // ep
    flat_idx = topk_idx.reshape(-1)                                    # [T*k]
    order = torch.argsort(flat_idx, stable=True)                       # rows grouped by global expert id
    token_of = order // k
    counts = torch.bincount(flat_idx, minlength=num_experts)           # rows per global expert
    if ep > 1:
        xs = x.index_select(0, token_of)                               # [T*k, H]  (autograd: index_add in bwd)
        # exchange per-expert counts: recv_counts[src, e_local]
        recv_counts = torch.empty_like(counts)
        dist.all_to_all_single(recv_counts, counts, group=ep_group)
        send_splits = counts.view(ep, n_local).sum(1).tolist()         # host sync (baseline backend)
        recv_counts_2d = recv_counts.view(ep, n_local)
        recv_splits = recv_counts_2d.sum(1).tolist()
        recv = AllToAllUneven.apply(xs, send_splits, recv_splits, ep_group)
        # received rows are grouped by (src rank, local expert): regroup by local expert
        rc = recv_counts_2d
        n_rows = int(sum(recv_splits))
        seg_expert = torch.arange(n_local, device=x.device).repeat(ep)             # expert id of each segment
        seg_len = rc.reshape(-1)
        row_expert = torch.repeat_interleave(seg_expert, seg_len, output_size=n_rows)
        perm = torch.argsort(row_expert, stable=True)
        local_counts = rc.sum(0)
        if _aligned_rows(x):
            from .grouped_gemm import _pad_groups

            slot_sorted, _, bound = _pad_groups(local_counts, n_rows, x.device)   # slot of the i-th row in expert order
            slot = torch.empty_like(perm)
            slot[perm] = slot_sorted                                              # slot of every received row
            grouped = recv.new_zeros(bound, H).index_copy(0, slot, recv)
            y = experts(grouped, _padded_counts(local_counts)).index_select(0, slot)
        else:
            grouped = recv.index_select(0, perm)
            y = experts(grouped, local_counts)
            inv = torch.empty_like(perm)
            inv[perm] = torch.arange(n_rows, device=x.device)
            y = y.index_select(0, inv)
        ys = AllToAllUneven.apply(y, recv_splits, send_splits, ep_group)
    elif _aligned_rows(x):
        # no expert parallelism: gather the token rows straight into the padded layout (padding slots read a zero row
        # appended to x and are combined with weight 0 into a scratch row) - no host sync, same number of passes
        from .grouped_gemm import _pad_groups

        slot, _, bound = _pad_groups(counts, T * k, x.device)
        src = torch.full((bound,), T, dtype=torch.int64, device=x.device).index_copy_(0, slot, token_of)
        x_ext = torch.cat([x, x.new_zeros(1, H)])
        ys = experts(x_ext.index_select(0, src), _padded_counts(counts))
        w_pad = torch.zeros(bound, dtype=ys.dtype, device=x.device).index_copy(
            0, slot, topk_w.reshape(-1).index_select(0, order).to(ys.dtype))
        out = torch.zeros(T + 1, H, dtype=ys.dtype, device=x.device).index_add(0, src, ys * w_pad.unsqueeze(-1))
        return out[:T]
    else:
        ys = experts(x.index_select(0, token_of), counts)
    # weighted combine back to token order
    wsorted = topk_w.reshape(-1).index_select(0, order).to(ys.dtype).unsqueeze(-1)
    out = torch.zeros(T, H, dtype=ys.dtype, device=x.device)
    out = out.index_add(0, token_of, ys * wsorted)
    return out
