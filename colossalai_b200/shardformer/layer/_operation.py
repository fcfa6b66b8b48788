"""Autograd collectives and comm-fused linear ops for tensor / sequence parallelism.

Parity: reference `colossalai/shardformer/layer/_operation.py:76-1393`
(`LinearWithAsyncCommunication`, `_LinearWithGatherForwardReduceScatterBackward`,
`_LinearWithReduceScatterForwardGatherBackward`, `_AllToAll`, split/gather/reduce fwd-bwd pairs, ring variants).

H100-first design: each comm-bound linear is ONE autograd Function with two interchangeable backends —
`nccl` (torch.distributed collectives + GEMM; also the gloo CPU tier and the correctness oracle) and `fused`
(`colossalai_b200.parallel.fused`: a single sm_90a kernel that overlaps the wgmma GEMM tiles with P2P /
multimem traffic over NVLink).  Weight-gradient GEMMs can be deferred (`WeightGradStore`) for zero-bubble PP.
"""
from __future__ import annotations

import os
from typing import Optional, Tuple

import torch
import torch.distributed as dist
from torch.distributed import ProcessGroup

from ... import ops
from ...parallel import comm
from ...pipeline.weight_grad_store import WeightGradStore

__all__ = [
    "linear_with_async_comm", "linear_with_grad_accum", "linear_gather_forward_reducescatter_backward",
    "linear_reducescatter_forward_gather_backward", "gather_forward_split_backward",
    "split_forward_gather_backward", "reduce_forward", "reduce_backward", "all_to_all_comm",
    "gather_forward_reducescatter_backward", "reducescatter_forward_gather_backward", "gather_sp_output",
    "split_batch_zigzag", "is_share_sp_tp", "set_comm_backend", "get_comm_backend",
]

_COMM_BACKEND = "nccl"


_SAVE_GATHERED = os.environ.get("CB200_SP_SAVE_GATHERED", "1") != "0"


def set_comm_backend(name: str) -> None:
    """'nccl' (torch.distributed) or 'fused' (sm_90a fused compute+collective kernels over peer memory)."""
    global _COMM_BACKEND
    assert name in ("nccl", "fused")
    _COMM_BACKEND = name


def get_comm_backend() -> str:
    return _COMM_BACKEND


def _use_fused(x: torch.Tensor, group) -> bool:
    if _COMM_BACKEND != "fused" or not x.is_cuda or comm.group_size(group) == 1:
        return False
    from ...parallel import fused

    return fused.available(group)


def _fused_rs_variant(a: torch.Tensor, weight: torch.Tensor, group, transpose_b: bool) -> str:
    """Implementation of GEMM->reduce-scatter for this shape: 'fused' (one sm_90a kernel: GEMM, then the reduction of
    this rank's chunk) or 'lib' (GEMM + NCCL reduce-scatter).  Measured once per shape on the live tensors by
    `parallel.fused.rs_variant` - round 1
    used a fixed reduction-depth threshold (K >= 2048) taken from the TP=8 timings, which was wrong at other TP
    degrees and froze the library fallback in place."""
    from ...parallel import fused

    return fused.rs_variant(a, weight, group, transpose_b)


def _accumulate_wgrad(weight: torch.Tensor, dy2: torch.Tensor, x2: torch.Tensor) -> Optional[torch.Tensor]:
    """dW = dy2^T @ x2.  When the parameter carries a persistent `main_grad` buffer (fp32 or bf16 flat gradient
    arena owned by the optimizer wrapper) the GEMM accumulates straight into it and autograd gets None."""
    if getattr(weight, "_cb200_inplace_wgrad", False) and weight.grad is not None \
            and weight.grad.dtype == dy2.dtype and weight.grad.is_contiguous():
        # gradient accumulation (micro-batches): fold `grad += dW` into the GEMM epilogue.  Only enabled by plugins
        # that do not hang post-accumulate hooks on the parameter (autograd receives None for this weight).
        ops.matmul_tn(dy2, x2, out=weight.grad, accumulate=True)
        return None
    mg = getattr(weight, "main_grad", None)
    if mg is not None:
        if mg.dtype == dy2.dtype:
            ops.matmul_tn(dy2, x2, out=mg, accumulate=True)
        else:
            mg.add_(ops.matmul_tn(dy2, x2).to(mg.dtype))
        return None
    return ops.matmul_tn(dy2, x2)


def _maybe_defer_wgrad(weight, dy2, x2, use_zbv: bool):
    if use_zbv and WeightGradStore.enabled:
        def _w(dy2=dy2, x2=x2, weight=weight):
            g = _accumulate_wgrad(weight, dy2, x2)
            if g is not None:
                weight.grad = g if weight.grad is None else weight.grad + g

        WeightGradStore.put(_w)
        return None
    return _accumulate_wgrad(weight, dy2, x2)


# =============================================================================== plain linear (ZBV dW deferral)
class _LinearWithGradAccum(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x, weight, bias, use_zbv):
        ctx.save_for_backward(x, weight)
        ctx.use_bias, ctx.use_zbv = bias is not None, use_zbv
        return ops.linear_forward(x, weight, bias)

    @staticmethod
    def backward(ctx, dy):
        x, weight = ctx.saved_tensors
        dy2 = dy.reshape(-1, dy.shape[-1])
        dx = ops.matmul_nn(dy2, weight).view(x.shape) if ctx.needs_input_grad[0] else None
        dw = _maybe_defer_wgrad(weight, dy2, x.reshape(-1, x.shape[-1]), ctx.use_zbv)
        db = dy2.sum(0) if ctx.use_bias else None
        return dx, dw, db, None


def linear_with_grad_accum(x, weight, bias=None, use_zbv: bool = False):
    return _LinearWithGradAccum.apply(x, weight, bias, use_zbv)


# =============================================================================== TP column linear (no SP)
class _LinearWithAsyncComm(torch.autograd.Function):
    """y = x W^T; backward all-reduces dX over the TP group asynchronously while the dW GEMM runs."""

    @staticmethod
    def forward(ctx, x, weight, bias, group, async_grad_allreduce, use_zbv):
        ctx.save_for_backward(x, weight)
        ctx.use_bias, ctx.group, ctx.async_ar, ctx.use_zbv = bias is not None, group, async_grad_allreduce, use_zbv
        ctx.fp8 = comm.fp8_enabled()
        return ops.linear_forward(x, weight, bias)

    @staticmethod
    def backward(ctx, dy):
        x, weight = ctx.saved_tensors
        dy2 = dy.reshape(-1, dy.shape[-1])
        dx = ops.matmul_nn(dy2, weight).view(x.shape)
        handle = None
        if comm.group_size(ctx.group) > 1:
            if ctx.fp8:                                  # fp8 payloads: quantise -> exchange -> reduce in fp32
                with comm.fp8_communication(True):
                    dx = comm.all_reduce(dx.contiguous(), ctx.group)
            elif ctx.async_ar:
                handle = dist.all_reduce(dx, group=ctx.group, async_op=True)
            else:
                dist.all_reduce(dx, group=ctx.group)
        dw = _maybe_defer_wgrad(weight, dy2, x.reshape(-1, x.shape[-1]), ctx.use_zbv)
        db = dy2.sum(0) if ctx.use_bias else None
        if handle is not None:
            handle.wait()
        return dx, dw, db, None, None, None


def linear_with_async_comm(x, weight, bias, process_group, async_grad_allreduce: bool = True, use_zbv: bool = False):
    return _LinearWithAsyncComm.apply(x, weight, bias, process_group, async_grad_allreduce, use_zbv)


# =============================================================================== SP column linear: AG -> GEMM
def _ring_gather_gemm(x_local, weight, group, dim):
    """all-gather decomposed into ws-1 P2P hops, each overlapped with the GEMM on the chunk already present
    (reference `_ring_as_gather`, `_operation.py:418-482`)."""
    ws, r = comm.group_size(group), comm.group_rank(group)
    chunks = [None] * ws
    outs = [None] * ws
    cur = x_local.contiguous()
    chunks[r] = cur
    for step in range(ws):
        src = (r - step) % ws
        if step < ws - 1:
            nxt = torch.empty_like(cur)
            works = comm.send_recv_ring(cur, nxt, group)
        outs[src] = ops.linear_forward(cur, weight)
        if step < ws - 1:
            for w in works:
                w.wait()
            cur = nxt
            chunks[(r - step - 1) % ws] = cur
    return torch.cat(outs, dim=dim), torch.cat(chunks, dim=dim)


class _LinearGatherFwdReduceScatterBwd(torch.autograd.Function):
    """Megatron-SP column linear.  fwd: X = all_gather(x_local, dim); y = X W^T.
    bwd: dX = dY W -> reduce_scatter(dim) overlapped with dW = dY^T X (X re-gathered, not saved)."""

    @staticmethod
    def forward(ctx, x_local, weight, bias, group, dim, ring, use_zbv):
        ctx.group, ctx.dim, ctx.ring, ctx.use_zbv = group, dim, ring, use_zbv
        ctx.use_bias = bias is not None
        ctx.fp8 = comm.fp8_enabled()
        ctx.fused = _use_fused(x_local, group) and dim == 0 and x_local.dim() == 2 and not ctx.fp8
        ctx.saved_gathered = False
        if ctx.fused:
            from ...parallel import fused

            y, gathered = fused.all_gather_gemm(x_local, weight, group)
            if _SAVE_GATHERED:
                # keep the gathered activations for the wgrad GEMM instead of pulling them again in backward
                # (T x K bf16 per column-parallel linear; set CB200_SP_SAVE_GATHERED=0 to trade it for a re-gather)
                if bias is not None:
                    y = y + bias
                ctx.saved_gathered = True
                ctx.save_for_backward(gathered, weight)
                return y
        elif ring and comm.group_size(group) > 1:
            y, _ = _ring_gather_gemm(x_local, weight, group, dim)
        else:
            x_full = comm.all_gather(x_local, dim, group)
            y = ops.linear_forward(x_full, weight)
        if bias is not None:
            y = y + bias
        ctx.save_for_backward(x_local, weight)
        return y

    @staticmethod
    def backward(ctx, dy):
        x_local, weight = ctx.saved_tensors
        group, dim = ctx.group, ctx.dim
        ws = comm.group_size(group)
        dy2 = dy.reshape(-1, dy.shape[-1])
        if ctx.fused:
            from ...parallel import fused

            # dX = dY @ W fused with the reduce-scatter; X comes from forward (saved) or is re-gathered over NVLink
            x_full = x_local if ctx.saved_gathered else fused.all_gather(x_local, group)
            h_rs = None
            variant = _fused_rs_variant(dy2, weight, group, False)
            if variant != "lib":
                dx_local = fused.gemm_reduce_scatter(dy2, weight, group, transpose_b=False, variant=variant)
            else:
                # communication-bound shape: cuBLAS dgrad, NCCL reduce-scatter in flight under the wgrad GEMM
                dx_full = ops.matmul_nn(dy2, weight)
                dx_local = torch.empty((dx_full.shape[0] // ws, dx_full.shape[1]), dtype=dx_full.dtype,
                                       device=dx_full.device)
                h_rs = dist.reduce_scatter_tensor(dx_local, dx_full, group=group, async_op=True)
            dw = _maybe_defer_wgrad(weight, dy2, x_full, ctx.use_zbv)
            db = dy2.sum(0) if ctx.use_bias else None
            if h_rs is not None:
                h_rs.wait()
            return dx_local, dw, db, None, None, None, None
        if ctx.fp8 and ws > 1:
            with comm.fp8_communication(True):
                x_full = comm.all_gather(x_local.contiguous(), dim, group)
                dx_local = comm.reduce_scatter(ops.matmul_nn(dy2, weight).view(x_full.shape), dim, group)
            dw = _maybe_defer_wgrad(weight, dy2, x_full.reshape(-1, x_full.shape[-1]), ctx.use_zbv)
            db = dy2.sum(0) if ctx.use_bias else None
            return dx_local, dw, db, None, None, None, None
        # re-gather X (async) while computing dX
        x_local_c = x_local.contiguous()
        if ws > 1:
            gathered = torch.empty((ws,) + tuple(x_local_c.shape), dtype=x_local_c.dtype, device=x_local_c.device)
            h_ag = dist.all_gather_into_tensor(gathered.view(-1), x_local_c.view(-1), group=group, async_op=True)
        full_shape = list(x_local.shape)
        full_shape[dim] *= ws
        dx_full = ops.matmul_nn(dy2, weight).view(full_shape)
        if ws > 1:
            # reduce-scatter dX (async) overlapped with the wgrad GEMM
            if dim != 0:
                dx_send = dx_full.reshape(full_shape[:dim] + [ws, full_shape[dim] // ws] + full_shape[dim + 1:]) \
                    .movedim(dim, 0).contiguous()
            else:
                dx_send = dx_full.contiguous()
            dx_local = torch.empty_like(x_local_c)
            h_rs = dist.reduce_scatter_tensor(dx_local.view(-1), dx_send.view(-1), group=group, async_op=True)
            h_ag.wait()
            x_full = gathered.view([ws * x_local_c.shape[0]] + list(x_local_c.shape[1:])) if dim == 0 else \
                gathered.movedim(0, dim).reshape(full_shape)
        else:
            dx_local, x_full, h_rs = dx_full, x_local_c, None
        dw = _maybe_defer_wgrad(weight, dy2, x_full.reshape(-1, x_full.shape[-1]), ctx.use_zbv)
        db = dy2.sum(0) if ctx.use_bias else None
        if h_rs is not None:
            h_rs.wait()
        return dx_local, dw, db, None, None, None, None


def linear_gather_forward_reducescatter_backward(x_local, weight, bias, process_group, dim: int = 0,
                                                 ring: bool = False, use_zbv: bool = False):
    return _LinearGatherFwdReduceScatterBwd.apply(x_local, weight, bias, process_group, dim, ring, use_zbv)


# =============================================================================== SP row linear: GEMM -> RS
def _ring_gemm_reducescatter(x, weight, group, dim):
    """GEMM + reduce-scatter decomposed into ws-1 P2P hops of partial sums (reference `_ring_as_reducescatter`)."""
    ws, r = comm.group_size(group), comm.group_rank(group)
    xs = x.chunk(ws, dim=dim)
    acc = None
    for step in range(ws):
        # chunk owned (finally) by rank (r + ws - 1 - step) ... travel so that the last step computes our own chunk
        idx = (r - step - 1) % ws
        part = ops.linear_forward(xs[idx].contiguous(), weight)
        if acc is not None:
            part = part + acc
        if step < ws - 1:
            recv = torch.empty_like(part)
            for w in comm.send_recv_ring(part.contiguous(), recv, group):
                w.wait()
            acc = recv
        else:
            acc = part
    return acc


class _LinearReduceScatterFwdGatherBwd(torch.autograd.Function):
    """Megatron-SP row linear.  fwd: y_local = reduce_scatter(x W^T, dim).  bwd: dY = all_gather(dy_local);
    dX = dY W; dW = dY^T X."""

    @staticmethod
    def forward(ctx, x, weight, bias, group, dim, ring, use_zbv):
        ctx.group, ctx.dim, ctx.use_zbv = group, dim, use_zbv
        ctx.use_bias = bias is not None
        ctx.fp8 = comm.fp8_enabled()
        ctx.fused = _use_fused(x, group) and dim == 0 and x.dim() == 2 and not ctx.fp8
        ctx.save_for_backward(x, weight)
        if ctx.fused:
            from ...parallel import fused

            y = fused.gemm_reduce_scatter(x, weight, group, transpose_b=True)      # autotuned variant per shape
        elif ring and comm.group_size(group) > 1:
            y = _ring_gemm_reducescatter(x, weight, group, dim)
        else:
            y = comm.reduce_scatter(ops.linear_forward(x, weight), dim, group)
        if bias is not None:
            y = y + bias
        return y

    @staticmethod
    def backward(ctx, dy_local):
        x, weight = ctx.saved_tensors
        if ctx.fused:
            from ...parallel import fused

            dx, dy_full = fused.all_gather_gemm(dy_local.contiguous(), weight, group=ctx.group, transpose_b=False)
        else:
            with comm.fp8_communication(ctx.fp8):
                dy_full = comm.all_gather(dy_local.contiguous(), ctx.dim, ctx.group)
            dx = ops.matmul_nn(dy_full.reshape(-1, dy_full.shape[-1]), weight).view(x.shape)
        dy2 = dy_full.reshape(-1, dy_full.shape[-1])
        dw = _maybe_defer_wgrad(weight, dy2, x.reshape(-1, x.shape[-1]), ctx.use_zbv)
        db = dy_local.reshape(-1, dy_local.shape[-1]).sum(0) if ctx.use_bias else None
        return dx, dw, db, None, None, None, None


def linear_reducescatter_forward_gather_backward(x, weight, bias, process_group, dim: int = 0, ring: bool = False,
                                                 use_zbv: bool = False):
    return _LinearReduceScatterFwdGatherBwd.apply(x, weight, bias, process_group, dim, ring, use_zbv)


# =============================================================================== row linear w/o SP: GEMM -> AR
class _LinearAllReduceFwd(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x, weight, group, use_zbv):
        ctx.save_for_backward(x, weight)
        ctx.use_zbv = use_zbv
        if _use_fused(x, group) and x.dim() == 2 and not comm.fp8_enabled():
            from ...parallel import fused

            return fused.gemm_all_reduce(x, weight, group)
        y = ops.linear_forward(x, weight)
        comm.all_reduce(y, group)
        return y

    @staticmethod
    def backward(ctx, dy):
        x, weight = ctx.saved_tensors
        dy2 = dy.reshape(-1, dy.shape[-1])
        dx = ops.matmul_nn(dy2, weight).view(x.shape)
        dw = _maybe_defer_wgrad(weight, dy2, x.reshape(-1, x.shape[-1]), ctx.use_zbv)
        return dx, dw, None, None


def linear_allreduce_forward(x, weight, process_group, use_zbv: bool = False):
    return _LinearAllReduceFwd.apply(x, weight, process_group, use_zbv)


# =============================================================================== pure collective fwd/bwd pairs
class _ReduceForward(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x, group, grad_scale):
        ctx.grad_scale = grad_scale
        return comm.all_reduce(x.clone() if x.requires_grad else x, group)

    @staticmethod
    def backward(ctx, dy):
        if ctx.grad_scale is not None:
            dy = dy * ctx.grad_scale
        return dy, None, None


class _ReduceBackward(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x, group):
        ctx.group = group
        return x

    @staticmethod
    def backward(ctx, dy):
        return comm.all_reduce(dy.contiguous().clone(), ctx.group), None


class _GatherForwardSplitBackward(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x, dim, group, grad_scale):
        ctx.dim, ctx.group, ctx.grad_scale = dim, group, grad_scale
        return comm.all_gather(x, dim, group)

    @staticmethod
    def backward(ctx, dy):
        if ctx.grad_scale == "up":
            dy = dy * comm.group_size(ctx.group)
        elif ctx.grad_scale == "down":
            dy = dy / comm.group_size(ctx.group)
        return comm.split_along(dy, ctx.dim, ctx.group), None, None, None


class _SplitForwardGatherBackward(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x, dim, group, grad_scale):
        ctx.dim, ctx.group, ctx.grad_scale = dim, group, grad_scale
        return comm.split_along(x, dim, group)

    @staticmethod
    def backward(ctx, dy):
        if ctx.grad_scale == "up":
            dy = dy * comm.group_size(ctx.group)
        elif ctx.grad_scale == "down":
            dy = dy / comm.group_size(ctx.group)
        return comm.all_gather(dy.contiguous(), ctx.dim, ctx.group), None, None, None


class _GatherForwardReduceScatterBackward(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x, group, dim):
        ctx.dim, ctx.group = dim, group
        return comm.all_gather(x, dim, group)

    @staticmethod
    def backward(ctx, dy):
        return comm.reduce_scatter(dy.contiguous(), ctx.dim, ctx.group), None, None


class _ReduceScatterForwardGatherBackward(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x, group, dim):
        ctx.dim, ctx.group = dim, group
        return comm.reduce_scatter(x, dim, group)

    @staticmethod
    def backward(ctx, dy):
        return comm.all_gather(dy.contiguous(), ctx.dim, ctx.group), None, None


class _AllToAll(torch.autograd.Function):
    """Ulysses layout switch: scatter along `scatter_dim`, gather along `gather_dim` (bwd swaps the dims)."""

    @staticmethod
    def forward(ctx, x, group, scatter_dim, gather_dim):
        ctx.group, ctx.scatter_dim, ctx.gather_dim = group, scatter_dim, gather_dim
        return comm.all_to_all_single(x, scatter_dim, gather_dim, group)

    @staticmethod
    def backward(ctx, dy):
        return comm.all_to_all_single(dy.contiguous(), ctx.gather_dim, ctx.scatter_dim, ctx.group), None, None, None


def reduce_forward(x, process_group, grad_scale=None):
    return _ReduceForward.apply(x, process_group, grad_scale)


def reduce_backward(x, process_group):
    return _ReduceBackward.apply(x, process_group)


def gather_forward_split_backward(x, dim, process_group, grad_scale=None):
    return _GatherForwardSplitBackward.apply(x, dim, process_group, grad_scale)


def split_forward_gather_backward(x, dim, process_group, grad_scale=None):
    return _SplitForwardGatherBackward.apply(x, dim, process_group, grad_scale)


def gather_forward_reducescatter_backward(x, process_group, dim):
    return _GatherForwardReduceScatterBackward.apply(x, process_group, dim)


def reducescatter_forward_gather_backward(x, process_group, dim):
    return _ReduceScatterForwardGatherBackward.apply(x, process_group, dim)


def all_to_all_comm(x, process_group, scatter_dim: int = 1, gather_dim: int = 0):
    return _AllToAll.apply(x, process_group, scatter_dim, gather_dim)


# =============================================================================== SP helpers
def is_share_sp_tp(sp_mode: Optional[str]) -> bool:
    """split_gather / ring reuse the TP group for sequence parallelism."""
    return sp_mode in ("split_gather", "ring")


def split_batch_zigzag(x: torch.Tensor, sp_group: Optional[ProcessGroup], seq_dim: int = 1) -> torch.Tensor:
    """Zigzag split for causal ring attention: rank r keeps chunks {r, 2*sp-1-r} of 2*sp equal chunks."""
    sp = comm.group_size(sp_group)
    if sp == 1:
        return x
    r = comm.group_rank(sp_group)
    assert x.shape[seq_dim] % (2 * sp) == 0, f"seq len {x.shape[seq_dim]} must divide 2*sp={2 * sp}"
    chunks = x.chunk(2 * sp, dim=seq_dim)
    return torch.cat([chunks[r], chunks[2 * sp - 1 - r]], dim=seq_dim).contiguous()


def zigzag_positions(seq_len: int, sp_size: int, sp_rank: int, device=None) -> torch.Tensor:
    c = seq_len // (2 * sp_size)
    a = torch.arange(sp_rank * c, (sp_rank + 1) * c, device=device)
    b = torch.arange((2 * sp_size - 1 - sp_rank) * c, (2 * sp_size - sp_rank) * c, device=device)
    return torch.cat([a, b])


def gather_sp_output(hidden: torch.Tensor, sp_group, sp_mode: Optional[str], sp_dim: int = 0,
                     fp8_communication: bool = False) -> torch.Tensor:
    """Gather the sequence-sharded final hidden states (undoing zigzag for ring_attn)."""
    if comm.group_size(sp_group) == 1:
        return hidden
    scale = None if is_share_sp_tp(sp_mode) else "up"
    out = gather_forward_split_backward(hidden, sp_dim, sp_group, grad_scale=scale)
    if sp_mode == "ring_attn":
        sp = comm.group_size(sp_group)
        chunks = out.chunk(2 * sp, dim=sp_dim)
        order = [None] * (2 * sp)
        for r in range(sp):
            order[r] = chunks[2 * r]
            order[2 * sp - 1 - r] = chunks[2 * r + 1]
        out = torch.cat(order, dim=sp_dim)
    return out
