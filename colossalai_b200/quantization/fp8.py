"""FP8 casting, FP8-compressed collectives, DDP/FSDP comm hooks and the FP8 linear.

Parity: reference `colossalai/quantization/fp8.py` (cast_to_fp8:51, cast_from_fp8:93, all_reduce_fp8:187,
all_to_all_single_fp8:258, cast_{to,from}_fp8_pipeline:285/327, reduce_scatter_fp8:401, DDP/FSDP hooks:408-600,
all_to_all_fp8:648, all_gather_fp8:680, linear_fp8:842).

Design: the amax reduction + scaled cast run as native kernels (kernel/csrc/quant.cu), payloads travel as raw bytes
(`uint8` views) so the same code drives NCCL and gloo; the FP8 matmul is cuBLASLt's scaled GEMM (`torch._scaled_mm`) or, with
`CB200_FP8_GEMM=native`, the hand-written wgmma fp8 kernel (kernel/csrc/gemm_wgmma.cu).
"""
from __future__ import annotations

import ctypes
from typing import Any, Callable, List, Optional, Tuple

import torch
import torch.distributed as dist
import torch.nn.functional as F

from ..kernel import loader
from ..ops._align import aligned
from ..ops._dispatch import use_native
from ..ops._dtypes import code

__all__ = ["Handle", "cast_to_fp8", "cast_from_fp8", "all_reduce_fp8", "all_to_all_single_fp8", "reduce_scatter_fp8",
           "all_gather_fp8", "all_to_all_fp8", "cast_to_fp8_pipeline", "cast_from_fp8_pipeline", "linear_fp8",
           "fp8_compress_ddp_grad_comm_hook_async", "fp8_compress_ddp_grad_comm_hook_sync",
           "fp8_compress_fsdp_grad_comm_hook", "fp8_compress_fsdp_params_comm_hook", "process_group_is_intranode",
           "split_chunk_by_channel"]

_FP8 = {"e4m3": torch.float8_e4m3fn, "e5m2": torch.float8_e5m2}
_FMT_CODE = {"e4m3": 0, "e5m2": 1}
_lib = None


def _get_lib():
    global _lib
    if _lib is None:
        _lib = loader.load("cb200_quant")
    return _lib


class Handle:
    """Async work list + the tail ops (dequantise, concat) to run after the transfers land."""

    def __init__(self, handles: Optional[list] = None, remain_ops: Optional[Callable] = None) -> None:
        self.handles = handles or []
        self.remain_ops = remain_ops

    def wait(self) -> None:
        for h in self.handles:
            h.wait()
        if self.remain_ops:
            self.remain_ops()


def process_group_is_intranode(pg) -> bool:
    if pg is None:
        from torch.distributed.distributed_c10d import _get_default_group

        pg = _get_default_group()
    local = torch.cuda.device_count() if torch.cuda.is_available() else dist.get_world_size(pg)
    ranks = dist.get_process_group_ranks(pg)
    return len({r // max(local, 1) for r in ranks}) == 1


# ------------------------------------------------------------------------------------------------ casts
def cast_to_fp8(inp: torch.Tensor, fp8_format: str = "e4m3", per_channel_scale: bool = False,
                out: Optional[torch.Tensor] = None) -> Tuple[torch.Tensor, torch.Tensor]:
    """-> (fp8 tensor, scale_inv).  per-channel: one scale per row of the (2-D) input."""
    if inp.dtype not in (torch.float32, torch.float16, torch.bfloat16):
        raise TypeError("Only float16, bfloat16, and float32 are allowed.")
    fp8_type = _FP8[fp8_format]
    fp8_max = torch.finfo(fp8_type).max
    if inp.numel() == 0:
        return inp.to(fp8_type), torch.tensor([1.0], device=inp.device)
    if use_native(inp) and inp.is_contiguous():
        lib = _get_lib()
        q = out.view(torch.uint8) if out is not None else torch.empty(inp.shape, dtype=torch.uint8, device=inp.device)
        if per_channel_scale:   # scalar loads and stores: any address
            rows, cols = inp.numel() // inp.shape[-1], inp.shape[-1]
            sinv = torch.empty(rows, dtype=torch.float32, device=inp.device)
            loader.check(lib.cb_fp8_quant_rows(loader.ptr(inp), loader.ptr(q), rows, cols, ctypes.c_int64(cols),
                                               loader.ptr(sinv), code(inp.dtype), _FMT_CODE[fp8_format],
                                               loader.stream_ptr()), "fp8_quant_rows")
            loader.launch_counter.add("fp8_quant_rows")
            return q.view(fp8_type), sinv.unsqueeze(0)
        # the per-tensor kernels read 16-byte vectors of `inp` and write 16 / elsize bytes of `q` at a time
        inp = aligned(inp)
        q_out, q = q, aligned(q, 16 // inp.element_size())
        buf = torch.empty(2, dtype=torch.float32, device=inp.device)
        loader.check(lib.cb_fp8_quant_tensor(loader.ptr(inp), loader.ptr(q), ctypes.c_int64(inp.numel()),
                                             loader.ptr(buf[0:1]), loader.ptr(buf[1:2]), code(inp.dtype),
                                             _FMT_CODE[fp8_format], loader.stream_ptr()), "fp8_quant_tensor")
        loader.launch_counter.add("fp8_quant_tensor", 2)
        if q is not q_out:
            q_out.copy_(q)
        return q_out.view(fp8_type), buf[1:2]
    if per_channel_scale:
        amax = inp.abs().max(dim=-1).values.float()
        amax = torch.where(amax > 0, amax, torch.ones_like(amax))
        scale, scale_inv = fp8_max / amax[:, None], amax / fp8_max
    else:
        amax = inp.abs().max().float()
        amax = torch.where(amax > 0, amax, torch.ones_like(amax))
        scale, scale_inv = fp8_max / amax, amax / fp8_max
    ret = (scale * inp.float()).clamp(-fp8_max, fp8_max).to(fp8_type)
    if out is not None:
        out.copy_(ret)
        ret = out
    return ret, scale_inv.unsqueeze(0)


def cast_from_fp8(inp: torch.Tensor, scale_inv: torch.Tensor, ret_type: torch.dtype, per_channel_scale: bool = False,
                  out: Optional[torch.Tensor] = None) -> torch.Tensor:
    if inp.dtype not in (torch.float8_e4m3fn, torch.float8_e5m2):
        raise TypeError("Only float8_e4m3fn and float8_e5m2 are allowed.")
    if inp.numel() == 0:
        return inp.to(ret_type)
    if use_native(inp) and inp.is_contiguous() and ret_type in (torch.float32, torch.float16, torch.bfloat16):
        dst = out if out is not None else torch.empty(inp.shape, dtype=ret_type, device=inp.device)
        inp = aligned(inp, 4)   # read as 4-byte words; `dst` is written element by element
        sinv = scale_inv.reshape(-1).float().contiguous()
        cols = inp.shape[-1] if per_channel_scale else 0
        fmt = 0 if inp.dtype == torch.float8_e4m3fn else 1
        loader.check(_get_lib().cb_fp8_dequant(loader.ptr(inp), loader.ptr(dst), ctypes.c_int64(inp.numel()),
                                               loader.ptr(sinv), cols, code(dst.dtype), fmt, loader.stream_ptr()),
                     "fp8_dequant")
        loader.launch_counter.add("fp8_dequant")
        return dst
    s = scale_inv.reshape(-1)
    ret = (s[:, None] * inp.float()) if per_channel_scale else (s * inp.float())
    if out is not None:
        out.copy_(ret)
        return out
    return ret.to(ret_type)


# ------------------------------------------------------------------------------------------------ collectives
def _bytes(t: torch.Tensor) -> torch.Tensor:
    return t.view(torch.uint8)


def all_reduce_fp8(tensor: torch.Tensor, fp8_format: str = "e4m3", op=dist.ReduceOp.SUM, group=None,
                   async_op: bool = False) -> Optional[Handle]:
    """In-place all-reduce with fp8 payloads: fp8 all-to-all of chunks -> local fp32 reduction -> fp8 all-gather."""
    world = dist.get_world_size(group)
    if world == 1:
        return Handle() if async_op else None
    shape, dtype, n = tensor.shape, tensor.dtype, tensor.numel()
    fp8_type = _FP8[fp8_format]
    flat = tensor.reshape(-1)
    pad = (-n) % world
    if pad:
        flat = F.pad(flat, (0, pad))
    chunk = flat.numel() // world
    q, sinv = cast_to_fp8(flat.contiguous(), fp8_format)
    recv = torch.empty_like(_bytes(q))
    dist.all_to_all_single(recv, _bytes(q).contiguous(), group=group)
    scales = [torch.empty_like(sinv) for _ in range(world)]
    dist.all_gather(scales, sinv.contiguous(), group=group)
    acc = torch.zeros(chunk, dtype=torch.float32, device=tensor.device)
    for r in range(world):
        acc += cast_from_fp8(recv[r * chunk:(r + 1) * chunk].view(fp8_type), scales[r], torch.float32)
    if op == dist.ReduceOp.AVG:
        acc /= world
    q2, sinv2 = cast_to_fp8(acc, fp8_format)
    out_q = torch.empty(world * chunk, dtype=torch.uint8, device=tensor.device)
    out_s = [torch.empty_like(sinv2) for _ in range(world)]
    h1 = dist.all_gather_into_tensor(out_q, _bytes(q2).contiguous(), group=group, async_op=async_op)
    h2 = dist.all_gather(out_s, sinv2.contiguous(), group=group, async_op=async_op)

    def finish():
        parts = [cast_from_fp8(out_q[r * chunk:(r + 1) * chunk].view(fp8_type), out_s[r], dtype) for r in range(world)]
        tensor.copy_(torch.cat(parts)[:n].view(shape))

    if async_op:
        return Handle([h1, h2], finish)
    finish()
    return None


def all_to_all_single_fp8(output: torch.Tensor, input: torch.Tensor, output_split_sizes=None, input_split_sizes=None,
                          fp8_format: str = "e5m2", group=None, async_op: bool = False) -> Optional[Handle]:
    world = dist.get_world_size(group)
    fp8_type = _FP8[fp8_format]
    q, sinv = cast_to_fp8(input.contiguous(), fp8_format)
    row_bytes = int(q[0].numel()) if q.dim() > 1 else 1
    out_q = torch.empty(output.shape, dtype=torch.uint8, device=output.device)
    in_b, out_b = _bytes(q).reshape(-1), out_q.reshape(-1)
    osz = [s * row_bytes for s in output_split_sizes] if output_split_sizes is not None else None
    isz = [s * row_bytes for s in input_split_sizes] if input_split_sizes is not None else None
    h1 = dist.all_to_all_single(out_b, in_b, osz, isz, group=group, async_op=async_op)
    scales = [torch.empty_like(sinv) for _ in range(world)]
    h2 = dist.all_gather(scales, sinv.contiguous(), group=group, async_op=async_op)

    def finish():
        sizes = osz if osz is not None else [out_b.numel() // world] * world
        off = 0
        flat_out = output.reshape(-1)
        for r, sz in enumerate(sizes):
            if sz:
                flat_out[off:off + sz].copy_(cast_from_fp8(out_b[off:off + sz].view(fp8_type), scales[r], output.dtype))
            off += sz

    if async_op:
        return Handle([h1, h2], finish)
    finish()
    return None


def reduce_scatter_fp8(output: torch.Tensor, input_list: List[torch.Tensor], group=None, fp8_format: str = "e5m2",
                       async_op: bool = False) -> Optional[Handle]:
    world = dist.get_world_size(group)
    fp8_type = _FP8[fp8_format]
    qs, ss = zip(*[cast_to_fp8(t.contiguous(), fp8_format) for t in input_list])
    send = torch.cat([_bytes(q).reshape(-1) for q in qs])
    recv = torch.empty_like(send)
    h1 = dist.all_to_all_single(recv, send, group=group, async_op=async_op)
    my_scales = torch.cat([s.reshape(1) for s in ss])
    got_scales = torch.empty_like(my_scales)
    h2 = dist.all_to_all_single(got_scales, my_scales, group=group, async_op=async_op)

    def finish():
        n = output.numel()
        acc = torch.zeros(n, dtype=torch.float32, device=output.device)
        for r in range(world):
            acc += cast_from_fp8(recv[r * n:(r + 1) * n].view(fp8_type), got_scales[r:r + 1], torch.float32)
        output.copy_(acc.view(output.shape))

    if async_op:
        return Handle([h1, h2], finish)
    finish()
    return None


def all_gather_fp8(output_list: List[torch.Tensor], input_: torch.Tensor, group=None, fp8_format: str = "e5m2",
                   async_op: bool = False) -> Optional[Handle]:
    world = dist.get_world_size(group)
    fp8_type = _FP8[fp8_format]
    q, sinv = cast_to_fp8(input_.contiguous(), fp8_format)
    out_q = torch.empty(world * q.numel(), dtype=torch.uint8, device=input_.device)
    h1 = dist.all_gather_into_tensor(out_q, _bytes(q).reshape(-1), group=group, async_op=async_op)
    scales = [torch.empty_like(sinv) for _ in range(world)]
    h2 = dist.all_gather(scales, sinv.contiguous(), group=group, async_op=async_op)

    def finish():
        n = q.numel()
        for r in range(world):
            output_list[r].copy_(cast_from_fp8(out_q[r * n:(r + 1) * n].view(fp8_type), scales[r],
                                               output_list[r].dtype).view(output_list[r].shape))

    if async_op:
        return Handle([h1, h2], finish)
    finish()
    return None


def split_chunk_by_channel(chunk: torch.Tensor, channel_size: int, num_channels: int, rank: int = 0,
                           world_size: int = 1) -> List[torch.Tensor]:
    offset = chunk.numel() * rank
    end = offset + chunk.numel()
    brk = [x for x in range(0, channel_size * num_channels + 1, channel_size) if offset <= x <= end]
    if not brk or brk[0] > offset:
        brk.insert(0, offset)
    if brk[-1] < end:
        brk.append(end)
    sizes = [b - a for a, b in zip(brk[:-1], brk[1:])]
    return list(chunk.split(sizes))


def all_to_all_fp8(output_list: List[torch.Tensor], input_list: List[torch.Tensor], group=None,
                   fp8_format: str = "e5m2", async_op: bool = False) -> Optional[Handle]:
    """List all-to-all (uneven tensors allowed) with fp8 payloads."""
    world = dist.get_world_size(group)
    fp8_type = _FP8[fp8_format]
    qs, ss = zip(*[cast_to_fp8(t.contiguous(), fp8_format) for t in input_list])
    send = torch.cat([_bytes(q).reshape(-1) for q in qs])
    isz = [q.numel() for q in qs]
    osz = [o.numel() for o in output_list]
    recv = torch.empty(sum(osz), dtype=torch.uint8, device=send.device)
    h1 = dist.all_to_all_single(recv, send, osz, isz, group=group, async_op=async_op)
    my_scales = torch.cat([s.reshape(1) for s in ss])
    got = torch.empty_like(my_scales)
    h2 = dist.all_to_all_single(got, my_scales, group=group, async_op=async_op)

    def finish():
        off = 0
        for r in range(world):
            if osz[r]:
                output_list[r].copy_(cast_from_fp8(recv[off:off + osz[r]].view(fp8_type), got[r:r + 1],
                                                   output_list[r].dtype).view(output_list[r].shape))
            off += osz[r]

    if async_op:
        return Handle([h1, h2], finish)
    finish()
    return None


# ------------------------------------------------------------------------------------------------ pipeline p2p
def cast_to_fp8_pipeline(inp: Any) -> None:
    """In place: replace `inp["hidden_states"]` by its fp8 bytes (+ scale stored under "fp8_scale")."""
    if not isinstance(inp, dict) or "hidden_states" not in inp:
        return
    t = inp["hidden_states"]
    if t.dtype not in (torch.float16, torch.bfloat16, torch.float32):
        return
    inp["dtype"] = t.dtype
    q, sinv = cast_to_fp8(t.contiguous(), "e5m2" if t.requires_grad is False and False else "e4m3")
    inp["hidden_states"] = q
    inp["fp8_scale"] = sinv.float().reshape(1)


def cast_from_fp8_pipeline(inp: Any, del_metadata: bool = True) -> None:
    if not isinstance(inp, dict) or "fp8_scale" not in inp:
        return
    inp["hidden_states"] = cast_from_fp8(inp["hidden_states"], inp["fp8_scale"], inp.get("dtype", torch.bfloat16))
    if del_metadata:
        inp.pop("fp8_scale", None)
        inp.pop("dtype", None)


# ------------------------------------------------------------------------------------------------ DDP / FSDP hooks
def fp8_compress_ddp_grad_comm_hook_sync(process_group, bucket) -> torch.futures.Future:
    buf = bucket.buffer()
    all_reduce_fp8(buf, fp8_format="e5m2", group=process_group)
    buf.div_(dist.get_world_size(process_group))
    fut: torch.futures.Future = torch.futures.Future()
    fut.set_result(buf)
    return fut


def fp8_compress_ddp_grad_comm_hook_async(process_group, bucket) -> torch.futures.Future:
    """Two-phase fp8 all-reduce chained on futures (all-to-all -> reduce -> all-gather)."""
    group = process_group if process_group is not None else dist.group.WORLD
    world = dist.get_world_size(group)
    buf = bucket.buffer()
    n, dtype = buf.numel(), buf.dtype
    pad = (-n) % world
    flat = F.pad(buf, (0, pad)) if pad else buf
    chunk = flat.numel() // world
    q, sinv = cast_to_fp8(flat.contiguous(), "e5m2")
    recv = torch.empty(flat.numel(), dtype=torch.uint8, device=buf.device)
    scales = torch.empty(world, dtype=torch.float32, device=buf.device)
    f1 = dist.all_to_all_single(recv, _bytes(q).reshape(-1), group=group, async_op=True).get_future()
    dist.all_gather_into_tensor(scales, sinv.float().reshape(1), group=group)

    def reduce_and_gather(_):
        acc = torch.zeros(chunk, dtype=torch.float32, device=buf.device)
        for r in range(world):
            acc += cast_from_fp8(recv[r * chunk:(r + 1) * chunk].view(torch.float8_e5m2), scales[r:r + 1], torch.float32)
        acc /= world
        q2, s2 = cast_to_fp8(acc, "e5m2")
        out_q = torch.empty(world * chunk, dtype=torch.uint8, device=buf.device)
        out_s = torch.empty(world, dtype=torch.float32, device=buf.device)
        dist.all_gather_into_tensor(out_s, s2.float().reshape(1), group=group)
        dist.all_gather_into_tensor(out_q, _bytes(q2).reshape(-1), group=group)
        parts = [cast_from_fp8(out_q[r * chunk:(r + 1) * chunk].view(torch.float8_e5m2), out_s[r:r + 1], dtype)
                 for r in range(world)]
        buf.copy_(torch.cat(parts)[:n])
        return buf

    return f1.then(reduce_and_gather)


def fp8_compress_fsdp_grad_comm_hook(state: object, unsharded_gradient_flattened: torch.Tensor,
                                     sharded_gradient: torch.Tensor, group=None) -> None:
    """FSDP gradient hook: fp8 reduce-scatter of the flat gradient into this rank's shard."""
    world = dist.get_world_size(group)
    reduce_scatter_fp8(sharded_gradient, list(unsharded_gradient_flattened.chunk(world)), group=group,
                       fp8_format="e5m2")
    sharded_gradient.div_(world)


def fp8_compress_fsdp_params_comm_hook(state: object, padded_unsharded_flat_param: torch.Tensor,
                                       sharded_flat_param: torch.Tensor, group=None) -> None:
    """FSDP parameter all-gather with fp8 payloads."""
    world = dist.get_world_size(group)
    all_gather_fp8(list(padded_unsharded_flat_param.chunk(world)), sharded_flat_param, group=group, fp8_format="e4m3")


# ------------------------------------------------------------------------------------------------ fp8 linear
def _scaled_mm(a_q, a_sinv, b_q_t, b_sinv, out_dtype):
    """a_q [M,K] row-major fp8, b_q_t [K,N] column-major fp8 (i.e. the transpose view of a row-major [N,K])."""
    if a_q.is_cuda:
        from ..ops import gemm_native

        if gemm_native.fp8_backend() == "native" and gemm_native.available():
            b_nk = b_q_t.t()                       # the row-major [N, K] view behind the column-major operand
            if gemm_native.supported_fp8_nt(a_q, b_nk):
                return gemm_native.gemm_fp8_nt(a_q, b_nk, a_sinv, b_sinv, out_dtype)
        return torch._scaled_mm(a_q, b_q_t, scale_a=a_sinv.reshape(()).float(), scale_b=b_sinv.reshape(()).float(),
                                out_dtype=out_dtype)
    return ((a_q.float() * a_sinv.reshape(())) @ (b_q_t.float() * b_sinv.reshape(()))).to(out_dtype)


class _LinearFp8(torch.autograd.Function):
    """y = x W^T with e4m3 operands; dgrad / wgrad with e5m2 gradients."""

    @staticmethod
    def forward(ctx, x: torch.Tensor, w: torch.Tensor, bias: Optional[torch.Tensor]) -> torch.Tensor:
        ctx.x_shape, ctx.has_bias, ctx.out_dtype = x.shape, bias is not None, x.dtype
        x2 = x.reshape(-1, x.shape[-1]).contiguous()
        xq, xs = cast_to_fp8(x2, "e4m3")
        wq, wsc = cast_to_fp8(w.contiguous(), "e4m3")
        ctx.save_for_backward(xq, xs, wq, wsc)
        y = _scaled_mm(xq, xs, wq.t(), wsc, x.dtype)
        if bias is not None:
            y = y + bias
        return y.view(*x.shape[:-1], w.shape[0])

    @staticmethod
    def backward(ctx, gy: torch.Tensor):
        xq, xs, wq, wsc = ctx.saved_tensors
        g2 = gy.reshape(-1, gy.shape[-1]).contiguous()
        gq, gs = cast_to_fp8(g2, "e5m2")
        # dgrad: [M,N] x [N,K]  (second operand must be column-major: transpose of a contiguous [K,N])
        gx = _scaled_mm(gq, gs, wq.t().contiguous().t(), wsc, ctx.out_dtype)
        # wgrad: [N,M] x [M,K]
        gw = _scaled_mm(gq.t().contiguous(), gs, xq.t().contiguous().t(), xs, ctx.out_dtype)
        gb = g2.sum(0) if ctx.has_bias else None
        return gx.view(ctx.x_shape), gw, gb


def linear_fp8(input: torch.Tensor, weight: torch.Tensor, bias: Optional[torch.Tensor] = None) -> torch.Tensor:
    """Drop-in `F.linear` with fp8 tensor-core operands; falls back for shapes the scaled GEMM cannot take."""
    n_rows = input.numel() // max(input.shape[-1], 1)
    if (input.shape[-1] % 16 or weight.shape[0] % 16 or n_rows % 16
            or input.dtype not in (torch.float16, torch.bfloat16)):
        return F.linear(input, weight, bias)
    return _LinearFp8.apply(input, weight, bias)
