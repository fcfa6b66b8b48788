"""Grouped (variable-M) linear: rows grouped by expert, one weight matrix per expert.

CUDA path: our wgmma grouped GEMM (`kernel/csrc/grouped_gemm_wgmma.cu`) - ONE persistent launch per GEMM walks a tile
list built on the device from the per-expert row counts (no host sync, no per-expert launches, no padding for the
forward / dgrad; the weight-gradient GEMM reduces over each expert's token rows and wants the row ranges aligned to the
128-row k-block, which `_pad_groups` arranges on the device when the caller's layout is not aligned already).
`CB200_GROUPED_GEMM=lib` selects `torch._grouped_mm` (library) instead; CPU tensors take a per-expert loop.
Replaces the reference's python loop over local experts (`shardformer/modeling/mixtral.py:177-191`).
"""
from __future__ import annotations

import ctypes
import os
from typing import Optional, Tuple

import torch

_lib = None
ALIGN = 128           # k-block of the wgrad kernel: group row ranges must start / end on multiples of it


def _get_lib():
    global _lib
    if _lib is None:
        from ..kernel import loader

        _lib = loader.load("cb200_grouped_gemm")
    return _lib


def native_ok(x: torch.Tensor, w: torch.Tensor) -> bool:
    if os.environ.get("CB200_GROUPED_GEMM", "native") != "native":
        return False
    return (x.is_cuda and x.dtype in (torch.bfloat16, torch.float16) and w.dtype == x.dtype and x.dim() == 2
            and w.dim() == 3 and x.shape[0] > 0 and x.shape[1] % 8 == 0 and w.shape[1] % 8 == 0 and w.shape[0] <= 512
            and w.is_contiguous() and torch.cuda.get_device_capability(x.device)[0] == 9)


def _offs(counts: torch.Tensor, device) -> torch.Tensor:
    return torch.cumsum(counts.to(device=device, dtype=torch.int64), 0).to(torch.int32)


def _native_fwd(x: torch.Tensor, w: torch.Tensor, offs: torch.Tensor, transpose_b: bool) -> torch.Tensor:
    """transpose_b: y = x @ w[e]^T with w [E, N, K];  else: y = x @ w[e] with w [E, K, N]."""
    from ..kernel import loader
    from ..ops._dtypes import code

    x = x.contiguous()
    E = w.shape[0]
    N = w.shape[1] if transpose_b else w.shape[2]
    K = x.shape[1]
    y = torch.empty(x.shape[0], N, dtype=x.dtype, device=x.device)
    rc = _get_lib().cb_grouped_gemm(loader.ptr(x), loader.ptr(w), loader.ptr(y), loader.ptr(offs), E, x.shape[0], N, K,
                                    x.stride(0), y.stride(0), int(transpose_b), code(x.dtype), loader.stream_ptr())
    loader.check(rc, "grouped_gemm")
    loader.launch_counter.add("grouped_gemm")
    return y


def _native_wgrad(dy: torch.Tensor, x: torch.Tensor, offs: torch.Tensor, E: int, out_dtype: torch.dtype) -> torch.Tensor:
    """dw[e] = dy[rows e]^T @ x[rows e]; every group's row range is a multiple of ALIGN."""
    from ..kernel import loader
    from ..ops._dtypes import code

    dy, x = dy.contiguous(), x.contiguous()
    M, N = dy.shape[1], x.shape[1]
    dw = torch.empty(E, M, N, dtype=out_dtype, device=x.device)
    rc = _get_lib().cb_grouped_gemm_wgrad(loader.ptr(dy), loader.ptr(x), loader.ptr(dw), loader.ptr(offs), E, x.shape[0],
                                          M, N, dy.stride(0), x.stride(0), code(x.dtype), code(out_dtype), 0,
                                          loader.stream_ptr())
    loader.check(rc, "grouped_gemm_wgrad")
    loader.launch_counter.add("grouped_gemm_wgrad")
    return dw


def _pad_groups(counts: torch.Tensor, rows: int, device) -> Tuple[torch.Tensor, torch.Tensor, int]:
    """Device-side map from the packed row layout to one where every group starts on a multiple of ALIGN.
    Returns (dest row of every packed row, padded cumulative offsets int32, static upper bound of padded rows)."""
    c = counts.to(device=device, dtype=torch.int64)
    E = c.numel()
    ends = torch.cumsum(c, 0)
    starts = ends - c
    pc = (c + ALIGN - 1) // ALIGN * ALIGN
    pends = torch.cumsum(pc, 0)
    pstarts = pends - pc
    row = torch.arange(rows, device=device)
    g = torch.searchsorted(ends, row, right=True)
    bound = (rows + E * (ALIGN - 1) + ALIGN - 1) // ALIGN * ALIGN
    # rows past the last group (a caller's over-allocated buffer) go to a dump row behind the padded layout
    dest = torch.where(g < E, row + (pstarts - starts)[g.clamp(max=E - 1)], torch.full_like(row, bound))
    return dest, pends.to(torch.int32), bound


class _GroupedLinearNative(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x, w, counts, aligned):
        offs = _offs(counts, x.device)
        ctx.save_for_backward(x, w, counts, offs)
        ctx.aligned = aligned
        return _native_fwd(x, w, offs, True)

    @staticmethod
    def backward(ctx, dy):
        x, w, counts, offs = ctx.saved_tensors
        dy = dy.contiguous()
        dx = dw = None
        if ctx.needs_input_grad[0]:
            if w.shape[1] % ALIGN == 0:
                dx = _native_fwd(dy, w, offs, False)         # dX = dY @ W[e]  (W [E, O, K] read as [E, K_red = O, N = K])
            else:
                dx = torch._grouped_mm(dy, w, offs=offs) if hasattr(torch, "_grouped_mm") else None
                if dx is None:
                    raise RuntimeError("grouped dgrad needs the expert output width to be a multiple of 128")
        if ctx.needs_input_grad[1]:
            if ctx.aligned:
                dw = _native_wgrad(dy, x, offs, w.shape[0], w.dtype)
            else:
                dest, poffs, bound = _pad_groups(counts, x.shape[0], x.device)
                xp = torch.zeros(bound + 1, x.shape[1], dtype=x.dtype, device=x.device).index_copy_(0, dest, x)
                dyp = torch.zeros(bound + 1, dy.shape[1], dtype=dy.dtype, device=x.device).index_copy_(0, dest, dy)
                dw = _native_wgrad(dyp[:bound], xp[:bound], poffs, w.shape[0], w.dtype)
        return dx, dw, None, None


class _GroupedLinear(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x, w, counts):
        # x [N, K]; w [E, O, K]; counts [E] (cpu or device int64)
        ctx.save_for_backward(x, w, counts)
        out = x.new_empty(x.shape[0], w.shape[1])
        c = counts.tolist()
        s = 0
        for e, n in enumerate(c):
            if n:
                out[s:s + n] = x[s:s + n] @ w[e].t()
            s += n
        return out

    @staticmethod
    def backward(ctx, dy):
        x, w, counts = ctx.saved_tensors
        dx = torch.empty_like(x)
        dw = torch.zeros_like(w)
        s = 0
        for e, n in enumerate(counts.tolist()):
            if n:
                dx[s:s + n] = dy[s:s + n] @ w[e]
                dw[e] = dy[s:s + n].t() @ x[s:s + n]
            s += n
        return dx, dw, None


def grouped_linear(x: torch.Tensor, w: torch.Tensor, counts: torch.Tensor, aligned: bool = False) -> torch.Tensor:
    """y[rows of expert e] = x[rows of expert e] @ w[e]^T.  `aligned`: the caller guarantees that every expert's row
    range starts and ends on a multiple of 128 (zero rows as padding) - the weight-gradient GEMM then runs without the
    re-layout pass."""
    if native_ok(x, w):
        return _GroupedLinearNative.apply(x, w, counts, aligned or getattr(counts, "cb200_aligned", False))
    if x.is_cuda and hasattr(torch, "_grouped_mm") and x.dtype == torch.bfloat16 and x.shape[0] > 0 \
            and x.shape[1] % 8 == 0 and w.shape[1] % 8 == 0:
        offs = _offs(counts, x.device)
        try:
            return torch._grouped_mm(x, w.transpose(-2, -1), offs=offs)
        except Exception:
            pass
    return _GroupedLinear.apply(x, w, counts.cpu() if counts.is_cuda else counts)
