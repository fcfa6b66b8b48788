"""Scaled masked / causal softmax (kernel/csrc/softmax.cu) with autograd.
Parity: reference `ScaledMaskedSoftmax` / `ScaledUpperTriangMaskedSoftmax` autograd functions
(colossalai/kernel/... `nn/layer/scaled_softmax.py:26-104`)."""
from __future__ import annotations

import ctypes
from typing import Optional

import torch

from ..kernel import loader
from ._dispatch import use_native
from ._dtypes import code

_lib = None


def _get_lib():
    global _lib
    if _lib is None:
        _lib = loader.load("cb200_softmax")
    return _lib


def scaled_masked_softmax_ref(x: torch.Tensor, mask: Optional[torch.Tensor], scale: float) -> torch.Tensor:
    s = x.float() * scale
    if mask is not None:
        s = s.masked_fill(mask.bool(), -10000.0)
    return torch.softmax(s, dim=-1).to(x.dtype)


def scaled_causal_softmax_ref(x: torch.Tensor, scale: float) -> torch.Tensor:
    sq, sk = x.shape[-2:]
    s = x.float() * scale
    keep = torch.ones(sq, sk, dtype=torch.bool, device=x.device).tril(diagonal=sk - sq)
    # with sq > sk the first sq - sk queries see no key: the kernel writes zeros there (softmax would give NaN),
    # and those rows are kept finite before the softmax so that its backward stays finite too
    empty = ~keep.any(-1, keepdim=True)
    s = s.masked_fill(~keep, float("-inf")).masked_fill(empty, 0.0)
    return torch.softmax(s, dim=-1).masked_fill(empty, 0.0).to(x.dtype)


class _ScaledMaskedSoftmax(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x, mask, scale):
        b, h, sq, sk = x.shape
        xc = x.contiguous()
        y = torch.empty_like(xc)
        m = None
        if mask is not None:
            m = mask.to(torch.uint8).contiguous()
            assert m.shape[-2:] == (sq, sk) and m.shape[0] in (1, b), "mask must be [b or 1, 1, sq, sk]"
        loader.check(_get_lib().cb_scaled_masked_softmax_fwd(
            loader.ptr(xc), loader.ptr(m), loader.ptr(y), ctypes.c_float(scale), b, h, sq, sk,
            1 if m is None else m.shape[0], code(x.dtype), loader.stream_ptr()), "scaled_masked_softmax_fwd")
        loader.launch_counter.add("scaled_masked_softmax_fwd")
        ctx.save_for_backward(y)
        ctx.scale = scale
        return y

    @staticmethod
    def backward(ctx, dy):
        (y,) = ctx.saved_tensors
        dyc = dy.contiguous()
        dx = torch.empty_like(y)
        rows = y.numel() // y.shape[-1]
        loader.check(_get_lib().cb_scaled_softmax_bwd(loader.ptr(dyc), loader.ptr(y), loader.ptr(dx),
                                                      ctypes.c_float(ctx.scale), ctypes.c_int64(rows), y.shape[-1],
                                                      code(y.dtype), loader.stream_ptr()), "scaled_softmax_bwd")
        loader.launch_counter.add("scaled_softmax_bwd")
        return dx, None, None


class _ScaledCausalSoftmax(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x, scale):
        sq, sk = x.shape[-2:]
        xc = x.contiguous()
        y = torch.empty_like(xc)
        loader.check(_get_lib().cb_scaled_causal_softmax_fwd(loader.ptr(xc), loader.ptr(y), ctypes.c_float(scale),
                                                             xc.numel() // (sq * sk), sq, sk, code(x.dtype),
                                                             loader.stream_ptr()), "scaled_causal_softmax_fwd")
        loader.launch_counter.add("scaled_causal_softmax_fwd")
        ctx.save_for_backward(y)
        ctx.scale = scale
        return y

    backward = _ScaledMaskedSoftmax.backward


def scaled_masked_softmax(x: torch.Tensor, mask: Optional[torch.Tensor], scale: float = 1.0) -> torch.Tensor:
    """x [b, heads, sq, sk]; mask [b or 1, 1, sq, sk] (True = masked out)."""
    if use_native(x) and x.dim() == 4:
        return _ScaledMaskedSoftmax.apply(x, mask, float(scale))
    return scaled_masked_softmax_ref(x, mask, scale)


def scaled_causal_softmax(x: torch.Tensor, scale: float = 1.0) -> torch.Tensor:
    """x [..., sq, sk] with the causal (upper-triangular) mask applied inside the kernel."""
    if use_native(x):
        return _ScaledCausalSoftmax.apply(x, float(scale))
    return scaled_causal_softmax_ref(x, scale)
