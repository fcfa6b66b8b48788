"""Fused RMSNorm / LayerNorm (fwd + bwd, optional fused residual add).

Native path: `kernel/csrc/norm.cu` (sm_90a).  Reference path (CPU tensors / CB200_FORCE_TORCH): plain PyTorch
fp32 math.  Parity: reference apex FusedRMSNorm / FusedLayerNorm wrappers
(`colossalai/shardformer/layer/normalization.py:27-135`) and `inference_ops.fused_add_rms_layernorm` (N17).
"""
from __future__ import annotations

import ctypes
from typing import Optional, Tuple

import torch

from ..kernel import loader
from ._align import aligned
from ._dispatch import use_native
from ._dtypes import code

_lib = None


def _get_lib():
    global _lib
    if _lib is None:
        lib = loader.load("cb200_norm")
        lib.cb_norm_max_hidden.restype = ctypes.c_int
        lib.cb_norm_bwd_grid.restype = ctypes.c_int
        _lib = lib
    return _lib


def _native_ok(x: torch.Tensor, w: torch.Tensor) -> bool:
    H = x.shape[-1]
    vec = 4 if x.dtype == torch.float32 else 8
    return (use_native(x) and x.dtype in (torch.float32, torch.float16, torch.bfloat16) and H % vec == 0
            and H <= 4096 * vec and w.dtype == x.dtype)


# ----------------------------------------------------------------------------------------------- reference
def rms_norm_ref(x, weight, eps, residual=None):
    h = x if residual is None else x + residual
    hf = h.float()
    rstd = torch.rsqrt(hf.pow(2).mean(-1, keepdim=True) + eps)
    y = (hf * rstd).to(x.dtype) * weight if weight.dtype != torch.float32 else (hf * rstd * weight).to(x.dtype)
    return (y, h) if residual is not None else y


def layer_norm_ref(x, weight, bias, eps):
    return torch.nn.functional.layer_norm(x.float(), (x.shape[-1],), weight.float(),
                                          None if bias is None else bias.float(), eps).to(x.dtype)


# ----------------------------------------------------------------------------------------------- native
class _RMSNormFn(torch.autograd.Function):
    """y = rmsnorm(x [+ residual]) * w.  With a residual the op also returns h = x + residual (the new residual
    stream); its incoming gradient is folded into dx inside the backward kernel."""

    @staticmethod
    def forward(ctx, x, weight, eps, residual):
        lib = _get_lib()
        shape = x.shape
        H = shape[-1]
        x2 = aligned(x.contiguous().view(-1, H))
        weight = aligned(weight)
        rows = x2.shape[0]
        y = torch.empty_like(x2)
        rstd = torch.empty(rows, dtype=torch.float32, device=x.device)
        has_res = residual is not None
        if has_res:
            r2 = aligned(residual.contiguous().view(-1, H))
            h = torch.empty_like(x2)
        else:
            r2, h = None, x2
        loader.check(lib.cb_rmsnorm_fwd(loader.ptr(x2), loader.ptr(r2), loader.ptr(weight), loader.ptr(y),
                                        loader.ptr(h if has_res else None), loader.ptr(rstd), rows, H,
                                        ctypes.c_float(eps), code(x.dtype), loader.stream_ptr()), "rmsnorm_fwd")
        loader.launch_counter.add("rmsnorm_fwd")
        ctx.save_for_backward(h, weight, rstd)
        ctx.has_res = has_res
        ctx.shape = shape
        if has_res:
            return y.view(shape), h.view(shape)
        return y.view(shape)

    @staticmethod
    def backward(ctx, dy, dh=None):
        lib = _get_lib()
        h, weight, rstd = ctx.saved_tensors
        rows, H = h.shape
        dy2 = aligned(dy.contiguous().view(-1, H))
        dres = aligned(dh.contiguous().view(-1, H)) if (ctx.has_res and dh is not None) else None
        dx = torch.empty_like(h)
        grid = lib.cb_norm_bwd_grid(rows)
        partial = torch.empty(grid, H, dtype=torch.float32, device=h.device)
        dw = torch.empty_like(weight)
        loader.check(lib.cb_rmsnorm_bwd(loader.ptr(dy2), loader.ptr(h), loader.ptr(weight), loader.ptr(rstd),
                                        loader.ptr(dres), loader.ptr(dx), loader.ptr(partial), loader.ptr(dw), 0,
                                        rows, H, code(h.dtype), loader.stream_ptr()), "rmsnorm_bwd")
        loader.launch_counter.add("rmsnorm_bwd", 2)
        dx = dx.view(ctx.shape)
        return dx, dw, None, (dx if ctx.has_res else None)


def rms_norm(x: torch.Tensor, weight: torch.Tensor, eps: float = 1e-6,
             residual: Optional[torch.Tensor] = None):
    """RMSNorm over the last dim.  With `residual`, returns `(norm(x + residual) * w, x + residual)`."""
    if _native_ok(x, weight):
        return _RMSNormFn.apply(x, weight, eps, residual)
    return rms_norm_ref(x, weight, eps, residual)


class _LayerNormFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x, weight, bias, eps):
        lib = _get_lib()
        shape = x.shape
        H = shape[-1]
        x2 = aligned(x.contiguous().view(-1, H))
        weight, bias = aligned(weight), aligned(bias)
        rows = x2.shape[0]
        y = torch.empty_like(x2)
        mean = torch.empty(rows, dtype=torch.float32, device=x.device)
        rstd = torch.empty_like(mean)
        loader.check(lib.cb_layernorm_fwd(loader.ptr(x2), loader.ptr(weight), loader.ptr(bias), loader.ptr(y),
                                          loader.ptr(mean), loader.ptr(rstd), rows, H, ctypes.c_float(eps),
                                          code(x.dtype), loader.stream_ptr()), "layernorm_fwd")
        loader.launch_counter.add("layernorm_fwd")
        ctx.save_for_backward(x2, weight, mean, rstd)
        ctx.has_bias = bias is not None
        ctx.shape = shape
        return y.view(shape)

    @staticmethod
    def backward(ctx, dy):
        lib = _get_lib()
        x2, weight, mean, rstd = ctx.saved_tensors
        rows, H = x2.shape
        dy2 = aligned(dy.contiguous().view(-1, H))
        dx = torch.empty_like(x2)
        grid = lib.cb_norm_bwd_grid(rows)
        pw = torch.empty(grid, H, dtype=torch.float32, device=x2.device)
        pb = torch.empty_like(pw)
        dw = torch.empty_like(weight)
        db = torch.empty_like(weight) if ctx.has_bias else None
        loader.check(lib.cb_layernorm_bwd(loader.ptr(dy2), loader.ptr(x2), loader.ptr(weight), loader.ptr(mean),
                                          loader.ptr(rstd), loader.ptr(dx), loader.ptr(pw), loader.ptr(pb),
                                          loader.ptr(dw), loader.ptr(db), 0, rows, H, code(x2.dtype),
                                          loader.stream_ptr()), "layernorm_bwd")
        loader.launch_counter.add("layernorm_bwd", 3 if ctx.has_bias else 2)
        return dx.view(ctx.shape), dw, db, None


def layer_norm(x: torch.Tensor, weight: torch.Tensor, bias: Optional[torch.Tensor] = None, eps: float = 1e-5):
    if _native_ok(x, weight) and (bias is None or bias.dtype == x.dtype):
        return _LayerNormFn.apply(x, weight, bias, eps)
    return layer_norm_ref(x, weight, bias, eps)
