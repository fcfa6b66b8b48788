"""GEMMs on weight-only-quantised linears (`quantization/bnb.py`: `Linear4bit` nf4 / fp4, `Linear8bit` int8).

`wq_linear(x, layer)` = x @ W^T (forward), `wq_matmul_nn(dy, layer)` = dy @ W (input gradient), `dequantize(layer)` = W
in the layer's compute dtype.  On the GPU each GEMM decodes W with the native kernel (kernel/csrc/wq_gemm_wgmma.cu)
into a scratch weight that the dense wgmma GEMM (`ops/gemm_native.py`) consumes and that is freed right after, so at
most one layer's 16-bit weight is alive at a time and none is kept for backward.  This module is the only caller of
`cb200_wq_gemm`.

CPU tensors, an fp32 compute dtype and shapes outside the kernel's envelope take the PyTorch reference: dequantize,
then matmul.  On a GPU a missing library is an error, not a fallback.
"""
from __future__ import annotations

import torch
import torch.nn.functional as F

from ..kernel import loader
from . import gemm_native
from ._dispatch import use_native
from ._dtypes import code

__all__ = ["dequantize", "wq_linear", "wq_matmul_nn", "gemm_supported"]

_lib = None
_FMT_4BIT, _FMT_INT8 = 0, 1


def _get_lib():
    global _lib
    if _lib is None:
        _lib = loader.load("cb200_wq_gemm")
    return _lib


def _is_4bit(layer) -> bool:
    return hasattr(layer, "packed")


def _weight_args(layer):
    """(fmt, q, absmax, absmax_q, meta, code, N, K, block_size) of a quantised layer, as the launchers take them."""
    N, K = layer.out_features, layer.in_features
    if _is_4bit(layer):
        if layer.double_quant:
            return (_FMT_4BIT, layer.packed, None, layer.absmax_q, layer.absmax_meta, layer.code, N, K,
                    layer.block_size)
        return _FMT_4BIT, layer.packed, layer.absmax, None, None, layer.code, N, K, layer.block_size
    return _FMT_INT8, layer.weight_q, layer.scale, None, None, None, N, K, 0


def _aligned(t: torch.Tensor) -> bool:
    return t.data_ptr() % 16 == 0


def _native_weight(layer) -> bool:
    """The packed weight is on the GPU in a layout the kernels read (contiguous fp32 state, K a multiple of 8)."""
    fmt, q, absmax, absmax_q, meta, cb, N, K, bs = _weight_args(layer)
    if not (use_native(q) and layer.compute_dtype in (torch.bfloat16, torch.float16) and K % 8 == 0 and _aligned(q)):
        return False
    state = [t for t in (absmax, meta, cb) if t is not None]
    if any(t.dtype != torch.float32 or not t.is_contiguous() for t in state) or not q.is_contiguous():
        return False
    return fmt == _FMT_INT8 or bs % 8 == 0


def gemm_supported(layer) -> bool:
    """The native path's envelope on the weight side: N and K multiples of 8 (the dense GEMM's row alignment), 4-bit
    blocks of a multiple of 8 elements."""
    return _native_weight(layer) and layer.out_features % 8 == 0


def dequantize(layer) -> torch.Tensor:
    """W[N, K] in the layer's compute dtype, bitwise equal to the PyTorch reference `layer.dequantize_reference()`."""
    if not _native_weight(layer):
        return layer.dequantize_reference()
    fmt, q, absmax, absmax_q, meta, cb, N, K, bs = _weight_args(layer)
    out = torch.empty(N, K, dtype=layer.compute_dtype, device=q.device)
    rc = _get_lib().cb_wq_dequantize(fmt, loader.ptr(q), loader.ptr(absmax), loader.ptr(absmax_q), loader.ptr(meta),
                                     loader.ptr(cb), N, K, bs, loader.ptr(out), code(out.dtype), loader.stream_ptr())
    loader.check(rc, "wq_dequantize")
    loader.launch_counter.add("wq_dequantize")
    return out


def _operand_ok(a: torch.Tensor, layer) -> bool:
    return (a.dtype == layer.compute_dtype and a.stride(-1) == 1 and a.is_contiguous() and _aligned(a)
            and a.device == _weight_args(layer)[1].device)


def wq_linear(x: torch.Tensor, layer) -> torch.Tensor:
    """y[..., N] = x[..., K] @ W[N, K]^T in the layer's compute dtype (no bias)."""
    if gemm_supported(layer) and _operand_ok(x, layer):
        x2 = x.reshape(-1, x.shape[-1])
        return gemm_native.gemm_nt(x2, dequantize(layer)).view(x.shape[:-1] + (layer.out_features,))
    return F.linear(x.to(layer.compute_dtype), dequantize(layer))


def wq_matmul_nn(dy: torch.Tensor, layer) -> torch.Tensor:
    """dx[..., K] = dy[..., N] @ W[N, K] in the layer's compute dtype."""
    if gemm_supported(layer) and _operand_ok(dy, layer):
        dy2 = dy.reshape(-1, dy.shape[-1])
        return gemm_native.gemm_nn(dy2, dequantize(layer)).view(dy.shape[:-1] + (layer.in_features,))
    return dy.to(layer.compute_dtype) @ dequantize(layer)
