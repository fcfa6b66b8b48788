"""ctypes face of the sm_90a flash-attention kernels (`kernel/csrc/flash_attn_wgmma.cu`): wgmma forward and wgmma
backward (dK / dV accumulated in registers per key tile over the whole GQA group, dQ through fp32 reductions).

`CB200_FLASH_NATIVE=1` (or `enable(True)`) routes `ops.attention` and the ring-attention block functions through them
for equal-length bf16 / fp16 batches (head_dim 64 / 128 forward, 128 backward; sequence length a multiple of 128);
everything else, and the default until the kernels match the library's speed, goes to SDPA.  `CB200_FLASH_BWD=lib`
keeps the native forward but uses the library backward (which only needs q, k, v, out and our log-sum-exp).
"""
from __future__ import annotations

import ctypes
import math
import os
from typing import Optional, Tuple

import torch

from ..kernel import loader
from ._dtypes import code

_ENABLED = os.environ.get("CB200_FLASH_NATIVE", "0") == "1"
_lib = None


def _get_lib():
    global _lib
    if _lib is None:
        _lib = loader.load("cb200_attn")
    return _lib


def enable(flag: bool = True) -> None:
    global _ENABLED
    _ENABLED = flag


def _tensor_ok(t: torch.Tensor) -> bool:
    return t.is_cuda and t.dim() == 3 and t.dtype in (torch.bfloat16, torch.float16) and t.is_contiguous() \
        and t.data_ptr() % 16 == 0


def supported(q, k, v, cu_seqlens_q=None, cu_seqlens_k=None, force: bool = False) -> bool:
    """Can the native kernels take this call?  Packed batches (`cu_seqlens`) are supported for self attention (the same
    boundaries for queries and keys).  `force` ignores the CB200_FLASH_NATIVE switch (packed batches use the native
    kernels by default: the library path there is a python loop over sequences with a host sync)."""
    if not (_ENABLED or force) or not torch.cuda.is_available():
        return False
    if cu_seqlens_q is not None and cu_seqlens_k is not None and cu_seqlens_k is not cu_seqlens_q:
        return False
    if not (_tensor_ok(q) and _tensor_ok(k) and _tensor_ok(v)) or torch.cuda.get_device_capability()[0] != 9:
        return False
    D = q.shape[-1]
    return D in (64, 128) and k.shape[-1] == D and v.shape[-1] == D and q.shape[1] % k.shape[1] == 0 \
        and k.shape[1] == v.shape[1] and q.dtype == k.dtype == v.dtype


def shapes_ok(q, k, batch: int, causal: bool, cu_seqlens=None) -> bool:
    """Sequence lengths need not be multiples of the 128-row tile (partial tiles are masked inside the kernel)."""
    if cu_seqlens is not None:
        return q.shape[0] == k.shape[0]
    Sq, Sk = q.shape[0] // batch, k.shape[0] // batch
    return q.shape[0] % batch == 0 and k.shape[0] % batch == 0 and Sq > 0 and Sk > 0 and (not causal or Sq == Sk)


def _cu32(cu_seqlens: torch.Tensor, device) -> torch.Tensor:
    return cu_seqlens.to(device=device, dtype=torch.int32).contiguous()


def flash_fwd(q: torch.Tensor, k: torch.Tensor, v: torch.Tensor, batch: int, causal: bool, scale: Optional[float],
              cu_seqlens: Optional[torch.Tensor] = None) -> Tuple[torch.Tensor, torch.Tensor]:
    """q [B*Sq, Hq, D], k / v [B*Sk, Hkv, D] -> (out [B*Sq, Hq, D], lse [B*Sq, Hq] fp32).  With `cu_seqlens`
    (int tensor [B+1], device resident - it is never copied to the host) the batch is packed / variable-length."""
    T, Hq, D = q.shape
    scale = scale if scale is not None else 1.0 / math.sqrt(D)
    out = torch.empty_like(q)
    lse = torch.empty(T, Hq, dtype=torch.float32, device=q.device)
    if cu_seqlens is not None:
        cu = _cu32(cu_seqlens, q.device)
        rc = _get_lib().cb_flash_attn_varlen_fwd(loader.ptr(q), loader.ptr(k), loader.ptr(v), loader.ptr(out),
                                                 loader.ptr(lse), loader.ptr(cu), cu.numel() - 1,
                                                 ctypes.c_longlong(T), Hq, k.shape[1], D, int(causal),
                                                 ctypes.c_float(scale), code(q.dtype), loader.stream_ptr())
        loader.check(rc, "flash_attn_varlen_fwd")
        loader.launch_counter.add("flash_attn_varlen_fwd")
        return out, lse
    rc = _get_lib().cb_flash_attn_fwd(loader.ptr(q), loader.ptr(k), loader.ptr(v), loader.ptr(out), loader.ptr(lse),
                                      batch, T // batch, k.shape[0] // batch, Hq, k.shape[1], D, int(causal),
                                      ctypes.c_float(scale), code(q.dtype), loader.stream_ptr())
    loader.check(rc, "flash_attn_fwd")
    loader.launch_counter.add("flash_attn_fwd")
    return out, lse


def flash_prefill(q: torch.Tensor, k: torch.Tensor, v: torch.Tensor, cu_seqlens: torch.Tensor, scale: Optional[float],
                  window: int = 0, alibi_slopes: Optional[torch.Tensor] = None) -> torch.Tensor:
    """Inference prefill over a packed batch (causal, forward only) with the two mask families the serving models need
    inside the kernel: a sliding window (`window` > 0: query q sees keys (q - window, q]; key tiles left of every
    window are never loaded) and ALiBi (`alibi_slopes` [Hq] fp32: score += slope * (key - query)).  Replaces the
    per-sequence fp32 reference loops of the paged runtime (reference `kernel/triton/context_attn_unpad.py:193`,
    alibi variant)."""
    T, Hq, D = q.shape
    scale = scale if scale is not None else 1.0 / math.sqrt(D)
    out = torch.empty_like(q)
    lse = torch.empty(T, Hq, dtype=torch.float32, device=q.device)
    cu = _cu32(cu_seqlens, q.device)
    slopes = alibi_slopes.to(device=q.device, dtype=torch.float32).contiguous() if alibi_slopes is not None else None
    rc = _get_lib().cb_flash_attn_varlen_fwd_ex(
        loader.ptr(q), loader.ptr(k), loader.ptr(v), loader.ptr(out), loader.ptr(lse), loader.ptr(cu), cu.numel() - 1,
        ctypes.c_longlong(T), Hq, k.shape[1], D, ctypes.c_float(scale), int(window or 0),
        loader.ptr(slopes) if slopes is not None else ctypes.c_void_p(0), code(q.dtype), loader.stream_ptr())
    loader.check(rc, "flash_attn_varlen_fwd_ex")
    loader.launch_counter.add("flash_attn_prefill")
    return out


def bwd_supported(q: torch.Tensor, k: torch.Tensor, batch: int) -> bool:
    return (os.environ.get("CB200_FLASH_BWD", "native") == "native" and q.shape[-1] == 128 and q.shape[0] == k.shape[0])


def flash_bwd(q: torch.Tensor, k: torch.Tensor, v: torch.Tensor, out: torch.Tensor, dout: torch.Tensor,
              lse: torch.Tensor, batch: int, causal: bool, scale: Optional[float],
              cu_seqlens: Optional[torch.Tensor] = None):
    """Gradients of `flash_fwd` for self attention: returns (dq, dk, dv) in the input dtype."""
    T, Hq, D = q.shape
    Hkv = k.shape[1]
    scale = scale if scale is not None else 1.0 / math.sqrt(D)
    dout = dout.contiguous()
    dq, dk, dv = torch.empty_like(q), torch.empty_like(k), torch.empty_like(v)
    delta = torch.empty(T, Hq, dtype=torch.float32, device=q.device)
    dq_acc = torch.empty(T, Hq, D, dtype=torch.float32, device=q.device)
    cu = _cu32(cu_seqlens, q.device) if cu_seqlens is not None else None
    nb = (cu.numel() - 1) if cu is not None else batch
    rc = _get_lib().cb_flash_attn_bwd(loader.ptr(q), loader.ptr(k), loader.ptr(v), loader.ptr(out), loader.ptr(dout),
                                      loader.ptr(lse), loader.ptr(dq), loader.ptr(dk), loader.ptr(dv), loader.ptr(delta),
                                      loader.ptr(dq_acc), nb, (T // batch) if cu is None else 0, Hq, Hkv, D, int(causal),
                                      ctypes.c_float(scale), code(q.dtype),
                                      loader.ptr(cu) if cu is not None else ctypes.c_void_p(0), ctypes.c_longlong(T),
                                      loader.stream_ptr())
    loader.check(rc, "flash_attn_bwd")
    loader.launch_counter.add("flash_attn_bwd")
    return dq, dk, dv


class _FlashFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, q, k, v, batch, causal, scale, cu_seqlens=None):
        out, lse = flash_fwd(q, k, v, batch, causal, scale, cu_seqlens)
        ctx.save_for_backward(q, k, v, out, lse)
        ctx.batch, ctx.causal, ctx.scale, ctx.cu = batch, causal, scale, cu_seqlens
        return out, lse

    @staticmethod
    def backward(ctx, dout, dlse):
        from ..shardformer.layer.attn import _block_bwd

        q, k, v, out, lse = ctx.saved_tensors
        scale = ctx.scale if ctx.scale is not None else 1.0 / math.sqrt(q.shape[-1])
        if bwd_supported(q, k, ctx.batch):
            dq, dk, dv = flash_bwd(q, k, v, out, dout, lse, ctx.batch, ctx.causal, scale, ctx.cu)
        else:
            assert ctx.cu is None, "packed batches need head_dim 128 for the native backward"
            dq, dk, dv = _block_bwd(dout.contiguous(), q, k, v, out, lse, ctx.batch, ctx.causal, scale)
        return dq, dk, dv, None, None, None, None


def flash_attention_with_lse(q, k, v, batch: int = 1, causal: bool = True, scale: Optional[float] = None):
    if not shapes_ok(q, k, batch, causal):
        from .attention import attention_with_lse_ref

        return attention_with_lse_ref(q, k, v, batch=batch, causal=causal, scale=scale)
    return _FlashFn.apply(q, k, v, batch, causal, scale)


def flash_attention(q, k, v, batch: int = 1, causal: bool = True, scale: Optional[float] = None,
                    cu_seqlens_q: Optional[torch.Tensor] = None, **unused):
    if not shapes_ok(q, k, batch, causal, cu_seqlens_q):
        from .attention import attention_ref

        return attention_ref(q, k, v, batch, causal, scale, cu_seqlens_q)
    return _FlashFn.apply(q, k, v, batch, causal, scale, cu_seqlens_q)[0]
