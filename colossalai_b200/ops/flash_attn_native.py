"""ctypes face of the sm_90a flash-attention kernels (`kernel/csrc/flash_attn_wgmma.cu`): wgmma forward and wgmma
backward (dK / dV accumulated in registers per key tile over the whole GQA group, dQ through fp32 reductions).  This is
the only module that calls the `cb200_attn` library.

`CB200_FLASH_NATIVE=1` (or `enable(True)`) routes `ops.attention` and the ring-attention block functions through them
for equal-length bf16 / fp16 batches (head_dim 64 / 128 forward, 128 backward); everything else, and the default until
the kernels match the library's speed, goes to SDPA.  The backward of the head_dim-64 forward is `_block_bwd` (the
library flash backward through aten, given our log-sum-exp).  `flash_block_fwd` / `flash_block_bwd` / `flash_delta`
are the building blocks of the fused ring attention.
"""
from __future__ import annotations

import ctypes
import math
import os
from typing import Optional, Tuple

import torch

from ..kernel import loader
from ._dtypes import code
from .attention import attention_ref, attention_with_lse_ref

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


def _p(addr: int) -> ctypes.c_void_p:
    return ctypes.c_void_p(addr)


def _fwd(what: str, q: int, k: int, v: int, out: int, lse: int, batch: int, seqlen_q: int, seqlen_k: int, hq: int,
         hkv: int, d: int, causal: bool, scale: float, dtype: torch.dtype, o_state: int = 0, has_prev: bool = False,
         cu_seqlens: int = 0, total_tokens: int = 0, window: int = 0, alibi: int = 0, block_tables: int = 0,
         seq_lens: int = 0, block_size: int = 0, max_blocks: int = 0, num_blocks: int = 0) -> None:
    """`cb_flash_attn_fwd` on byte addresses (0 = null); the launcher picks uniform / packed / prefill / block / paged
    mode."""
    rc = _get_lib().cb_flash_attn_fwd(_p(q), _p(k), _p(v), _p(out), _p(lse), _p(o_state), int(has_prev),
                                      _p(cu_seqlens), ctypes.c_longlong(total_tokens), batch, seqlen_q, seqlen_k, hq,
                                      hkv, d, int(causal), ctypes.c_float(scale), int(window), _p(alibi),
                                      _p(block_tables), _p(seq_lens), int(block_size), int(max_blocks),
                                      int(num_blocks), code(dtype), loader.stream_ptr())
    loader.check(rc, what)


def flash_fwd(q: torch.Tensor, k: torch.Tensor, v: torch.Tensor, batch: int, causal: bool, scale: Optional[float],
              cu_seqlens: Optional[torch.Tensor] = None) -> Tuple[torch.Tensor, torch.Tensor]:
    """q [B*Sq, Hq, D], k / v [B*Sk, Hkv, D] -> (out [B*Sq, Hq, D], lse [B*Sq, Hq] fp32).  With `cu_seqlens`
    (int tensor [B+1], device resident - it is never copied to the host) the batch is packed / variable-length."""
    T, Hq, D = q.shape
    scale = scale if scale is not None else 1.0 / math.sqrt(D)
    out = torch.empty_like(q)
    lse = torch.empty(T, Hq, dtype=torch.float32, device=q.device)
    args = (q.data_ptr(), k.data_ptr(), v.data_ptr(), out.data_ptr(), lse.data_ptr())
    if cu_seqlens is not None:
        cu = _cu32(cu_seqlens, q.device)
        _fwd("flash_attn_varlen_fwd", *args, cu.numel() - 1, 0, 0, Hq, k.shape[1], D, causal, scale, q.dtype,
             cu_seqlens=cu.data_ptr(), total_tokens=T)
        loader.launch_counter.add("flash_attn_varlen_fwd")
        return out, lse
    _fwd("flash_attn_fwd", *args, batch, T // batch, k.shape[0] // batch, Hq, k.shape[1], D, causal, scale, q.dtype)
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
    _fwd("flash_attn_prefill", q.data_ptr(), k.data_ptr(), v.data_ptr(), out.data_ptr(), lse.data_ptr(),
         cu.numel() - 1, 0, 0, Hq, k.shape[1], D, True, scale, q.dtype, cu_seqlens=cu.data_ptr(), total_tokens=T,
         window=window or 0, alibi=slopes.data_ptr() if slopes is not None else 0)
    loader.launch_counter.add("flash_attn_prefill")
    return out


def flash_prefill_paged(q: torch.Tensor, k_cache: torch.Tensor, v_cache: torch.Tensor, block_tables: torch.Tensor,
                        cu_seqlens_q: torch.Tensor, seq_lens: torch.Tensor, scale: Optional[float], window: int = 0,
                        alibi_slopes: Optional[torch.Tensor] = None) -> torch.Tensor:
    """Causal prefill of new query rows against keys held in a paged KV cache.  q [T, Hq, D] packs the new rows of
    every sequence by `cu_seqlens_q` ([B+1]); sequence b's `seq_lens[b]` ([B], cached + new tokens) keys live in the
    caches [num_blocks, block_size, Hkv, D] (bf16 / fp16, q's dtype) at the blocks `block_tables[b]` ([B, max_blocks]),
    and its new rows sit at the last n_b of those positions.  `window` / `alibi_slopes` as `flash_prefill`, on absolute
    positions.  All index tensors stay on the device (no host sync); the table entries past a sequence's last block
    are never read.  Returns out [T, Hq, D]."""
    T, Hq, D = q.shape
    nb, bs, Hkv, _ = k_cache.shape
    scale = scale if scale is not None else 1.0 / math.sqrt(D)
    out = torch.empty_like(q)
    cu = _cu32(cu_seqlens_q, q.device)
    tables = block_tables.to(device=q.device, dtype=torch.int32).contiguous()
    lens = seq_lens.to(device=q.device, dtype=torch.int32).contiguous()
    slopes = alibi_slopes.to(device=q.device, dtype=torch.float32).contiguous() if alibi_slopes is not None else None
    _fwd("flash_attn_paged_prefill", q.data_ptr(), k_cache.data_ptr(), v_cache.data_ptr(), out.data_ptr(), 0,
         cu.numel() - 1, 0, 0, Hq, Hkv, D, True, scale, q.dtype, cu_seqlens=cu.data_ptr(), total_tokens=T,
         window=window or 0, alibi=slopes.data_ptr() if slopes is not None else 0, block_tables=tables.data_ptr(),
         seq_lens=lens.data_ptr(), block_size=bs, max_blocks=tables.shape[1], num_blocks=nb)
    loader.launch_counter.add("flash_attn_paged_prefill")
    return out


def flash_block_fwd(q: int, k: int, v: int, o_state: int, lse: int, rows: int, hq: int, hkv: int, d: int,
                    causal: bool, has_prev: bool, scale: float, dtype: torch.dtype) -> None:
    """Ring-attention block forward on byte addresses: `rows` queries (q [rows, hq, d]) against one key / value block
    (k / v [rows, hkv, d], possibly peer-mapped).  The fp32 online-softmax state (o_state [rows, hq, d], lse [rows, hq])
    is resumed when `has_prev` and written back merged with this block."""
    _fwd("flash_attn_block_fwd", q, k, v, 0, lse, 1, rows, rows, hq, hkv, d, causal, scale, dtype, o_state=o_state,
         has_prev=has_prev)


def flash_block_bwd(q: int, k: int, v: int, dout: int, lse: int, delta: int, dq_acc: int, dk_acc: int, dv_acc: int,
                    rows: int, hq: int, hkv: int, d: int, causal: bool, scale: float, dtype: torch.dtype) -> None:
    """Ring-attention block backward on byte addresses: adds this block's dQ into the fp32 `dq_acc` [rows, hq, d] and
    its dK / dV into the fp32 `dk_acc` / `dv_acc` [rows, hkv, d] (possibly peer-mapped); lse and delta [rows, hq] are
    those of the merged forward (`flash_delta`)."""
    rc = _get_lib().cb_flash_attn_block_bwd(_p(q), _p(k), _p(v), _p(dout), _p(lse), _p(delta), _p(dq_acc), _p(dk_acc),
                                            _p(dv_acc), rows, hq, hkv, d, int(causal), ctypes.c_float(scale),
                                            code(dtype), loader.stream_ptr())
    loader.check(rc, "flash_attn_block_bwd")


def flash_delta(out: torch.Tensor, dout: torch.Tensor) -> torch.Tensor:
    """delta = rowsum(dO o O): [T, H] fp32 for contiguous out / dout [T, H, D]."""
    T, H, D = out.shape
    delta = torch.empty(T, H, dtype=torch.float32, device=out.device)
    loader.check(_get_lib().cb_flash_attn_delta(loader.ptr(out), loader.ptr(dout), loader.ptr(delta),
                                                ctypes.c_longlong(T * H), D, code(out.dtype), loader.stream_ptr()),
                 "flash_attn_delta")
    return delta


def bwd_supported(q: torch.Tensor, k: torch.Tensor, batch: int) -> bool:
    return q.shape[-1] == 128 and q.shape[0] == k.shape[0]


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
                                      ctypes.c_float(scale), code(q.dtype), loader.ptr(cu), ctypes.c_longlong(T),
                                      loader.stream_ptr())
    loader.check(rc, "flash_attn_bwd")
    loader.launch_counter.add("flash_attn_bwd")
    return dq, dk, dv


# ------------------------------------------------------------------ one attention block with its log-sum-exp
def _to_bhsd(x: torch.Tensor, batch: int, rep: int = 1) -> torch.Tensor:
    T, H, D = x.shape
    xb = x.view(batch, T // batch, H, D).transpose(1, 2)
    return xb if rep == 1 else xb.repeat_interleave(rep, dim=1)


def _lib_flash_ok(q: torch.Tensor) -> bool:
    return q.is_cuda and q.dtype in (torch.float16, torch.bfloat16) and q.shape[-1] <= 256 and q.shape[-1] % 8 == 0 \
        and hasattr(torch.ops.aten, "_scaled_dot_product_flash_attention")


def _block_fwd(q, k, v, batch, causal, scale):
    """One attention block returning (out [T,Hq,D], lse [T,Hq] fp32): the native kernels when they take the call, else
    the library flash kernel through aten (it returns the log-sum-exp needed by the online-softmax merge); CPU:
    explicit softmax."""
    if q.is_cuda and supported(q, k, v, None):
        return flash_attention_with_lse(q, k, v, batch=batch, causal=causal, scale=scale)
    if _lib_flash_ok(q) and (not causal or q.shape[0] == k.shape[0]):
        g = q.shape[1] // k.shape[1]
        res = torch.ops.aten._scaled_dot_product_flash_attention(_to_bhsd(q, batch), _to_bhsd(k, batch, g),
                                                                 _to_bhsd(v, batch, g), 0.0, causal, False, scale=scale)
        out, lse = res[0], res[1]                       # [B,H,S,D], [B,H,S]
        return out.transpose(1, 2).reshape(q.shape), lse.transpose(1, 2).reshape(q.shape[0], q.shape[1])
    return attention_with_lse_ref(q, k, v, batch=batch, causal=causal, scale=scale)


def _block_bwd(do, q, k, v, o, lse, batch, causal, scale):
    """Gradients of one attention block GIVEN the final (merged) lse: p = exp(s - lse_final)."""
    if _lib_flash_ok(q) and (not causal or q.shape[0] == k.shape[0]) \
            and hasattr(torch.ops.aten, "_scaled_dot_product_flash_attention_backward"):
        Hq, Hkv = q.shape[1], k.shape[1]
        g = Hq // Hkv
        Sq, Sk = q.shape[0] // batch, k.shape[0] // batch
        qb, kb, vb = _to_bhsd(q, batch), _to_bhsd(k, batch, g), _to_bhsd(v, batch, g)
        ob, dob = _to_bhsd(o.to(q.dtype), batch), _to_bhsd(do.to(q.dtype), batch)
        lb = lse.view(batch, Sq, Hq).transpose(1, 2).contiguous().float()
        z = torch.zeros((), dtype=torch.int64, device=q.device)
        dq, dk, dv = torch.ops.aten._scaled_dot_product_flash_attention_backward(
            dob.contiguous(), qb.contiguous(), kb.contiguous(), vb.contiguous(), ob.contiguous(), lb, None, None, Sq, Sk,
            0.0, causal, z, z, scale=scale)
        dq = dq.transpose(1, 2).reshape(q.shape).float()
        dk = dk.float().view(batch, Hkv, g, Sk, -1).sum(2).transpose(1, 2).reshape(k.shape)
        dv = dv.float().view(batch, Hkv, g, Sk, -1).sum(2).transpose(1, 2).reshape(v.shape)
        return dq, dk, dv
    T, Hq, D = q.shape
    Tk, Hkv = k.shape[0], k.shape[1]
    Sq, Sk, g = T // batch, Tk // batch, Hq // Hkv
    qb = q.view(batch, Sq, Hq, D).transpose(1, 2).float()
    kb = k.view(batch, Sk, Hkv, D).transpose(1, 2).float().repeat_interleave(g, 1)
    vb = v.view(batch, Sk, Hkv, D).transpose(1, 2).float().repeat_interleave(g, 1)
    dob = do.view(batch, Sq, Hq, D).transpose(1, 2).float()
    ob = o.view(batch, Sq, Hq, D).transpose(1, 2).float()
    lb = lse.view(batch, Sq, Hq).transpose(1, 2).float()
    s = torch.matmul(qb, kb.transpose(-1, -2)) * scale
    if causal:
        m = torch.ones(Sq, Sk, dtype=torch.bool, device=q.device).tril(diagonal=Sk - Sq)
        s = s.masked_fill(~m, float("-inf"))
    p = torch.exp(s - lb.unsqueeze(-1))
    p = torch.nan_to_num(p, nan=0.0)
    dv = torch.matmul(p.transpose(-1, -2), dob)
    dp = torch.matmul(dob, vb.transpose(-1, -2))
    delta = (dob * ob).sum(-1, keepdim=True)
    ds = p * (dp - delta) * scale
    dq = torch.matmul(ds, kb)
    dk = torch.matmul(ds.transpose(-1, -2), qb)
    dq = dq.transpose(1, 2).reshape(T, Hq, D)
    dk = dk.view(batch, Hkv, g, Sk, D).sum(2).transpose(1, 2).reshape(Tk, Hkv, D)
    dv = dv.view(batch, Hkv, g, Sk, D).sum(2).transpose(1, 2).reshape(Tk, Hkv, D)
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
        return attention_with_lse_ref(q, k, v, batch=batch, causal=causal, scale=scale)
    return _FlashFn.apply(q, k, v, batch, causal, scale)


def flash_attention(q, k, v, batch: int = 1, causal: bool = True, scale: Optional[float] = None,
                    cu_seqlens_q: Optional[torch.Tensor] = None, **unused):
    if not shapes_ok(q, k, batch, causal, cu_seqlens_q):
        return attention_ref(q, k, v, batch, causal, scale, cu_seqlens_q)
    return _FlashFn.apply(q, k, v, batch, causal, scale, cu_seqlens_q)[0]
