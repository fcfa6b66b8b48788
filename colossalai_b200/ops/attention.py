"""Attention front-end on token-major (packed / varlen) tensors.

q: [T, Hq, D]; k, v: [Tk, Hkv, D].  Sequences are either uniform (`batch` x `seqlen`) or described by
`cu_seqlens` (packed).  Backends: `native` = our sm_90a flash-attention (kernel/csrc/flash_attn_wgmma.cu),
`torch` = SDPA reference (CPU tier, oracle).  Parity: reference `ColoAttention.attention`
(`colossalai/shardformer/layer/attn.py:82-331`) and its FlashAttention*Loader dispatch.
"""
from __future__ import annotations

import math
from typing import Optional, Tuple

import torch
import torch.nn.functional as F

from ._dispatch import use_native

__all__ = ["attention", "attention_ref", "attention_with_lse_ref", "AttnMaskType"]


class AttnMaskType:
    CUSTOM = 0
    PADDED = 1
    CAUSAL = 2
    PADDED_CAUSAL = 3


def _sdpa(q, k, v, causal, scale, attn_mask=None):
    # q [B,Hq,Sq,D], k/v [B,Hkv,Sk,D]
    Hq, Hkv = q.shape[1], k.shape[1]
    if Hq != Hkv and q.is_cuda and attn_mask is None and q.shape[2] == k.shape[2]:
        # grouped-query attention handled inside the library kernel: no 4x K/V expansion, no reduce in backward
        try:
            return F.scaled_dot_product_attention(q, k, v, is_causal=causal, scale=scale, enable_gqa=True)
        except (TypeError, RuntimeError):
            pass
    if Hq != Hkv:
        rep = Hq // Hkv
        k = k.repeat_interleave(rep, dim=1)
        v = v.repeat_interleave(rep, dim=1)
    if causal and q.shape[2] != k.shape[2]:
        # bottom-right aligned causal mask (decode / chunked prefill)
        Sq, Sk = q.shape[2], k.shape[2]
        m = torch.ones(Sq, Sk, dtype=torch.bool, device=q.device).tril(diagonal=Sk - Sq)
        attn_mask = m if attn_mask is None else (attn_mask & m)
        causal = False
    return F.scaled_dot_product_attention(q, k, v, attn_mask=attn_mask, is_causal=causal and attn_mask is None,
                                          scale=scale)


def attention_ref(q: torch.Tensor, k: torch.Tensor, v: torch.Tensor, batch: int = 1, causal: bool = True,
                  scale: Optional[float] = None, cu_seqlens_q: Optional[torch.Tensor] = None,
                  cu_seqlens_k: Optional[torch.Tensor] = None, attn_mask: Optional[torch.Tensor] = None) -> torch.Tensor:
    T, Hq, D = q.shape
    if scale is None:
        scale = 1.0 / math.sqrt(D)
    if cu_seqlens_q is None:
        Sq, Sk = T // batch, k.shape[0] // batch
        qb = q.view(batch, Sq, Hq, D).transpose(1, 2)
        kb = k.view(batch, Sk, k.shape[1], D).transpose(1, 2)
        vb = v.view(batch, Sk, v.shape[1], v.shape[2]).transpose(1, 2)
        o = _sdpa(qb, kb, vb, causal, scale, attn_mask)
        return o.transpose(1, 2).reshape(T, Hq, v.shape[2])
    if cu_seqlens_k is None:
        cu_seqlens_k = cu_seqlens_q
    outs = []
    cq, ck = cu_seqlens_q.tolist(), cu_seqlens_k.tolist()
    for i in range(len(cq) - 1):
        qi = q[cq[i]:cq[i + 1]].transpose(0, 1).unsqueeze(0)
        ki = k[ck[i]:ck[i + 1]].transpose(0, 1).unsqueeze(0)
        vi = v[ck[i]:ck[i + 1]].transpose(0, 1).unsqueeze(0)
        outs.append(_sdpa(qi, ki, vi, causal, scale).squeeze(0).transpose(0, 1))
    return torch.cat(outs, 0)


def attention_with_lse_ref(q, k, v, batch: int = 1, causal: bool = True, scale: Optional[float] = None,
                           mask: Optional[torch.Tensor] = None) -> Tuple[torch.Tensor, torch.Tensor]:
    """Explicit-softmax reference that also returns the log-sum-exp ([T, Hq], fp32) — used by ring attention's
    online-softmax merge on the CPU tier and as the oracle for the native kernel's LSE."""
    T, Hq, D = q.shape
    Tk, Hkv = k.shape[0], k.shape[1]
    if scale is None:
        scale = 1.0 / math.sqrt(D)
    Sq, Sk = T // batch, Tk // batch
    qb = q.view(batch, Sq, Hq, D).transpose(1, 2).float()
    kb = k.view(batch, Sk, Hkv, D).transpose(1, 2).float().repeat_interleave(Hq // Hkv, dim=1)
    vb = v.view(batch, Sk, Hkv, v.shape[2]).transpose(1, 2).float().repeat_interleave(Hq // Hkv, dim=1)
    s = torch.matmul(qb, kb.transpose(-1, -2)) * scale
    if causal:
        m = torch.ones(Sq, Sk, dtype=torch.bool, device=q.device).tril(diagonal=Sk - Sq)
        s = s.masked_fill(~m, float("-inf"))
    if mask is not None:
        s = s.masked_fill(~mask, float("-inf"))
    lse = torch.logsumexp(s, dim=-1)  # [B,H,Sq]
    p = torch.exp(s - lse.unsqueeze(-1))
    p = torch.nan_to_num(p, nan=0.0)
    o = torch.matmul(p, vb)
    o = o.transpose(1, 2).reshape(T, Hq, v.shape[2]).to(q.dtype)
    return o, lse.transpose(1, 2).reshape(T, Hq)


def attention(q: torch.Tensor, k: torch.Tensor, v: torch.Tensor, batch: int = 1, causal: bool = True,
              scale: Optional[float] = None, cu_seqlens_q: Optional[torch.Tensor] = None,
              cu_seqlens_k: Optional[torch.Tensor] = None, max_seqlen: Optional[int] = None,
              attn_mask: Optional[torch.Tensor] = None, dropout_p: float = 0.0) -> torch.Tensor:
    """Scaled-dot-product attention with GQA on packed token-major tensors; returns [T, Hq, Dv]."""
    if use_native(q) and attn_mask is None and dropout_p == 0.0:
        from . import flash_attn_native as fa

        # packed (cu_seqlens) batches always take the native kernels when they can: the boundaries stay on the device and
        # one launch covers the whole batch (the library path below loops over sequences after a `.tolist()` host sync)
        needs_grad = torch.is_grad_enabled() and (q.requires_grad or k.requires_grad or v.requires_grad)
        packed = cu_seqlens_q is not None and (q.shape[-1] == 128 or (q.shape[-1] == 64 and not needs_grad))
        if fa.supported(q, k, v, cu_seqlens_q, cu_seqlens_k, force=packed):
            return fa.flash_attention(q, k, v, batch=batch, causal=causal, scale=scale, cu_seqlens_q=cu_seqlens_q)
    return attention_ref(q, k, v, batch, causal, scale, cu_seqlens_q, cu_seqlens_k, attn_mask)
