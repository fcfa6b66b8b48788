"""Attention front-ends: `ColoAttention` (mask preparation + dispatch) and `RingAttention` (context parallel).

Parity: reference `colossalai/shardformer/layer/attn.py:82-331` (ColoAttention.prepare_attn_kwargs / attention)
and `:406-1247` (RingAttention: zigzag ring, online-softmax merge, dKV ring in backward, varlen).
H100-first: tensors are token-major `[T, H, D]`; on one NVSwitch box every peer is one hop, so the "double ring"
topology heuristics are dropped; KV (only the H_kv GQA heads, never repeat_kv'ed) is fetched from the owner rank —
through NCCL P2P on the baseline backend, straight from peer HBM inside the attention kernel on the fused backend.
"""
from __future__ import annotations

import math
from typing import Dict, Optional, Tuple

import torch
import torch.distributed as dist
from torch.distributed import ProcessGroup

from ... import ops
from ...ops.attention import AttnMaskType
from ...ops.flash_attn_native import _block_bwd, _block_fwd
from ...parallel import comm
from .utils import RingComm

__all__ = ["AttnMaskType", "ColoAttention", "RingAttention", "get_pad_info"]


def get_pad_info(padding_mask: torch.Tensor, invert: bool = False, return_indices: bool = True):
    """padding_mask [B, S] (1 = keep) -> (max_seqlen, cu_seqlens[int32], flat indices of kept tokens)."""
    if invert:
        padding_mask = padding_mask.logical_not()
    seqlens = padding_mask.sum(dim=-1, dtype=torch.int32)
    indices = torch.nonzero(padding_mask.flatten(), as_tuple=False).flatten() if return_indices else None
    max_seqlen = int(seqlens.max().item())
    cu = torch.nn.functional.pad(torch.cumsum(seqlens, 0, dtype=torch.int32), (1, 0))
    return max_seqlen, cu, indices


class ColoAttention:
    """Stateless attention dispatcher."""

    @staticmethod
    def prepare_attn_kwargs(shape_4d: Tuple[int, ...], dtype: torch.dtype, device: torch.device,
                            q_padding_mask: Optional[torch.Tensor] = None,
                            kv_padding_mask: Optional[torch.Tensor] = None, is_causal: bool = False,
                            invert: bool = True) -> Dict[str, torch.Tensor]:
        """Returns kwargs for `attention`: mask type, cu_seqlens / indices for padded batches."""
        b, _, s_q, s_kv = shape_4d
        out: Dict[str, torch.Tensor] = {}
        if q_padding_mask is None:
            out["attention_mask_type"] = AttnMaskType.CAUSAL if is_causal else AttnMaskType.CUSTOM
            return out
        if kv_padding_mask is None:
            kv_padding_mask = q_padding_mask
        max_q, cu_q, idx_q = get_pad_info(q_padding_mask, invert=False)
        max_kv, cu_kv, idx_kv = get_pad_info(kv_padding_mask, invert=False)
        out.update(cu_seqlens_q=cu_q, cu_seqlens_kv=cu_kv, max_seqlen_q=max_q, max_seqlen_kv=max_kv,
                   q_indices=idx_q, kv_indices=idx_kv,
                   attention_mask_type=AttnMaskType.PADDED_CAUSAL if is_causal else AttnMaskType.PADDED)
        return out

    @staticmethod
    def attention(q: torch.Tensor, k: torch.Tensor, v: torch.Tensor, attention_mask: Optional[torch.Tensor] = None,
                  attention_mask_type: int = AttnMaskType.CUSTOM, cu_seqlens_q=None, cu_seqlens_kv=None,
                  max_seqlen_q=None, max_seqlen_kv=None, q_indices=None, kv_indices=None, dropout_p: float = 0.0,
                  scale: Optional[float] = None, **kwargs) -> torch.Tensor:
        """q/k/v in the reference's [B, H, S, D] layout -> [B, H, S, D] (API-compatible entry point)."""
        B, Hq, Sq, D = q.shape
        causal = attention_mask_type in (AttnMaskType.CAUSAL, AttnMaskType.PADDED_CAUSAL)
        if attention_mask_type in (AttnMaskType.PADDED, AttnMaskType.PADDED_CAUSAL) and q_indices is not None:
            qt = q.transpose(1, 2).reshape(B * Sq, Hq, D)[q_indices]
            kt = k.transpose(1, 2).reshape(-1, k.shape[1], D)[kv_indices]
            vt = v.transpose(1, 2).reshape(-1, v.shape[1], v.shape[-1])[kv_indices]
            o = ops.attention(qt, kt, vt, causal=causal, scale=scale, cu_seqlens_q=cu_seqlens_q,
                              cu_seqlens_k=cu_seqlens_kv, max_seqlen=max_seqlen_q)
            full = q.new_zeros(B * Sq, Hq, v.shape[-1])
            full[q_indices] = o
            return full.view(B, Sq, Hq, -1).transpose(1, 2)
        qt = q.transpose(1, 2).reshape(B * Sq, Hq, D)
        kt = k.transpose(1, 2).reshape(-1, k.shape[1], D)
        vt = v.transpose(1, 2).reshape(-1, v.shape[1], v.shape[-1])
        mask = None
        if attention_mask is not None and attention_mask_type == AttnMaskType.CUSTOM:
            mask = attention_mask if attention_mask.dtype == torch.bool else attention_mask >= 0
        o = ops.attention(qt, kt, vt, batch=B, causal=causal, scale=scale, attn_mask=mask, dropout_p=dropout_p)
        return o.view(B, Sq, Hq, -1).transpose(1, 2)


# ======================================================================================= ring attention
def _merge(out: Optional[torch.Tensor], lse: Optional[torch.Tensor], blk_out: torch.Tensor, blk_lse: torch.Tensor):
    """Online-softmax merge of two partial attention results (fp32 out / lse)."""
    if out is None:
        return blk_out.float(), blk_lse.float()
    new_lse = torch.logaddexp(lse, blk_lse)
    w_old = torch.exp(lse - new_lse).unsqueeze(-1)
    w_new = torch.exp(blk_lse - new_lse).unsqueeze(-1)
    w_old = torch.nan_to_num(w_old, nan=0.0)
    w_new = torch.nan_to_num(w_new, nan=0.0)
    return out * w_old + blk_out.float() * w_new, new_lse


def _p2p_gather_kv(kv: torch.Tensor, sp_group) -> Optional[torch.Tensor]:
    """[2, T, Hkv, D] local KV -> [sp, 2, T, Hkv, D] from every rank by the P2P pull kernel, or None if unavailable."""
    import os

    if not kv.is_cuda or kv.dtype not in (torch.float16, torch.bfloat16) \
            or os.environ.get("CB200_RING_ATTN_P2P", "1") == "0":
        return None
    try:
        from ...parallel import fused

        if not fused.available(sp_group):
            return None
        flat = kv.reshape(1, -1)
        if flat.shape[1] % 8 != 0:
            return None
        return fused.all_gather(flat, sp_group).view((comm.group_size(sp_group),) + tuple(kv.shape))
    except Exception:
        return None


def _halves(x: torch.Tensor, batch: int):
    """Token-major [B*S_local, ...] -> (first half, second half) of every sequence (zigzag chunk pair)."""
    S = x.shape[0] // batch
    xb = x.view(batch, S, *x.shape[1:])
    return (xb[:, : S // 2].reshape(batch * (S // 2), *x.shape[1:]),
            xb[:, S // 2:].reshape(batch * (S // 2), *x.shape[1:]))


def _join_halves(a: torch.Tensor, b: torch.Tensor, batch: int) -> torch.Tensor:
    Sh = a.shape[0] // batch
    return torch.cat([a.view(batch, Sh, *a.shape[1:]), b.view(batch, Sh, *b.shape[1:])], 1) \
        .reshape(batch * 2 * Sh, *a.shape[1:])


class RingAttention(torch.autograd.Function):
    """Causal context-parallel attention over `sp_group` with zigzag-balanced sequence shards.

    Inputs are this rank's local tokens (zigzag chunk pair {r, 2*sp-1-r} of each sequence), token-major
    q [B*S_loc, Hq, D], k/v [B*S_loc, Hkv, D].  Forward circulates KV (GQA heads only) around the ring and merges
    block results with online softmax; backward circulates KV again together with fp32 dKV accumulators.
    """

    @staticmethod
    def forward(ctx, q, k, v, sp_group, batch, scale):
        sp, r = comm.group_size(sp_group), comm.group_rank(sp_group)
        D = q.shape[-1]
        if scale is None:
            scale = 1.0 / math.sqrt(D)
        ring = RingComm(sp_group)
        kv = torch.stack([k, v], 0).contiguous()
        out = lse = None
        q0, q1 = _halves(q, batch)
        out1 = lse1 = None  # second-half accumulators when only half of q participates
        cur = kv
        # NVSwitch path: every rank publishes its KV once in symmetric memory and the peers PULL all blocks in one
        # P2P kernel (no ring forwarding, no NCCL); the loop below then only indexes the gathered blocks
        kv_all = _p2p_gather_kv(kv, sp_group) if sp > 1 else None
        ctx.p2p = kv_all is not None
        for step in range(sp):
            nxt = None
            src = (r - step) % sp
            if kv_all is not None:
                cur = kv_all[src]
            elif step < sp - 1:
                nxt = ring.send_recv(cur)
            kk, vv = cur[0], cur[1]
            if step == 0:
                # local block.  zigzag halves: q0 x k0 causal; q1 x (k0 full, k1 causal)
                k0, k1 = _halves(kk, batch)
                v0, v1 = _halves(vv, batch)
                o00, l00 = _block_fwd(q0, k0, v0, batch, True, scale)
                o10, l10 = _block_fwd(q1, k0, v0, batch, False, scale)
                o11, l11 = _block_fwd(q1, k1, v1, batch, True, scale)
                oa, la = o00.float(), l00.float()
                ob, lb = _merge(*_merge(None, None, o10, l10), o11, l11)
            elif src < r:
                # every local q sees ONLY the first half (chunk src) of the remote KV, un-masked
                k0, _ = _halves(kk, batch)
                v0, _ = _halves(vv, batch)
                ob_, lb_ = _block_fwd(q, k0, v0, batch, False, scale)
                o0_, o1_ = _halves(ob_, batch)
                l0_, l1_ = _halves(lb_, batch)
                oa, la = _merge(oa, la, o0_, l0_)
                ob, lb = _merge(ob, lb, o1_, l1_)
            else:
                # only the second half of local q sees the remote KV (both chunks), un-masked
                o1_, l1_ = _block_fwd(q1, kk, vv, batch, False, scale)
                ob, lb = _merge(ob, lb, o1_, l1_)
            if nxt is not None:
                ring.wait()
                cur = nxt
        out = _join_halves(oa, ob, batch)
        lse = _join_halves(la, lb, batch)
        out_c = out.to(q.dtype)
        ctx.save_for_backward(q, k, v, out_c, lse)
        ctx.sp_group, ctx.batch, ctx.scale = sp_group, batch, scale
        return out_c

    @staticmethod
    def backward(ctx, dout):
        q, k, v, out, lse = ctx.saved_tensors
        sp_group, batch, scale = ctx.sp_group, ctx.batch, ctx.scale
        sp, r = comm.group_size(sp_group), comm.group_rank(sp_group)
        kv_ring, dkv_ring = RingComm(sp_group), RingComm(sp_group)
        dout = dout.contiguous()
        if getattr(ctx, "p2p", False):
            return RingAttention._backward_p2p(ctx, dout, q, k, v, out, lse)
        q0, q1 = _halves(q, batch)
        do0, do1 = _halves(dout, batch)
        o0, o1 = _halves(out, batch)
        l0, l1 = _halves(lse, batch)
        dq = torch.zeros_like(q, dtype=torch.float32)
        dq0, dq1 = _halves(dq, batch)
        dq0, dq1 = dq0.clone(), dq1.clone()
        cur = torch.stack([k, v], 0).contiguous()
        dkv = torch.zeros_like(cur, dtype=torch.float32)  # travels with the KV block it belongs to
        for step in range(sp):
            nxt = None
            if step < sp - 1:
                nxt = kv_ring.send_recv(cur)
            src = (r - step) % sp
            kk, vv = cur[0], cur[1]
            k0, k1 = _halves(kk, batch)
            v0, v1 = _halves(vv, batch)
            dk_blk = torch.zeros_like(kk, dtype=torch.float32)
            dv_blk = torch.zeros_like(vv, dtype=torch.float32)
            dk0, dk1 = _halves(dk_blk, batch)
            dv0, dv1 = _halves(dv_blk, batch)
            dk0, dk1, dv0, dv1 = dk0.clone(), dk1.clone(), dv0.clone(), dv1.clone()
            if step == 0:
                a, b, c = _block_bwd(do0, q0, k0, v0, o0, l0, batch, True, scale)
                dq0 += a; dk0 += b; dv0 += c
                a, b, c = _block_bwd(do1, q1, k0, v0, o1, l1, batch, False, scale)
                dq1 += a; dk0 += b; dv0 += c
                a, b, c = _block_bwd(do1, q1, k1, v1, o1, l1, batch, True, scale)
                dq1 += a; dk1 += b; dv1 += c
            elif src < r:
                a, b, c = _block_bwd(dout, q, k0, v0, out, lse, batch, False, scale)
                a0, a1 = _halves(a, batch)
                dq0 += a0; dq1 += a1; dk0 += b; dv0 += c
            else:
                a, b, c = _block_bwd(do1, q1, kk, vv, o1, l1, batch, False, scale)
                dq1 += a
                b0, b1 = _halves(b, batch)
                c0, c1 = _halves(c, batch)
                dk0 += b0; dk1 += b1; dv0 += c0; dv1 += c1
            contrib = torch.stack([_join_halves(dk0, dk1, batch), _join_halves(dv0, dv1, batch)], 0)
            # dkv accumulator arrives from the previous rank (it has been following this KV block)
            if step > 0:
                dkv_ring.wait()
                dkv = dkv_recv
            dkv = dkv + contrib
            if nxt is not None:
                kv_ring.wait()
                cur = nxt
            # pass the accumulator along with its KV block (after the last step it needs one more hop home)
            dkv_recv = dkv_ring.send_recv(dkv.contiguous())
        dkv_ring.wait()
        dkv = dkv_recv
        dq = _join_halves(dq0, dq1, batch)
        return dq.to(q.dtype), dkv[0].to(k.dtype), dkv[1].to(v.dtype), None, None, None

    @staticmethod
    def _backward_p2p(ctx, dout, q, k, v, out, lse):
        """Backward of the NVSwitch path: KV blocks are pulled again in one P2P kernel, every rank computes the dKV
        contributions of ALL blocks locally (fp32) and one fused reduce-scatter (in-switch reduction) returns each
        block's gradient to its owner."""
        from ...parallel import fused

        sp_group, batch, scale = ctx.sp_group, ctx.batch, ctx.scale
        sp, r = comm.group_size(sp_group), comm.group_rank(sp_group)
        kv_all = _p2p_gather_kv(torch.stack([k, v], 0).contiguous(), sp_group)
        q0, q1 = _halves(q, batch)
        do0, do1 = _halves(dout, batch)
        o0, o1 = _halves(out, batch)
        l0, l1 = _halves(lse, batch)
        dq0 = torch.zeros_like(q0, dtype=torch.float32)
        dq1 = torch.zeros_like(q1, dtype=torch.float32)
        dkv_all = torch.zeros((sp,) + tuple(kv_all.shape[1:]), dtype=torch.float32, device=q.device)
        for src in range(sp):
            kk, vv = kv_all[src][0], kv_all[src][1]
            k0, k1 = _halves(kk, batch)
            v0, v1 = _halves(vv, batch)
            if src == r:
                a, b, c = _block_bwd(do0, q0, k0, v0, o0, l0, batch, True, scale)
                dq0 += a
                dk0, dv0 = b.clone(), c.clone()
                a, b, c = _block_bwd(do1, q1, k0, v0, o1, l1, batch, False, scale)
                dq1 += a; dk0 += b; dv0 += c
                a, dk1, dv1 = _block_bwd(do1, q1, k1, v1, o1, l1, batch, True, scale)
                dq1 += a
                dkv_all[src, 0] = _join_halves(dk0, dk1, batch)
                dkv_all[src, 1] = _join_halves(dv0, dv1, batch)
            elif src < r:
                a, b, c = _block_bwd(dout, q, k0, v0, out, lse, batch, False, scale)
                a0, a1 = _halves(a, batch)
                dq0 += a0; dq1 += a1
                z = torch.zeros_like(b)
                dkv_all[src, 0] = _join_halves(b, z, batch)
                dkv_all[src, 1] = _join_halves(c, z, batch)
            else:
                a, b, c = _block_bwd(do1, q1, kk, vv, o1, l1, batch, False, scale)
                dq1 += a
                dkv_all[src, 0], dkv_all[src, 1] = b, c
        dkv = fused.reduce_scatter(dkv_all.view(sp, -1), sp_group).view(kv_all.shape[1:])
        dq = _join_halves(dq0, dq1, batch)
        return dq.to(q.dtype), dkv[0].to(k.dtype), dkv[1].to(v.dtype), None, None, None

    @staticmethod
    def attention(q, k, v, sp_group: ProcessGroup, batch: int = 1, scale: Optional[float] = None, **kwargs):
        """Entry point used by the model forwards."""
        if comm.group_size(sp_group) == 1:
            return ops.attention(q, k, v, batch=batch, causal=True, scale=scale)
        from . import ring_attn_fused as rf

        if rf.available(q, k, sp_group, batch):
            # sm_90a path: KV tiles are TMA-loaded from the owner's HBM inside the attention main loop, the softmax
            # state is merged in registers, dK / dV are reduced into the owner's accumulators (ring_attn_fused.py)
            return rf.ring_attention_fused(q, k, v, sp_group, batch, scale)
        return RingAttention.apply(q, k, v, sp_group, batch, scale)
