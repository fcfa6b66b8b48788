"""Fused ring (context-parallel) attention over NVSwitch peer memory.

Reference being replaced: `RingAttention` in `colossalai/shardformer/layer/attn.py:406-1247` - a python ring of
flash-attn-2 calls with NCCL `batch_isend_irecv` of the (head-expanded) KV per hop, an elementwise `_rescale_out_lse`
pass per hop on a second stream, and fp32 dKV buffers circulating around the ring in backward.

H100-first design (one NVSwitch domain: every peer is one hop away at full bandwidth):

  * every rank PUBLISHES its K / V once per layer (GQA heads only) in a symmetric buffer; nobody forwards anything;
  * BACKWARD: the kernel of rank r reads the key / value tiles of block `src` STRAIGHT FROM RANK `src`'s HBM - its TMA
    loads are issued on a tensor map over the peer-mapped address, so the NVLink transfer is the kernel's own operand
    fetch (one CTA owns one key tile, so every remote byte crosses NVLink exactly once);
  * FORWARD: one CTA owns one QUERY tile and walks over the whole key block, so direct peer loads would pull the block
    once per query tile (peer memory is not cached in the local L2: measured at sp = 8, 16k local tokens, 34 GB per
    hop over NVLink and 1.47x slower than the library ring).  The forward therefore pulls the next hop's K/V block
    (GQA heads only, 67 MB at 16k tokens) over NVLink into a double-buffered local copy on a side stream while the
    tensor cores work on the current hop; the kernels then read it through the L2 like local K/V.  No up-front
    gather of all blocks, one hop of look-ahead;
  * the online-softmax state (fp32 output + log-sum-exp per query row) is carried from block to block INSIDE the
    kernel (`has_prev`): no separate merge / rescale pass, no fp32 `[T, H, D]` temporaries per hop;
  * backward: dQ accumulates locally in fp32 across blocks; the dK / dV contribution of rank r to block `src` is
    reduced by the kernel's epilogue directly into the OWNER's fp32 accumulator (vector `red.global.add.f32` on the
    peer mapping) - gradients travel once, as results, instead of following their KV block around the ring;
  * load balance uses the zigzag layout of the reference (chunk pair {r, 2 sp - 1 - r} per rank), so every rank runs
    the same number of equally sized blocks; with all-to-all connectivity the visiting ORDER is free, and rank r starts
    with its own block and then walks r-1, r-2, ... so the eight ranks never pull from the same peer at once.

Synchronisation is two stream-ordered control-plane barriers per layer (a 4-byte NCCL all-reduce): "everybody has
published" and, in backward, "everybody's reductions have landed".
"""
from __future__ import annotations

import math
import os
from typing import Dict, Optional, Tuple

import torch
import torch.distributed as dist

from ...kernel import loader
from ...ops import flash_attn_native as fa
from ...parallel import comm

__all__ = ["available", "ring_attention_fused", "stats"]

stats = {"fwd_blocks": 0, "bwd_blocks": 0, "layers_fwd": 0, "layers_bwd": 0}
_workspaces: Dict[tuple, "_RingWorkspace"] = {}


def available(q: torch.Tensor, k: torch.Tensor, sp_group, batch: int) -> bool:
    """bf16 / fp16, head_dim 128, CUDA, symmetric memory over the sp group, an even number of local tokens per
    sequence (zigzag chunk pair)."""
    if os.environ.get("CB200_RING_ATTN", "fused") != "fused":
        return False
    if not (q.is_cuda and q.dtype in (torch.bfloat16, torch.float16) and q.shape[-1] == 128):
        return False
    if q.shape[0] % (2 * batch) != 0 or k.shape[0] != q.shape[0] or q.shape[1] % k.shape[1] != 0:
        return False
    try:
        from ...parallel import fused

        return fused.available(sp_group)
    except Exception:
        return False


class _RingWorkspace:
    """Symmetric buffers of one (group, local KV size): published K/V (double-buffered for the forward, where one
    barrier per layer is enough) and the fp32 dK/dV accumulators peers reduce into."""

    def __init__(self, group, kv_bytes: int) -> None:
        from ...parallel.fused import _SymmBuffer

        self.group = group
        self.world = comm.group_size(group)
        self.rank = comm.group_rank(group)
        self.kv = [_SymmBuffer(kv_bytes, group), _SymmBuffer(kv_bytes, group)]
        self.dkv = _SymmBuffer(2 * kv_bytes, group, zero=True)        # fp32 accumulators: twice the 16-bit bytes
        # forward: local landing buffers for the next hop's K/V block + the side stream that fills them
        self.stage = [torch.empty(kv_bytes, dtype=torch.uint8, device="cuda") for _ in range(2)]
        self.copy_stream = torch.cuda.Stream()
        self.toggle = 0
        self.token = torch.zeros(1, device="cuda", dtype=torch.float32)
        torch.cuda.synchronize()
        dist.barrier(group=group)

    def peer_bytes(self, which: int, src: int, nbytes: int) -> torch.Tensor:
        """uint8 view of the first `nbytes` of rank `src`'s copy of published buffer `which` (peer-mapped memory)."""
        return self.kv[which].handle.get_buffer(src, (nbytes,), torch.uint8)

    def barrier(self) -> None:
        """Stream-ordered rendezvous of the group (control plane, 4 bytes over NCCL)."""
        dist.all_reduce(self.token, op=dist.ReduceOp.MAX, group=self.group)


def _workspace(group, kv_bytes: int) -> _RingWorkspace:
    size = 1 << max(20, (kv_bytes - 1).bit_length())
    key = (comm.group_key(group), size, torch.cuda.current_device())
    if key not in _workspaces:
        _workspaces[key] = _RingWorkspace(group, size)
    return _workspaces[key]


def _blocks(r: int, src: int):
    """(query half, key half, causal) block list of rank r against the KV of rank `src` under the zigzag layout:
    rank x holds chunks {x, 2 sp - 1 - x} as (half 0, half 1)."""
    if src == r:
        return [(0, 0, True), (1, 0, False), (1, 1, True)]
    if src < r:
        return [(0, 0, False), (1, 0, False)]        # both local chunks see the remote FRONT chunk, un-masked
    return [(1, 0, False), (1, 1, False)]            # only the local BACK chunk sees the remote block


def _visit_order(r: int, sp: int):
    return [(r - step) % sp for step in range(sp)]


class _FusedRing(torch.autograd.Function):
    @staticmethod
    def forward(ctx, q, k, v, sp_group, batch, scale):
        sp, r = comm.group_size(sp_group), comm.group_rank(sp_group)
        T, Hq, D = q.shape
        Hkv = k.shape[1]
        S = T // batch
        half = S // 2
        scale = scale if scale is not None else 1.0 / math.sqrt(D)
        es = q.element_size()
        kv_elems = T * Hkv * D
        ws = _workspace(sp_group, 2 * kv_elems * es)
        which = ws.toggle
        buf = ws.kv[which]
        ws.toggle ^= 1
        # publish K then V (one contiguous [2, T, Hkv, D] block in the symmetric buffer)
        kv_bytes = 2 * kv_elems * es
        pub = buf.tensor[:kv_bytes].view(q.dtype).view(2, T, Hkv, D)
        pub[0].copy_(k)
        pub[1].copy_(v)
        ws.barrier()
        main = torch.cuda.current_stream()
        published = torch.cuda.Event()
        published.record(main)
        order = _visit_order(r, sp)
        landed = [None] * sp            # event: hop i's block is in stage[i % 2]
        consumed = [None] * sp          # event: hop i's kernels are done with their K/V source

        def pull(i: int) -> None:
            with torch.cuda.stream(ws.copy_stream):
                ws.copy_stream.wait_event(published)
                if i >= 2 and consumed[i - 2] is not None:
                    ws.copy_stream.wait_event(consumed[i - 2])      # stage[i % 2] was read by hop i - 2
                ws.stage[i % 2][:kv_bytes].copy_(ws.peer_bytes(which, order[i], kv_bytes), non_blocking=True)
                landed[i] = torch.cuda.Event()
                landed[i].record(ws.copy_stream)

        staged = os.environ.get("CB200_RING_STAGE", "1") == "1"      # 0: the kernels read the peer block directly
        if sp > 1 and staged:
            pull(1)
        o_state = torch.empty(T, Hq, D, dtype=torch.float32, device=q.device)
        lse = torch.empty(T, Hq, dtype=torch.float32, device=q.device)
        row_q, row_kv, row_o, row_l = Hq * D * es, Hkv * D * es, Hq * D * 4, Hq * 4
        started = [[False, False] for _ in range(batch)]
        for i, src in enumerate(order):
            if i == 0 or not staged:
                base = buf.peer_ptrs[src]                    # own block: the published copy itself
            else:
                main.wait_event(landed[i])
                base = ws.stage[i % 2].data_ptr()
            if i + 1 < sp and staged:
                pull(i + 1)                                  # overlaps with this hop's kernels
            for b in range(batch):
                for qh, kh, causal in _blocks(r, src):
                    q_off = b * S + qh * half
                    k_off = b * S + kh * half
                    fa.flash_block_fwd(
                        q.data_ptr() + q_off * row_q, base + k_off * row_kv, base + (kv_elems * es) + k_off * row_kv,
                        o_state.data_ptr() + q_off * row_o, lse.data_ptr() + q_off * row_l, half, Hq, Hkv, D, causal,
                        started[b][qh], scale, q.dtype)
                    started[b][qh] = True
                    stats["fwd_blocks"] += 1
            consumed[i] = torch.cuda.Event()
            consumed[i].record(main)
        loader.launch_counter.add("ring_attn_block_fwd", sp * batch * 2 + batch)
        stats["layers_fwd"] += 1
        out = o_state.to(q.dtype)
        ctx.save_for_backward(q, k, v, out, lse)
        ctx.sp_group, ctx.batch, ctx.scale = sp_group, batch, scale
        return out

    @staticmethod
    def backward(ctx, dout):
        q, k, v, out, lse = ctx.saved_tensors
        sp_group, batch, scale = ctx.sp_group, ctx.batch, ctx.scale
        sp, r = comm.group_size(sp_group), comm.group_rank(sp_group)
        T, Hq, D = q.shape
        Hkv = k.shape[1]
        S = T // batch
        half = S // 2
        es = q.element_size()
        kv_elems = T * Hkv * D
        ws = _workspace(sp_group, 2 * kv_elems * es)
        buf = ws.kv[ws.toggle]
        ws.toggle ^= 1
        dout = dout.contiguous()
        pub = buf.tensor[: 2 * kv_elems * es].view(q.dtype).view(2, T, Hkv, D)
        pub[0].copy_(k)
        pub[1].copy_(v)
        acc = ws.dkv.tensor[: 2 * kv_elems * 4].view(torch.float32)
        acc.zero_()
        ws.barrier()                                  # K/V published and accumulators cleared everywhere
        delta = fa.flash_delta(out, dout)
        dq_acc = torch.zeros(T, Hq, D, dtype=torch.float32, device=q.device)
        row_q, row_kv, row_dq, row_l, row_acc = Hq * D * es, Hkv * D * es, Hq * D * 4, Hq * 4, Hkv * D * 4
        for src in _visit_order(r, sp):
            base = buf.peer_ptrs[src]
            acc_base = ws.dkv.peer_ptrs[src]
            for b in range(batch):
                for qh, kh, causal in _blocks(r, src):
                    q_off = b * S + qh * half
                    k_off = b * S + kh * half
                    fa.flash_block_bwd(
                        q.data_ptr() + q_off * row_q, base + k_off * row_kv, base + kv_elems * es + k_off * row_kv,
                        dout.data_ptr() + q_off * row_q, lse.data_ptr() + q_off * row_l,
                        delta.data_ptr() + q_off * row_l, dq_acc.data_ptr() + q_off * row_dq,
                        acc_base + k_off * row_acc, acc_base + kv_elems * 4 + k_off * row_acc, half, Hq, Hkv, D,
                        causal, scale, q.dtype)
                    stats["bwd_blocks"] += 1
        loader.launch_counter.add("ring_attn_block_bwd", sp * batch * 2 + batch)
        stats["layers_bwd"] += 1
        ws.barrier()                                  # every rank's reductions into my accumulators have landed
        dkv = acc.view(2, T, Hkv, D)
        dk, dv = dkv[0].to(k.dtype), dkv[1].to(v.dtype)
        return dq_acc.to(q.dtype), dk, dv, None, None, None


def ring_attention_fused(q: torch.Tensor, k: torch.Tensor, v: torch.Tensor, sp_group, batch: int = 1,
                         scale: Optional[float] = None) -> torch.Tensor:
    """Causal context-parallel attention of this rank's zigzag shard (token-major q [B*S_loc, Hq, D], k / v
    [B*S_loc, Hkv, D], contiguous) against the whole distributed sequence."""
    return _FusedRing.apply(q.contiguous(), k.contiguous(), v.contiguous(), sp_group, batch, scale)
