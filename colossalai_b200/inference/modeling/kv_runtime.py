"""Runtime object handed to the model as `kv_cache`: writes K/V into the paged cache and runs attention.

Replaces the reference's no-padding model forwards + attention backends (`inference/modeling/models/nopadding_llama.py`,
`modeling/backends/{attention_backend,pre_attention_backend}.py`): our generic model already works on flattened
un-padded tokens, so inference only has to (a) scatter the step's K/V into the block tables and (b) run varlen
flash-attention for prefill or the paged split-KV kernel for decode.
"""
from __future__ import annotations

from typing import List, Optional

import torch

from ... import ops
from ...ops import inference as iops

__all__ = ["PagedKVRuntime"]


class PagedKVRuntime:
    def __init__(self, k_caches: List[torch.Tensor], v_caches: List[torch.Tensor], block_size: int) -> None:
        self.k_caches, self.v_caches = k_caches, v_caches
        self.block_size = block_size
        self.block_tables: Optional[torch.Tensor] = None      # [bsz, max_blocks] int32 (device)
        self.seq_lens: Optional[torch.Tensor] = None          # [bsz] int32, INCLUDING the tokens of this step
        self.is_prompt = True
        self.token_seq: Optional[torch.Tensor] = None         # [tokens] int32 sequence index of every token
        self.token_pos: Optional[torch.Tensor] = None         # [tokens] int32 position of every token
        self.cu_seqlens: Optional[torch.Tensor] = None
        self.max_seqlen: int = 0
        self.q_per_seq: int = 1                               # decode: tokens verified per sequence (spec-dec)
        self.max_len_host: int = 0                            # longest sequence of the step (host side, no sync)
        self.cached_prefix = False                            # prompt step where some sequence hit the prefix cache
        self.chunk_seqs = 0                                   # chunked-prefill step: leading sequences feeding chunks
        self.chunk_tokens = 0                                 # ... and their rows, which come first

    def set_chunked_step(self, block_tables: torch.Tensor, seq_lens: torch.Tensor, num_cached: List[int],
                         device) -> torch.Tensor:
        """Prepare a chunked-prefill step; returns the int64 position of every input token.  The first
        B_p = len(num_cached) sequences feed a prompt chunk: positions num_cached[b] .. seq_lens[b] - 1, so `seq_lens`
        counts the cached tokens plus the chunk.  Every other sequence feeds one decode token, at seq_lens[i] - 1.
        Rows are the chunks, packed by `cu_seqlens` (which covers them only), then the decode rows."""
        self.block_tables = block_tables.to(device=device, dtype=torch.int32).contiguous()
        self.seq_lens = seq_lens.to(device=device, dtype=torch.int32).contiguous()
        self.is_prompt, self.q_per_seq, self.cached_prefix = False, 1, False
        lens = seq_lens.tolist()
        self.max_len_host = max(lens)
        bp = len(num_cached)
        new = [l - c for l, c in zip(lens[:bp], num_cached)] + [1] * (len(lens) - bp)
        seq = torch.repeat_interleave(torch.arange(len(lens)), torch.tensor(new))
        pos = torch.cat([torch.arange(l - n, l) for l, n in zip(lens, new)])
        cu = torch.zeros(bp + 1, dtype=torch.int32)
        cu[1:] = torch.cumsum(torch.tensor(new[:bp]), 0)
        self.cu_seqlens = cu.to(device)
        self.max_seqlen = max(new[:bp])
        self.chunk_seqs, self.chunk_tokens = bp, int(cu[-1])
        self.token_seq = seq.to(device=device, dtype=torch.int32)
        self.token_pos = pos.to(device=device, dtype=torch.int32)
        return pos.to(device=device, dtype=torch.int64)

    def set_step(self, block_tables: torch.Tensor, seq_lens: torch.Tensor, is_prompt: bool, device,
                 q_per_seq: int = 1, num_cached: Optional[List[int]] = None) -> torch.Tensor:
        """Prepare per-step metadata; returns the int64 position of every input token.  `num_cached` (prompt steps):
        per sequence, the leading prompt tokens whose K/V the cache already holds - only positions c_i .. L_i - 1 are
        fed, and `cu_seqlens` runs over L_i - c_i while `seq_lens` stays L_i."""
        self.block_tables = block_tables.to(device=device, dtype=torch.int32).contiguous()
        self.seq_lens = seq_lens.to(device=device, dtype=torch.int32).contiguous()
        self.is_prompt = is_prompt
        self.q_per_seq = q_per_seq
        lens = seq_lens.tolist()
        self.max_len_host = max(lens) if lens else 0
        self.cached_prefix = False
        self.chunk_seqs = 0
        if is_prompt:
            cached = num_cached if num_cached is not None else [0] * len(lens)
            self.cached_prefix = any(c > 0 for c in cached)
            new = [l - c for l, c in zip(lens, cached)]
            seq = torch.repeat_interleave(torch.arange(len(lens)), torch.tensor(new))
            pos = torch.cat([torch.arange(c, l) for c, l in zip(cached, lens)])
            cu = torch.zeros(len(lens) + 1, dtype=torch.int32)
            cu[1:] = torch.cumsum(torch.tensor(new), 0)
            self.cu_seqlens = cu.to(device)
            self.max_seqlen = max(new)
        else:
            seq = torch.repeat_interleave(torch.arange(len(lens)), q_per_seq)
            pos = torch.cat([torch.arange(l - q_per_seq, l) for l in lens])
            self.cu_seqlens = None
        self.token_seq = seq.to(device=device, dtype=torch.int32)
        self.token_pos = pos.to(device=device, dtype=torch.int32)
        return pos.to(device=device, dtype=torch.int64)

    def attend(self, layer_idx: int, q: torch.Tensor, k: torch.Tensor, v: torch.Tensor, meta, scale: float,
               alibi_slopes: Optional[torch.Tensor] = None, sliding_window: Optional[int] = None) -> torch.Tensor:
        kc, vc = self.k_caches[layer_idx], self.v_caches[layer_idx]
        iops.kv_cache_write(k, v, kc, vc, self.block_tables, self.token_seq, self.token_pos)
        if self.chunk_seqs:
            return self._attend_chunked(q, kc, vc, scale, alibi_slopes, sliding_window)
        if self.is_prompt and self.cached_prefix:
            # prefix-cache hit: the new rows attend over the cached prefix and their own K/V, all in the paged cache
            window = sliding_window if sliding_window is not None and self.max_len_host > sliding_window else None
            return iops.paged_prefill_attention(q, kc, vc, self.block_tables, self.cu_seqlens, self.seq_lens, scale,
                                                alibi_slopes=alibi_slopes, window=window)
        if sliding_window is not None and self.max_len_host > sliding_window:
            return self._attend_windowed(q, k, v, kc, vc, scale, alibi_slopes, sliding_window)
        return self._attend_full(q, k, v, kc, vc, scale, alibi_slopes)

    def _attend_chunked(self, q, kc, vc, scale, alibi_slopes, sliding_window) -> torch.Tensor:
        """Chunked-prefill step: the chunk rows attend through the paged prefill (each chunk follows its prompt's
        earlier chunks, already in the cache), the decode rows through the split-KV paged decode.  The boundaries
        are host values, so nothing syncs."""
        bp, tp = self.chunk_seqs, self.chunk_tokens
        window = sliding_window if sliding_window is not None and self.max_len_host > sliding_window else None
        out = iops.paged_prefill_attention(q[:tp], kc, vc, self.block_tables[:bp], self.cu_seqlens,
                                           self.seq_lens[:bp], scale, alibi_slopes=alibi_slopes, window=window)
        if tp == q.shape[0]:
            return out
        dec = iops.paged_decode_attention(q[tp:], kc, vc, self.block_tables[bp:], self.seq_lens[bp:], scale,
                                          alibi_slopes=alibi_slopes, window=window)
        return torch.cat([out, dec])

    def _native_prefill(self, q, k, v, scale, window: int, alibi_slopes) -> Optional[torch.Tensor]:
        """Sliding-window / ALiBi prefill inside the wgmma flash kernel (packed batch, device-resident boundaries);
        None when the tensors are outside the kernel's envelope (CPU tests, head_dim other than 64 / 128, fp32)."""
        from ...ops import flash_attn_native as fan

        q, k, v = q.contiguous(), k.contiguous(), v.contiguous()
        if not fan.supported(q, k, v, self.cu_seqlens, self.cu_seqlens, force=True):
            return None
        return fan.flash_prefill(q, k, v, self.cu_seqlens, scale, window=window, alibi_slopes=alibi_slopes)

    def _attend_windowed(self, q, k, v, kc, vc, scale, alibi_slopes, window: int) -> torch.Tensor:
        """Sliding-window attention (Mistral): a sequence longer than the window takes the banded reference path —
        prefill with an explicit band mask per sequence, decode over the last `window` cached tokens."""
        from ...ops.attention import attention_ref

        if self.is_prompt:
            native = self._native_prefill(q, k, v, scale, window, alibi_slopes)
            if native is not None:
                return native
            cu = self.cu_seqlens.tolist()
            outs = []
            for i in range(len(cu) - 1):
                a, b = cu[i], cu[i + 1]
                S = b - a
                pos = torch.arange(S, device=q.device)
                rel = pos[None, :] - pos[:, None]
                keep = (rel <= 0) & (rel > -window)
                bias = torch.zeros(S, S, device=q.device, dtype=torch.float32)
                if alibi_slopes is not None:
                    bias = rel.clamp(max=0).float()[None] * alibi_slopes.float()[:, None, None]
                bias = bias.expand(q.shape[1], S, S) if bias.dim() == 3 else bias[None].expand(q.shape[1], S, S)
                bias = bias.masked_fill(~keep[None], float("-inf")).to(q.dtype)[None]
                outs.append(attention_ref(q[a:b], k[a:b], v[a:b], batch=1, causal=False, scale=scale, attn_mask=bias))
            return torch.cat(outs, 0)
        return iops.paged_decode_attention(q, kc, vc, self.block_tables, self.seq_lens, scale,
                                           alibi_slopes=alibi_slopes, window=window, q_len=self.q_per_seq)

    def _attend_full(self, q, k, v, kc, vc, scale, alibi_slopes) -> torch.Tensor:
        if alibi_slopes is not None:
            # ALiBi families (Baichuan-13B, BLOOM): biased varlen prefill through the reference backend, the paged
            # decode kernel takes the slopes natively
            from .backends.attention_backend import AttentionMetaData, ReferenceAttentionBackend

            if self.is_prompt:
                native = self._native_prefill(q, k, v, scale, 0, alibi_slopes)
                if native is not None:
                    return native
                md = AttentionMetaData(q, k, v, kc, vc, self.block_tables, self.block_size, cu_seqlens=self.cu_seqlens,
                                       sm_scale=scale, alibi_slopes=alibi_slopes)
                return ReferenceAttentionBackend().prefill(md)
            return iops.paged_decode_attention(q, kc, vc, self.block_tables, self.seq_lens, scale,
                                               alibi_slopes=alibi_slopes, q_len=self.q_per_seq)
        if self.is_prompt:
            return ops.attention(q, k, v, causal=True, scale=scale, cu_seqlens_q=self.cu_seqlens,
                                 cu_seqlens_k=self.cu_seqlens, max_seqlen=self.max_seqlen)
        # decode (q_per_seq = 1) or speculative verification (q_per_seq tokens per sequence, each sees the cache up to
        # its own position): one pass over the cache either way
        return iops.paged_decode_attention(q, kc, vc, self.block_tables, self.seq_lens, scale, q_len=self.q_per_seq)
