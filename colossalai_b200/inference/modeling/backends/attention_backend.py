"""Attention backends of the inference engine: prefill (varlen causal attention over the un-padded token stream) and
decode (paged split-KV attention over the block tables).

Parity: reference `colossalai/inference/modeling/backends/attention_backend.py:40-170` (`AttentionMetaData`,
`CudaAttentionBackend`, `TritonAttentionBackend`, `get_attention_backend`).  There is no Triton here: the CUDA backend
uses the flash varlen kernel for prefill and our sm_90a paged-decode kernel (`kernel/csrc/inference.cu`); the
reference backend is plain PyTorch (CPU tests, numerics oracle).
"""
from __future__ import annotations

from abc import ABC, abstractmethod
from dataclasses import dataclass
from typing import Optional

import torch

from .... import ops
from ....ops import inference as iops

__all__ = ["AttentionMetaData", "AttentionBackend", "CudaAttentionBackend", "ReferenceAttentionBackend",
           "get_attention_backend"]


@dataclass
class AttentionMetaData:
    query_states: torch.Tensor                 # [tokens, Hq, D]
    key_states: torch.Tensor                   # [tokens, Hkv, D]
    value_states: torch.Tensor
    k_cache: torch.Tensor                      # [blocks, block_size, Hkv, D]
    v_cache: torch.Tensor
    block_tables: torch.Tensor                 # [bsz, max_blocks] int32
    block_size: int
    kv_seq_len: int = None
    sequence_lengths: torch.Tensor = None      # [bsz] int32 (incl. this step's tokens)
    cu_seqlens: Optional[torch.Tensor] = None
    sm_scale: Optional[float] = None
    alibi_slopes: Optional[torch.Tensor] = None
    output_tensor: Optional[torch.Tensor] = None
    use_spec_dec: bool = False
    use_alibi_attn: bool = False


class AttentionBackend(ABC):
    @abstractmethod
    def prefill(self, attn_metadata: AttentionMetaData, **kwargs) -> torch.Tensor:
        ...

    @abstractmethod
    def decode(self, attn_metadata: AttentionMetaData, **kwargs) -> torch.Tensor:
        ...


class CudaAttentionBackend(AttentionBackend):
    """Flash varlen prefill + the hand-written paged decode kernel."""

    def prefill(self, m: AttentionMetaData, **kwargs) -> torch.Tensor:
        return ops.attention(m.query_states, m.key_states, m.value_states, causal=True, scale=m.sm_scale,
                             cu_seqlens_q=m.cu_seqlens, cu_seqlens_k=m.cu_seqlens, max_seqlen=m.kv_seq_len)

    def decode(self, m: AttentionMetaData, **kwargs) -> torch.Tensor:
        return iops.paged_decode_attention(m.query_states, m.k_cache, m.v_cache, m.block_tables, m.sequence_lengths,
                                           m.sm_scale, alibi_slopes=m.alibi_slopes)


class ReferenceAttentionBackend(AttentionBackend):
    """Pure PyTorch (any device): the oracle the CUDA backend is tested against."""

    def prefill(self, m: AttentionMetaData, **kwargs) -> torch.Tensor:
        q, k, v = m.query_states, m.key_states, m.value_states
        cu = m.cu_seqlens.tolist()
        G = q.shape[1] // k.shape[1]
        scale = m.sm_scale if m.sm_scale is not None else q.shape[-1] ** -0.5
        out = torch.empty_like(q)
        for a, b in zip(cu[:-1], cu[1:]):
            qi = q[a:b].transpose(0, 1).float()
            ki = k[a:b].repeat_interleave(G, 1).transpose(0, 1).float()
            vi = v[a:b].repeat_interleave(G, 1).transpose(0, 1).float()
            s = qi @ ki.transpose(1, 2) * scale
            L = b - a
            if m.alibi_slopes is not None:
                pos = torch.arange(L, device=q.device)
                s = s + m.alibi_slopes.float()[:, None, None] * (pos[None, :] - pos[:, None]).clamp(max=0)[None]
            s = s.masked_fill(~torch.ones(L, L, dtype=torch.bool, device=q.device).tril(), float("-inf"))
            out[a:b] = (s.softmax(-1) @ vi).transpose(0, 1).to(q.dtype)
        return out

    def decode(self, m: AttentionMetaData, **kwargs) -> torch.Tensor:
        return iops.paged_decode_attention_ref(m.query_states, m.k_cache, m.v_cache, m.block_tables,
                                               m.sequence_lengths, m.sm_scale, alibi_slopes=m.alibi_slopes)


def get_attention_backend(model_shard_infer_config=None, use_cuda_kernel: Optional[bool] = None) -> AttentionBackend:
    """CUDA backend when kernels are enabled and a GPU is present, otherwise the PyTorch reference."""
    if use_cuda_kernel is None:
        use_cuda_kernel = getattr(model_shard_infer_config, "use_cuda_kernel", True)
    if use_cuda_kernel and torch.cuda.is_available():
        return CudaAttentionBackend()
    return ReferenceAttentionBackend()
