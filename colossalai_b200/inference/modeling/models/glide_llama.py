"""GLIDE drafter: a small Llama whose layers carry an extra cross-attention block that "glimpses" the LARGE model's
KV cache (read straight out of the paged cache through the block tables), which lifts the draft acceptance rate.

Parity: reference `colossalai/inference/modeling/models/glide_llama.py:1-480` (`GlideLlamaConfig`,
`LlamaCrossAttention`, `GlideLlamaDecoderLayer`, `GlideLlamaForCausalLM`).
"""
from __future__ import annotations

import math
from dataclasses import dataclass
from typing import Dict, Optional

import torch
import torch.nn as nn
import torch.nn.functional as F

from ....models.config import ModelConfig
from ....models.transformer import DecoderLayer, TransformerLMHeadModel, build_norm
from ....ops.inference import gather_paged_kv
from ...spec.struct import GlideInput

__all__ = ["GlideLlamaConfig", "LlamaCrossAttention", "GlideLlamaDecoderLayer", "GlideLlamaForCausalLM",
           "gather_paged_kv"]


@dataclass
class GlideLlamaConfig(ModelConfig):
    """Drafter shape + the shape of the large model whose cache is glimpsed."""

    large_hidden_size: int = 4096
    large_num_attention_heads: int = 32
    large_num_key_value_heads: Optional[int] = None
    large_head_dim: Optional[int] = None

    def __post_init__(self) -> None:
        super().__post_init__()
        if self.large_num_key_value_heads is None:
            self.large_num_key_value_heads = self.large_num_attention_heads
        if self.large_head_dim is None:
            self.large_head_dim = self.large_hidden_size // self.large_num_attention_heads


class LlamaCrossAttention(nn.Module):
    """Queries from the drafter's hidden states, keys/values = the large model's cached K/V (no projection: the
    drafter learns to address the large model's key space directly)."""

    def __init__(self, cfg: GlideLlamaConfig) -> None:
        super().__init__()
        self.cfg = cfg
        self.num_heads, self.head_dim = cfg.large_num_attention_heads, cfg.large_head_dim
        self.num_kv_heads = cfg.large_num_key_value_heads
        self.q_proj = nn.Linear(cfg.hidden_size, self.num_heads * self.head_dim, bias=False)
        self.o_proj = nn.Linear(self.num_heads * self.head_dim, cfg.hidden_size, bias=False)

    def forward(self, x: torch.Tensor, glide: GlideInput, batch: int) -> torch.Tensor:
        """`x` [B*S, H] batch-major; sequence b attends to the first `sequence_lengths[b]` cached tokens."""
        T = x.shape[0]
        S = T // batch
        q = self.q_proj(x).reshape(batch, S, self.num_heads, self.head_dim).transpose(1, 2)
        G = self.num_heads // self.num_kv_heads
        outs = []
        for b in range(batch):
            L = int(glide.sequence_lengths[b])
            k = gather_paged_kv(glide.large_k_cache, glide.block_tables[b], L, q.dtype)
            v = gather_paged_kv(glide.large_v_cache, glide.block_tables[b], L, q.dtype)
            k = k.repeat_interleave(G, 1).transpose(0, 1)
            v = v.repeat_interleave(G, 1).transpose(0, 1)
            outs.append(F.scaled_dot_product_attention(q[b], k, v, scale=1.0 / math.sqrt(self.head_dim)))
        o = torch.stack(outs, 0).transpose(1, 2).reshape(T, self.num_heads * self.head_dim)
        return self.o_proj(o)


class GlideLlamaDecoderLayer(DecoderLayer):
    def __init__(self, cfg: GlideLlamaConfig, layer_idx: int) -> None:
        super().__init__(cfg, layer_idx)
        self.cross_attn = LlamaCrossAttention(cfg)
        self.cross_attn_layernorm = build_norm(cfg)
        self.glide_input: Optional[GlideInput] = None

    def forward(self, x: torch.Tensor, meta, rope=None, kv_cache=None) -> torch.Tensor:
        x = x + self.self_attn(self.input_layernorm(x), meta, rope, kv_cache)
        g = self.glide_input
        if g is not None and g.glimpse_ready:
            x = x + self.cross_attn(self.cross_attn_layernorm(x), g, meta.batch)
        return x + self.mlp(self.post_attention_layernorm(x))


class GlideLlamaForCausalLM(TransformerLMHeadModel):
    def __init__(self, config: Optional[GlideLlamaConfig] = None, **kw) -> None:
        cfg = config or GlideLlamaConfig(**kw)
        super().__init__(cfg)
        self.model.layers = nn.ModuleList([GlideLlamaDecoderLayer(cfg, i) for i in range(cfg.num_hidden_layers)])
        self.apply(self._init_weights)

    def forward(self, input_ids: Optional[torch.Tensor] = None, glide_input: Optional[GlideInput] = None,
                **kw) -> Dict[str, torch.Tensor]:
        for layer in self.model.layers:
            layer.glide_input = glide_input
        try:
            return super().forward(input_ids=input_ids, **kw)
        finally:
            for layer in self.model.layers:
                layer.glide_input = None
