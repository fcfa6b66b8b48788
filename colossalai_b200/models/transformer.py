"""Generic decoder/encoder transformer used by every model family in the zoo.

Design (SURVEY §7.1): we own small explicit model definitions whose forward is parallel-aware instead of
monkey-patching HuggingFace modules.  A freshly constructed model is an ordinary single-device module built from
`nn.Linear` / `nn.Embedding`; `ShardFormer.optimize(model, policy)` swaps those for TP/SP layers (one fused QKV
GEMM, one fused gate|up GEMM per block) and attaches a `ShardConfig`; the forward reads it to route sequence-
parallel layouts and pipeline stages.  Activations are token-major `[T, H]` with `T = batch * seq`.

Parity: replaces the reference's per-model forwards in `colossalai/shardformer/modeling/*.py` (llama.py:43-600 etc.:
pipeline-stage-aware model / LM-head forwards, flash / ring / Ulysses attention forwards, SP split/gather,
dist-CE loss).
"""
from __future__ import annotations

import math
from dataclasses import dataclass
from typing import Any, Dict, List, Optional, Tuple

import torch
import torch.nn as nn
import torch.nn.functional as F
from torch.utils.checkpoint import checkpoint as torch_checkpoint

from .. import ops
from ..parallel import comm
from ..shardformer.layer._operation import (
    all_to_all_comm,
    gather_forward_split_backward,
    gather_sp_output,
    split_batch_zigzag,
    split_forward_gather_backward,
    zigzag_positions,
)
from ..shardformer.layer.attn import RingAttention
from ..shardformer.layer.loss import dist_cross_entropy
from ..shardformer.layer.normalization import FusedLayerNorm, FusedRMSNorm
from .config import ModelConfig

__all__ = ["SeqMeta", "Attention", "MLP", "DecoderLayer", "TransformerModel", "TransformerLMHeadModel",
           "build_norm"]


@dataclass
class SeqMeta:
    """Per-forward sequence metadata shared by all layers."""

    batch: int
    seqlen: int                      # full (global) sequence length of each batch element
    positions: torch.Tensor          # [T_attn] int64 position of every token seen by attention/rope
    cu_seqlens: Optional[torch.Tensor] = None
    max_seqlen: Optional[int] = None
    attn_mask: Optional[torch.Tensor] = None   # [B, S] padding mask (1 = keep) for encoder models
    local_seqlen: Optional[int] = None          # per-sequence tokens held by this rank under a2a / ring_attn


def _use_fused_a2a(x: torch.Tensor, sp_group) -> bool:
    """Ulysses all-to-all through the sm_90a pull kernel: CUDA tensors under the `fused` comm backend."""
    from ..shardformer.layer._operation import get_comm_backend

    if not x.is_cuda or get_comm_backend() != "fused" or comm.group_size(sp_group) == 1:
        return False
    from ..parallel import fused

    return fused.available(sp_group)


def build_norm(cfg: ModelConfig, hidden: Optional[int] = None) -> nn.Module:
    h = hidden or cfg.hidden_size
    if cfg.norm_type == "rms":
        return FusedRMSNorm(h, eps=cfg.norm_eps)
    return FusedLayerNorm(h, eps=cfg.norm_eps)


def _sc(module: nn.Module):
    return getattr(module, "shard_config", None)


def _alibi_slopes(n_heads: int) -> torch.Tensor:
    def pow2(n):
        start = 2 ** (-(2 ** -(math.log2(n) - 3)))
        return [start * (start ** i) for i in range(n)]

    if math.log2(n_heads).is_integer():
        return torch.tensor(pow2(n_heads))
    c = 2 ** math.floor(math.log2(n_heads))
    return torch.tensor(pow2(c) + pow2(2 * c)[0::2][: n_heads - c])


class Attention(nn.Module):
    def __init__(self, cfg: ModelConfig, layer_idx: int = 0) -> None:
        super().__init__()
        self.cfg, self.layer_idx = cfg, layer_idx
        self.num_heads, self.num_kv_heads, self.head_dim = cfg.num_attention_heads, cfg.num_key_value_heads, cfg.head_dim
        self.qkv_proj = nn.Linear(cfg.hidden_size, cfg.q_size + 2 * cfg.kv_size, bias=cfg.attention_bias)
        self.o_proj = nn.Linear(cfg.q_size, cfg.hidden_size, bias=cfg.attention_out_bias)
        if cfg.qk_norm:
            self.q_norm = FusedRMSNorm(cfg.head_dim, eps=cfg.norm_eps)
            self.k_norm = FusedRMSNorm(cfg.head_dim, eps=cfg.norm_eps)
        self.shard_config = None
        self.scale = 1.0 / math.sqrt(cfg.head_dim)

    def forward(self, x: torch.Tensor, meta: SeqMeta, rope: Optional[Tuple[torch.Tensor, torch.Tensor]] = None,
                kv_cache=None) -> torch.Tensor:
        cfg, sc = self.cfg, self.shard_config
        D = self.head_dim
        qkv = self.qkv_proj(x)                                  # [T*, (hq + 2 hkv) * D] local heads
        hq = self.num_heads
        hkv = self.num_kv_heads
        sp_mode = sc.sp_mode if sc is not None else None
        sp_group = sc.sp_group if sc is not None else None
        if sp_mode == "all_to_all" and comm.group_size(sp_group) > 1:
            # Ulysses: [B*S/sp, heads*D] -> [B*S, (heads/sp)*D]: scatter heads, gather sequence
            sp = comm.group_size(sp_group)
            B, Sl = meta.batch, qkv.shape[0] // meta.batch
            fused_qkv = None
            if _use_fused_a2a(qkv, sp_group):
                # ONE pull kernel over peer memory moves q, k and v together (no chunk / stack / cat copies)
                from ..parallel import fused

                fused_qkv = fused.ulysses_all_to_all(qkv, sp_group, True, B, Sl,
                                                     [hq // sp * D, hkv // sp * D, hkv // sp * D])
            if fused_qkv is not None:
                hq, hkv = hq // sp, hkv // sp
                qkv = fused_qkv
            else:
                q, k, v = qkv.split([hq * D, hkv * D, hkv * D], dim=-1)
                def a2a(t, nh):
                    t = t.reshape(B, Sl, nh, D)
                    t = all_to_all_comm(t, sp_group, scatter_dim=2, gather_dim=1)
                    return t.reshape(B * Sl * sp, (nh // sp) * D)
                hq, hkv = hq // sp, hkv // sp
                qkv = torch.cat([a2a(q, hq * sp), a2a(k, hkv * sp), a2a(v, hkv * sp)], dim=-1)
        T = qkv.shape[0]
        if cfg.qk_norm:
            q, k, v = qkv.split([hq * D, hkv * D, hkv * D], dim=-1)
            q = self._head_norm(self.q_norm, q.reshape(T, hq, D)).reshape(T, hq * D)
            k = self._head_norm(self.k_norm, k.reshape(T, hkv, D)).reshape(T, hkv * D)
            qkv = torch.cat([q, k, v], dim=-1)
        if rope is not None:
            qkv = ops.rope_qkv(qkv, meta.positions, rope[0], rope[1], hq, hkv, D, rot_dim=cfg.rotary_dim,
                               interleaved=cfg.rope_interleaved)
        q, k, v = qkv.split([hq * D, hkv * D, hkv * D], dim=-1)
        q, k, v = q.reshape(T, hq, D), k.reshape(T, hkv, D), v.reshape(T, hkv, D)
        if kv_cache is not None:
            slopes = self._local_alibi_slopes(q.device) if cfg.pos_type == "alibi" else None
            extra = {} if slopes is None else {"alibi_slopes": slopes}
            if cfg.sliding_window:
                extra["sliding_window"] = cfg.sliding_window
            o = kv_cache.attend(self.layer_idx, q, k, v, meta, self.scale, **extra)
        elif sp_mode == "ring_attn" and comm.group_size(sp_group) > 1:
            o = RingAttention.attention(q, k, v, sp_group, batch=meta.batch, scale=self.scale)
        else:
            mask = None
            windowed = bool(cfg.sliding_window) and (meta.max_seqlen or T // meta.batch) > cfg.sliding_window
            if windowed and meta.cu_seqlens is not None:
                raise NotImplementedError("sliding-window attention over packed (varlen) batches longer than the "
                                          "window is not supported; pad to equal lengths")
            if cfg.pos_type == "alibi" or meta.attn_mask is not None or windowed:
                mask = self._build_mask(meta, T, hq, q.device, q.dtype)
            o = ops.attention(q, k, v, batch=meta.batch, causal=cfg.causal and mask is None, scale=self.scale,
                              cu_seqlens_q=meta.cu_seqlens, max_seqlen=meta.max_seqlen, attn_mask=mask,
                              dropout_p=cfg.attn_dropout if self.training else 0.0)
        o = o.reshape(T, hq * D)
        if sp_mode == "all_to_all" and comm.group_size(sp_group) > 1:
            sp = comm.group_size(sp_group)
            B, S = meta.batch, T // meta.batch
            fused_o = None
            if _use_fused_a2a(o, sp_group):
                from ..parallel import fused

                fused_o = fused.ulysses_all_to_all(o, sp_group, False, B, S // sp, [hq * D])
            if fused_o is not None:
                o = fused_o
            else:
                o = all_to_all_comm(o.reshape(B, S, hq, D), sp_group, scatter_dim=1, gather_dim=2)
                o = o.reshape(B * (S // sp), hq * sp * D)
        return self.o_proj(o)

    def _head_norm(self, norm: nn.Module, t: torch.Tensor) -> torch.Tensor:
        """Per-head q/k RMSNorm.  Its [head_dim] weight is replicated over TP while every rank only sees its own
        heads, so the weight gradient is a partial sum: identity forward / all-reduce backward over the TP group."""
        sc = self.shard_config
        w = norm.weight
        if sc is not None and sc.enable_tensor_parallelism and sc.tensor_parallel_size > 1:
            from ..shardformer.layer._operation import reduce_backward

            w = reduce_backward(w, sc.tp_group)
        if w.dtype != t.dtype:
            w = w.to(t.dtype)
        return ops.rms_norm(t, w, norm.eps, None)

    def _local_alibi_slopes(self, device) -> torch.Tensor:
        sc = self.shard_config
        slopes = _alibi_slopes(self.cfg.num_attention_heads).to(device=device, dtype=torch.float32)
        if sc is not None and sc.enable_tensor_parallelism and sc.tensor_parallel_size > 1:
            slopes = slopes.chunk(sc.tensor_parallel_size)[comm.group_rank(sc.tp_group)]
        return slopes.contiguous()

    def _build_mask(self, meta: SeqMeta, T: int, hq: int, device, dtype) -> torch.Tensor:
        """Additive/boolean mask [B, H, S, S] for ALiBi and padded encoder inputs (reference path only)."""
        B, S = meta.batch, T // meta.batch
        keep = torch.ones(B, 1, S, S, dtype=torch.bool, device=device)
        if self.cfg.causal:
            keep = keep & torch.ones(S, S, dtype=torch.bool, device=device).tril()
        if meta.attn_mask is not None:
            keep = keep & meta.attn_mask.bool()[:, None, None, :]
        if self.cfg.sliding_window and S > self.cfg.sliding_window:       # Mistral: the last `window` keys only
            idx = torch.arange(S, device=device)
            keep = keep & ((idx[None, :] - idx[:, None]) > -self.cfg.sliding_window)
        if self.cfg.pos_type != "alibi":
            return keep
        sc = self.shard_config
        slopes = _alibi_slopes(self.cfg.num_attention_heads).to(device)
        if sc is not None and sc.tensor_parallel_size > 1:
            slopes = slopes.chunk(sc.tensor_parallel_size)[comm.group_rank(sc.tp_group)]
        pos = torch.arange(S, device=device)
        bias = (pos[None, :] - pos[:, None]).clamp(max=0).float()[None, None] * slopes[None, :, None, None]
        bias = bias.masked_fill(~keep, float("-inf"))
        return bias.to(dtype)


class MLAttention(nn.Module):
    """Multi-head latent attention (DeepSeek-V2 / V3): queries through a low-rank bottleneck, keys / values rebuilt
    from one shared `kv_lora_rank` latent per token plus a single rotary key shared by all heads.

    Parity: reference `shardformer/policies/deepseek_v3.py` drives HF's `DeepseekV3Attention`
    (transformers `modeling_deepseek_v3.py`), whose parameter names are kept so checkpoints map one to one.  Under
    tensor parallelism the up-projections (`q_b_proj`, `kv_b_proj`) are column-split by heads and `o_proj` is
    row-split; the small down-projections and their norms stay replicated.  With a KV cache the value heads are
    zero-padded to the key width so one paged layout serves both."""

    def __init__(self, cfg: ModelConfig, layer_idx: int = 0) -> None:
        super().__init__()
        self.cfg, self.layer_idx = cfg, layer_idx
        self.num_heads = self.num_kv_heads = cfg.num_attention_heads
        self.qk_nope, self.qk_rope, self.v_dim = cfg.qk_nope_head_dim, cfg.qk_rope_head_dim, cfg.v_head_dim
        self.head_dim = self.qk_nope + self.qk_rope
        H, hid = cfg.num_attention_heads, cfg.hidden_size
        if cfg.q_lora_rank is None:
            self.q_proj = nn.Linear(hid, H * self.head_dim, bias=False)
        else:
            self.q_a_proj = nn.Linear(hid, cfg.q_lora_rank, bias=cfg.attention_bias)
            self.q_a_layernorm = FusedRMSNorm(cfg.q_lora_rank, eps=cfg.norm_eps)
            self.q_b_proj = nn.Linear(cfg.q_lora_rank, H * self.head_dim, bias=False)
        self.kv_a_proj_with_mqa = nn.Linear(hid, cfg.kv_lora_rank + self.qk_rope, bias=cfg.attention_bias)
        self.kv_a_layernorm = FusedRMSNorm(cfg.kv_lora_rank, eps=cfg.norm_eps)
        self.kv_b_proj = nn.Linear(cfg.kv_lora_rank, H * (self.qk_nope + self.v_dim), bias=False)
        self.o_proj = nn.Linear(H * self.v_dim, hid, bias=cfg.attention_bias)
        self.shard_config = None
        self.scale = 1.0 / math.sqrt(self.head_dim)
        rs = cfg.rope_scaling or {}
        if rs.get("rope_type", rs.get("type", "default")) == "yarn" and rs.get("mscale_all_dim"):
            f = rs.get("factor", 1.0)
            m = 1.0 if f <= 1 else 0.1 * rs["mscale_all_dim"] * math.log(f) + 1.0
            self.scale = self.scale * m * m

    def _replicated_in_tp(self, t: torch.Tensor) -> torch.Tensor:
        """The shared rotary key comes from a replicated projection but feeds this rank's heads only: its gradient is a
        partial sum over the TP group (identity forward / all-reduce backward).  The latents entering `q_b_proj` /
        `kv_b_proj` need nothing here, the column-parallel linears already all-reduce their input gradient."""
        sc = self.shard_config
        if sc is not None and sc.enable_tensor_parallelism and sc.tensor_parallel_size > 1 and t.requires_grad:
            from ..shardformer.layer._operation import reduce_backward

            return reduce_backward(t, sc.tp_group)
        return t

    def forward(self, x: torch.Tensor, meta: SeqMeta, rope: Optional[Tuple[torch.Tensor, torch.Tensor]] = None,
                kv_cache=None) -> torch.Tensor:
        cfg, sc = self.cfg, self.shard_config
        if sc is not None and sc.sp_mode in ("all_to_all", "ring_attn") and comm.group_size(sc.sp_group) > 1:
            raise NotImplementedError("multi-head latent attention supports tensor / pipeline / expert parallelism "
                                      "and Megatron-style sequence parallelism is not wired for it yet")
        T, Hl = x.shape[0], self.num_heads
        if cfg.q_lora_rank is None:
            q = self.q_proj(x)
        else:
            q = self.q_b_proj(self.q_a_layernorm(self.q_a_proj(x)))
        q = q.view(T, Hl, self.head_dim)
        ckv = self.kv_a_proj_with_mqa(x)
        c, k_pe = ckv.split([cfg.kv_lora_rank, self.qk_rope], dim=-1)
        kv = self.kv_b_proj(self.kv_a_layernorm(c)).view(T, Hl, self.qk_nope + self.v_dim)
        k_nope, v = kv.split([self.qk_nope, self.v_dim], dim=-1)
        q_nope, q_pe = q.split([self.qk_nope, self.qk_rope], dim=-1)
        k_pe = self._replicated_in_tp(k_pe).reshape(T, 1, self.qk_rope)
        if rope is not None:
            q_pe = ops.rope_ref(q_pe, meta.positions, rope[0], rope[1], self.qk_rope, cfg.rope_interleaved)
            k_pe = ops.rope_ref(k_pe, meta.positions, rope[0], rope[1], self.qk_rope, cfg.rope_interleaved)
        q = torch.cat([q_nope, q_pe], dim=-1)
        k = torch.cat([k_nope, k_pe.expand(T, Hl, self.qk_rope)], dim=-1)
        if kv_cache is not None:
            vp = F.pad(v, (0, self.head_dim - self.v_dim)) if self.v_dim < self.head_dim else v
            o = kv_cache.attend(self.layer_idx, q.contiguous(), k.contiguous(), vp.contiguous(), meta, self.scale)
            o = o.reshape(T, Hl, -1)[..., : self.v_dim]
        else:
            o = ops.attention(q, k, v.contiguous(), batch=meta.batch, causal=cfg.causal, scale=self.scale,
                              cu_seqlens_q=meta.cu_seqlens, max_seqlen=meta.max_seqlen,
                              dropout_p=cfg.attn_dropout if self.training else 0.0)
        return self.o_proj(o.reshape(T, Hl * self.v_dim))


class MLP(nn.Module):
    def __init__(self, cfg: ModelConfig, intermediate_size: Optional[int] = None) -> None:
        super().__init__()
        self.cfg = cfg
        inter = intermediate_size or cfg.intermediate_size
        self.intermediate_size = inter
        if cfg.glu:
            self.gate_up_proj = nn.Linear(cfg.hidden_size, 2 * inter, bias=cfg.mlp_bias)
        else:
            self.up_proj = nn.Linear(cfg.hidden_size, inter, bias=cfg.mlp_bias)
        self.down_proj = nn.Linear(inter, cfg.hidden_size, bias=cfg.mlp_bias)
        self.shard_config = None

    def forward(self, x: torch.Tensor) -> torch.Tensor:
        if self.cfg.glu:
            h = ops.glu(self.gate_up_proj(x), self.cfg.hidden_act)
        else:
            up = self.up_proj
            if self.cfg.hidden_act in ("gelu", "gelu_new", "gelu_tanh", "gelu_pytorch_tanh") and x.is_cuda \
                    and getattr(up, "skip_bias_add", False):
                y, b = up(x)
                h = ops.bias_act(y, b, self.cfg.hidden_act)
            else:
                h = ops.get_activation(self.cfg.hidden_act)(up(x))
        return self.down_proj(h)


class DecoderLayer(nn.Module):
    def __init__(self, cfg: ModelConfig, layer_idx: int) -> None:
        super().__init__()
        self.cfg, self.layer_idx = cfg, layer_idx
        self.input_layernorm = build_norm(cfg)
        self.self_attn = MLAttention(cfg, layer_idx) if cfg.use_mla else Attention(cfg, layer_idx)
        if not cfg.parallel_block:
            self.post_attention_layernorm = build_norm(cfg)
        moe = cfg.moe
        if moe is not None and layer_idx >= moe.first_k_dense_replace and (layer_idx % moe.moe_layer_freq == 0):
            from .moe import SparseMoE

            self.mlp = SparseMoE(cfg)
        else:
            self.mlp = MLP(cfg)
        self.shard_config = None

    def forward(self, x: torch.Tensor, meta: SeqMeta, rope=None, kv_cache=None) -> torch.Tensor:
        cfg = self.cfg
        if cfg.post_norm:   # BERT: x = LN(x + attn(x)); x = LN(x + mlp(x))
            x = self.input_layernorm(x + self.self_attn(x, meta, rope, kv_cache))
            return self.post_attention_layernorm(x + self.mlp(x))
        if cfg.parallel_block:
            h = self.input_layernorm(x)
            return x + self.self_attn(h, meta, rope, kv_cache) + self.mlp(h)
        h = self.input_layernorm(x)
        a = self.self_attn(h, meta, rope, kv_cache)
        if cfg.norm_type == "rms":
            h, x = self.post_attention_layernorm(a, residual=x)     # fused residual-add + norm
        else:
            x = x + a
            h = self.post_attention_layernorm(x)
        return x + self.mlp(h)


class TransformerModel(nn.Module):
    """Embedding + layers + final norm.  Pipeline-stage aware: under PP the model keeps only its own layers
    (`held_layers`), the first stage owns the embedding and the last stage the final norm."""

    def __init__(self, cfg: ModelConfig) -> None:
        super().__init__()
        self.cfg = cfg
        self.embed_tokens = nn.Embedding(cfg.vocab_size, cfg.hidden_size, padding_idx=cfg.pad_token_id)
        if cfg.pos_type == "learned":
            self.embed_positions = nn.Embedding(cfg.max_position_embeddings, cfg.hidden_size)
        if cfg.type_vocab_size > 0:
            self.embed_token_types = nn.Embedding(cfg.type_vocab_size, cfg.hidden_size)
        if cfg.embed_norm:
            self.embed_layernorm = build_norm(cfg)
        self.layers = nn.ModuleList([DecoderLayer(cfg, i) for i in range(cfg.num_hidden_layers)])
        if cfg.final_norm:
            self.norm = build_norm(cfg)
        self.shard_config = None
        self.gradient_checkpointing = False
        self._rope_cache: Dict[Tuple, Tuple[torch.Tensor, torch.Tensor]] = {}

    # ------------------------------------------------------------------ helpers
    def rope_cache(self, device, min_len: int = 0) -> Optional[Tuple[torch.Tensor, torch.Tensor]]:
        """cos / sin tables [positions, rotary_dim / 2].  Sized by the config, but never shorter than the sequence in
        flight (`min_len`, rounded up to a power of two): a 128k-token context on a checkpoint configured for 8k must
        not index past the table."""
        cfg = self.cfg
        if cfg.pos_type != "rope":
            return None
        n_pos = cfg.max_position_embeddings
        if min_len > n_pos:
            n_pos = 1 << (min_len - 1).bit_length()
        key = (str(device), n_pos)
        if key not in self._rope_cache:
            llama3 = cfg.rope_scaling if (cfg.rope_scaling and cfg.rope_scaling.get("rope_type") == "llama3") else None
            factor = 1.0
            if cfg.rope_scaling and cfg.rope_scaling.get("rope_type", cfg.rope_scaling.get("type")) == "linear":
                factor = cfg.rope_scaling.get("factor", 1.0)
            self._rope_cache[key] = ops.build_rope_cache(n_pos, cfg.rotary_dim, cfg.rope_theta,
                                                         device=device, scaling_factor=factor, llama3_scaling=llama3)
        return self._rope_cache[key]

    def layer_range(self) -> Tuple[int, int]:
        sc = self.shard_config
        sm = sc.pipeline_stage_manager if sc is not None else None
        if sm is None:
            return 0, len(self.layers)
        return sm.get_stage_index(sm.distribute_layers(len(self.layers)))

    def _num_ckpt_layers(self, n_local: int) -> int:
        sc = self.shard_config
        gcc = sc.gradient_checkpoint_config if sc is not None else None
        if gcc is not None:
            sm = sc.pipeline_stage_manager
            if hasattr(gcc, "num_ckpt_layers_per_stage") and sm is not None:
                return gcc.get_num_ckpt_layers(sm.stage, sm.num_stages, n_local)
            return gcc.get_num_ckpt_layers(n_local)
        return n_local if self.gradient_checkpointing else 0

    def gradient_checkpointing_enable(self, *a, **k) -> None:
        self.gradient_checkpointing = True

    # ------------------------------------------------------------------ forward
    def embed(self, input_ids: Optional[torch.Tensor], meta: SeqMeta, positions_local: torch.Tensor,
              token_type_ids: Optional[torch.Tensor] = None,
              inputs_embeds: Optional[torch.Tensor] = None) -> torch.Tensor:
        cfg = self.cfg
        x = inputs_embeds if inputs_embeds is not None else self.embed_tokens(input_ids)
        if cfg.embed_scale != 1.0:
            x = x * cfg.embed_scale
        if cfg.pos_type == "learned":
            x = x + self.embed_positions(positions_local)
        if cfg.type_vocab_size > 0:
            tt = token_type_ids if token_type_ids is not None else positions_local.new_zeros(x.shape[0])
            x = x + self.embed_token_types(tt)
        if cfg.embed_norm:
            x = self.embed_layernorm(x)
        if cfg.hidden_dropout > 0 and self.training:
            x = F.dropout(x, cfg.hidden_dropout)
        return x

    def forward(self, input_ids: Optional[torch.Tensor] = None, hidden_states: Optional[torch.Tensor] = None,
                attention_mask: Optional[torch.Tensor] = None, position_ids: Optional[torch.Tensor] = None,
                token_type_ids: Optional[torch.Tensor] = None, batch: Optional[int] = None,
                seqlen: Optional[int] = None, kv_cache=None, meta: Optional[SeqMeta] = None,
                inputs_embeds: Optional[torch.Tensor] = None) -> torch.Tensor:
        """`input_ids` [B, S] on the first stage (or `hidden_states` [T_local, H] from the previous stage, or
        `inputs_embeds` [B, S, H] replacing the token-embedding lookup — multimodal prefixes).
        Returns token-major hidden states in the stage's activation layout."""
        cfg, sc = self.cfg, self.shard_config
        sm = sc.pipeline_stage_manager if sc is not None else None
        first = sm is None or sm.is_first_stage()
        last = sm is None or sm.is_last_stage()
        sp_mode = sc.sp_mode if sc is not None else None
        sp_group = sc.sp_group if sc is not None else None
        sp = sc.sequence_parallel_size if sp_mode else 1
        if input_ids is not None:
            B, S = input_ids.shape
            device = input_ids.device
        elif inputs_embeds is not None:
            B, S = inputs_embeds.shape[:2]
            device = inputs_embeds.device
        else:
            assert batch is not None and seqlen is not None, "later PP stages need batch/seqlen"
            B, S, device = batch, seqlen, hidden_states.device
        if sp > 1:
            # fail here with a sentence, not inside a collective with mismatched shard sizes
            if sp_mode == "ring_attn":
                assert S % (2 * sp) == 0, (f"ring attention splits every sequence into 2 x sp = {2 * sp} zigzag blocks: "
                                           f"pad the sequence length {S} to a multiple of {2 * sp}")
            elif sp_mode == "all_to_all":
                assert S % sp == 0, (f"all_to_all sequence parallelism shards the sequence over {sp} ranks: pad the "
                                     f"sequence length {S} to a multiple of {sp}")
            elif sp_mode in ("split_gather", "ring"):
                assert (B * S) % sp == 0, (f"{sp_mode} sequence parallelism shards the {B} x {S} tokens over {sp} ranks: "
                                           f"pad batch x sequence to a multiple of {sp}")
        if meta is None:
            # positions seen by rope/attention
            if position_ids is not None:
                pos_full = position_ids.reshape(-1).long()
            else:
                pos_full = torch.arange(S, device=device).repeat(B)
            if sp_mode == "ring_attn" and sp > 1:
                zz = zigzag_positions(S, sp, comm.group_rank(sp_group), device)
                positions = zz.repeat(B)
                local_S = S // sp
            elif sp_mode == "all_to_all" and sp > 1:
                positions = pos_full      # attention runs on the full sequence after the all-to-all
                local_S = S // sp
            else:
                positions = pos_full
                local_S = S
            meta = SeqMeta(batch=B, seqlen=S, positions=positions, attn_mask=attention_mask, local_seqlen=local_S)
        if first and inputs_embeds is not None:
            assert not (sp_mode in ("ring_attn", "all_to_all") and sp > 1), \
                "inputs_embeds is not supported together with ring_attn / all_to_all sequence parallelism"
            x = self.embed(None, meta, meta.positions, None if token_type_ids is None else token_type_ids.reshape(-1),
                           inputs_embeds=inputs_embeds.reshape(B * S, -1))
            if sp_mode in ("split_gather", "ring") and sp > 1:
                x = split_forward_gather_backward(x, 0, sp_group)
        elif first:
            ids = input_ids
            tt = token_type_ids
            if sp_mode == "ring_attn" and sp > 1:
                ids = split_batch_zigzag(ids, sp_group, seq_dim=1)
                pos_local = zigzag_positions(S, sp, comm.group_rank(sp_group), device).repeat(B)
            elif sp_mode == "all_to_all" and sp > 1:
                r = comm.group_rank(sp_group)
                ids = ids.chunk(sp, dim=1)[r]
                pos_local = torch.arange(r * (S // sp), (r + 1) * (S // sp), device=device).repeat(B)
            else:
                pos_local = meta.positions
            x = self.embed(ids.reshape(-1), meta, pos_local, None if tt is None else tt.reshape(-1))
            if sp_mode in ("split_gather", "ring") and sp > 1:
                x = split_forward_gather_backward(x, 0, sp_group)
            elif sp_mode == "all_to_all" and sp > 1:
                # loss is averaged over the dp x sp group -> scale grads like the reference (modeling/llama.py:165)
                pass
        else:
            x = hidden_states
        rope = self.rope_cache(device, min_len=int(getattr(meta, "seqlen", 0) or 0))
        start, end = self.layer_range()
        n_ckpt = self._num_ckpt_layers(end - start) if self.training else 0
        for i in range(start, end):
            layer = self.layers[i]
            if i - start < n_ckpt:
                x = torch_checkpoint(layer, x, meta, rope, kv_cache, use_reentrant=False)
            else:
                x = layer(x, meta, rope, kv_cache)
        if last and cfg.final_norm:
            x = self.norm(x)
        return x


class TransformerLMHeadModel(nn.Module):
    """Causal (or masked) LM: backbone + LM head + (distributed) cross entropy."""

    def __init__(self, cfg: ModelConfig) -> None:
        super().__init__()
        self.cfg = cfg
        self.config = cfg
        self.model = TransformerModel(cfg)
        self.lm_head = nn.Linear(cfg.hidden_size, cfg.vocab_size, bias=cfg.lm_head_bias)
        if cfg.tie_word_embeddings:
            self.lm_head.weight = self.model.embed_tokens.weight
        self.shard_config = None
        self.apply(self._init_weights)

    def _init_weights(self, m: nn.Module) -> None:
        std = self.cfg.initializer_range
        # (on the meta device these calls only land in the lazy-init log: `materialize(reproduce_eager=True)` replays them)
        if isinstance(m, nn.Linear):
            nn.init.normal_(m.weight, mean=0.0, std=std)
            if m.bias is not None:
                nn.init.zeros_(m.bias)
        elif isinstance(m, nn.Embedding):
            nn.init.normal_(m.weight, mean=0.0, std=std)
            if m.padding_idx is not None and m.weight.device.type != "meta":
                with torch.no_grad():
                    m.weight[m.padding_idx].zero_()

    def gradient_checkpointing_enable(self, *a, **k) -> None:
        self.model.gradient_checkpointing = True

    def get_input_embeddings(self):
        return self.model.embed_tokens

    def get_output_embeddings(self):
        return self.lm_head

    def forward(self, input_ids: Optional[torch.Tensor] = None, labels: Optional[torch.Tensor] = None,
                attention_mask: Optional[torch.Tensor] = None, position_ids: Optional[torch.Tensor] = None,
                hidden_states: Optional[torch.Tensor] = None, token_type_ids: Optional[torch.Tensor] = None,
                batch: Optional[int] = None, seqlen: Optional[int] = None, return_logits: bool = True,
                kv_cache=None, meta=None, inputs_embeds: Optional[torch.Tensor] = None,
                **unused) -> Dict[str, torch.Tensor]:
        cfg, sc = self.cfg, self.shard_config
        sm = sc.pipeline_stage_manager if sc is not None else None
        if input_ids is not None:
            B, S = input_ids.shape
        elif inputs_embeds is not None:
            B, S = inputs_embeds.shape[:2]
        else:
            B, S = batch, seqlen
        h = self.model(input_ids=input_ids, hidden_states=hidden_states, attention_mask=attention_mask,
                       position_ids=position_ids, token_type_ids=token_type_ids, batch=B, seqlen=S,
                       kv_cache=kv_cache, meta=meta, inputs_embeds=inputs_embeds)
        if sm is not None and not sm.is_last_stage():
            return {"hidden_states": h}
        sp_mode = sc.sp_mode if sc is not None else None
        sp_group = sc.sp_group if sc is not None else None
        # split_gather/ring: the LM head (a col-parallel linear in SP mode) gathers the tokens itself.
        # all_to_all / ring_attn: logits stay sequence-sharded when the loss is computed in parallel.
        keep_sp_sharded = sp_mode in ("all_to_all", "ring_attn") and labels is not None and \
            (sc is not None and sc.parallel_output)
        if sp_mode in ("all_to_all", "ring_attn") and not keep_sp_sharded and comm.group_size(sp_group) > 1:
            Sl = h.shape[0] // B
            h = gather_sp_output(h.view(B, Sl, -1), sp_group, sp_mode, sp_dim=1).reshape(B * S, -1)
        if cfg.norm_head:
            # Baichuan-2 NormHead: L2-normalised rows.  Rows are vocabulary entries, so the normalisation is local to
            # a vocab-parallel shard too; run the (possibly parallel) head with the normalised weight swapped in.
            w = F.normalize(self.lm_head.weight, dim=-1)
            logits = F.linear(h, w) if isinstance(self.lm_head, nn.Linear) else \
                torch.func.functional_call(self.lm_head, {"weight": w}, (h,))
        else:
            logits = self.lm_head(h)
        if cfg.logit_scale != 1.0:
            logits = logits * cfg.logit_scale
        out: Dict[str, torch.Tensor] = {}
        if labels is not None:
            class _NoShard:
                enable_tensor_parallelism = False
                enable_sequence_parallelism = False
                parallel_output = False
                tensor_parallel_process_group = None
                sequence_parallel_process_group = None
                sequence_parallelism_mode = None

            out["loss"] = dist_cross_entropy(labels, logits, sc if sc is not None else _NoShard, cfg.vocab_size,
                                             dtype=torch.float32, shift=cfg.causal)
        if return_logits:
            V = cfg.vocab_size
            out["logits"] = logits if logits.shape[-1] == V or (sc is not None and sc.parallel_output and
                                                                sc.tensor_parallel_size > 1) else logits[..., :V]
        return out
