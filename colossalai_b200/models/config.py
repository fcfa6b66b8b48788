"""Typed model configs + the zoo of named presets used by examples, tests and bench.py.

Parity: the model table in reference `examples/language/llama/benchmark.py:33-59` (100m/5b/7b/13b/70b) plus the
HF config fields the reference's policies read (`shardformer/policies/*.py`).
"""
from __future__ import annotations

from dataclasses import asdict, dataclass, field, replace
from typing import Any, Dict, List, Optional

__all__ = ["ModelConfig", "MoEConfig", "MODEL_ZOO", "get_config"]


@dataclass
class MoEConfig:
    num_experts: int = 8
    top_k: int = 2
    moe_intermediate_size: Optional[int] = None  # per-expert FFN width (defaults to intermediate_size)
    n_shared_experts: int = 0                     # DeepSeekMoE shared experts
    first_k_dense_replace: int = 0                # leading dense layers (DeepSeek)
    moe_layer_freq: int = 1
    norm_topk_prob: bool = True
    router_aux_loss_coef: float = 0.02
    router_z_loss_coef: float = 0.0
    scoring_func: str = "softmax"                 # "softmax" | "sigmoid" (DeepSeek-V3)
    n_group: int = 1                              # grouped top-k (DeepSeek-V3)
    topk_group: int = 1
    routed_scaling_factor: float = 1.0
    capacity_factor: float = 0.0                  # 0 = dropless


@dataclass
class ModelConfig:
    model_type: str = "llama"
    vocab_size: int = 32000
    hidden_size: int = 4096
    intermediate_size: int = 11008
    num_hidden_layers: int = 32
    num_attention_heads: int = 32
    num_key_value_heads: Optional[int] = None
    head_dim: Optional[int] = None
    max_position_embeddings: int = 4096
    norm_eps: float = 1e-5
    norm_type: str = "rms"            # "rms" | "layer"
    hidden_act: str = "silu"
    glu: bool = True                  # gated MLP (SwiGLU / GeGLU) vs. plain 2-layer MLP
    attention_bias: bool = False
    attention_out_bias: Optional[bool] = None
    mlp_bias: bool = False
    pos_type: str = "rope"            # "rope" | "learned" | "alibi" | "none"
    rope_theta: float = 10000.0
    rope_scaling: Optional[Dict[str, Any]] = None
    rope_interleaved: bool = False    # GPT-J / ChatGLM pair layout
    partial_rotary_factor: float = 1.0
    qk_norm: bool = False             # Qwen3 / Cohere per-head q/k norm
    parallel_block: bool = False      # attn and mlp read the same normed input (GPT-J, Falcon, Cohere)
    tie_word_embeddings: bool = False
    causal: bool = True
    embed_scale: float = 1.0
    logit_scale: float = 1.0
    type_vocab_size: int = 0          # BERT token types
    post_norm: bool = False           # BERT-style post-LN
    final_norm: bool = True
    embed_norm: bool = False          # Bloom / BERT embedding layernorm
    initializer_range: float = 0.02
    attn_dropout: float = 0.0
    hidden_dropout: float = 0.0
    sliding_window: Optional[int] = None
    lm_head_bias: bool = False        # GPT-J
    norm_head: bool = False           # Baichuan-2 NormHead: L2-normalised LM-head rows
    moe: Optional[MoEConfig] = None
    # multi-head latent attention (DeepSeek-V2 / V3): low-rank q and kv projections, decoupled rope key
    q_lora_rank: Optional[int] = None
    kv_lora_rank: Optional[int] = None
    qk_nope_head_dim: int = 0
    qk_rope_head_dim: int = 0
    v_head_dim: int = 0
    pad_token_id: Optional[int] = None
    bos_token_id: int = 1
    eos_token_id: int = 2

    def __post_init__(self) -> None:
        if self.num_key_value_heads is None:
            self.num_key_value_heads = self.num_attention_heads
        if self.kv_lora_rank is not None:
            # MLA: q / k heads are nope + rope wide (the KV cache stores that width; v is padded up to it)
            self.head_dim = self.qk_nope_head_dim + self.qk_rope_head_dim
            self.num_key_value_heads = self.num_attention_heads
            self.v_head_dim = self.v_head_dim or self.head_dim
        if self.head_dim is None:
            self.head_dim = self.hidden_size // self.num_attention_heads
        if self.attention_out_bias is None:
            self.attention_out_bias = self.attention_bias
        if isinstance(self.moe, dict):
            self.moe = MoEConfig(**self.moe)

    @property
    def q_size(self) -> int:
        return self.num_attention_heads * self.head_dim

    @property
    def kv_size(self) -> int:
        return self.num_key_value_heads * self.head_dim

    @property
    def use_mla(self) -> bool:
        return self.kv_lora_rank is not None

    @property
    def rotary_dim(self) -> int:
        if self.use_mla:
            return self.qk_rope_head_dim
        return int(self.head_dim * self.partial_rotary_factor)

    def num_params(self, include_embeddings: bool = True) -> int:
        h, L = self.hidden_size, self.num_hidden_layers
        attn = h * (self.q_size + 2 * self.kv_size) + self.q_size * h
        if self.moe is not None:
            ei = self.moe.moe_intermediate_size or self.intermediate_size
            per_expert = h * ei * (3 if self.glu else 2)
            mlp = per_expert * (self.moe.num_experts + self.moe.n_shared_experts) + h * self.moe.num_experts
        else:
            mlp = h * self.intermediate_size * (3 if self.glu else 2)
        n = L * (attn + mlp + 2 * h) + h
        if include_embeddings:
            n += self.vocab_size * h * (1 if self.tie_word_embeddings else 2)
        return n

    def flops_per_token(self, seq_len: int, backward: bool = True, checkpoint: bool = False) -> float:
        """Model FLOPs per token (matmul only; causal attention counted at half)."""
        h, L = self.hidden_size, self.num_hidden_layers
        attn_proj = 2 * h * (self.q_size + 2 * self.kv_size) + 2 * self.q_size * h
        if self.moe is not None:
            ei = self.moe.moe_intermediate_size or self.intermediate_size
            act = self.moe.top_k + self.moe.n_shared_experts
            mlp = 2 * h * ei * (3 if self.glu else 2) * act
        else:
            mlp = 2 * h * self.intermediate_size * (3 if self.glu else 2)
        attn_sdp = 4 * seq_len * self.q_size * (0.5 if self.causal else 1.0)
        fwd = L * (attn_proj + mlp + attn_sdp) + 2 * h * self.vocab_size
        mult = (3.0 if backward else 1.0) + (1.0 if (checkpoint and backward) else 0.0)
        return fwd * mult

    def to_dict(self) -> Dict[str, Any]:
        return asdict(self)

    def replace(self, **kw) -> "ModelConfig":
        return replace(self, **kw)


def _llama(**kw) -> ModelConfig:
    return ModelConfig(model_type="llama", **kw)


MODEL_ZOO: Dict[str, ModelConfig] = {
    # ---- reference benchmark table (Llama-2 shapes, examples/language/llama/benchmark.py:33-59)
    "llama-100m": _llama(hidden_size=1024, intermediate_size=2048, num_hidden_layers=4, num_attention_heads=32),
    "llama-5b": _llama(num_key_value_heads=8),
    "llama2-7b": _llama(),
    "llama2-13b": _llama(hidden_size=5120, intermediate_size=13824, num_hidden_layers=40, num_attention_heads=40),
    "llama2-70b": _llama(hidden_size=8192, intermediate_size=28672, num_hidden_layers=80, num_attention_heads=64,
                         num_key_value_heads=8),
    # ---- Llama-3 (BASELINE.json flagship)
    "llama3-8b": _llama(vocab_size=128256, hidden_size=4096, intermediate_size=14336, num_hidden_layers=32,
                        num_attention_heads=32, num_key_value_heads=8, max_position_embeddings=8192,
                        rope_theta=500000.0),
    # Llama-3.2-1B shape (untied head): the largest Llama-3 that trains with fp32 master weights and AdamW moments on
    # one 80 GB GPU without offload
    "llama3.2-1b": _llama(vocab_size=128256, hidden_size=2048, intermediate_size=8192, num_hidden_layers=16,
                          num_attention_heads=32, num_key_value_heads=8, max_position_embeddings=8192,
                          rope_theta=500000.0),
    "llama3-70b": _llama(vocab_size=128256, hidden_size=8192, intermediate_size=28672, num_hidden_layers=80,
                         num_attention_heads=64, num_key_value_heads=8, max_position_embeddings=8192,
                         rope_theta=500000.0),
    "llama-tiny": _llama(vocab_size=512, hidden_size=64, intermediate_size=128, num_hidden_layers=4,
                         num_attention_heads=4, num_key_value_heads=2, max_position_embeddings=256),
    # ---- MoE
    "mixtral-8x7b": ModelConfig(model_type="mixtral", vocab_size=32000, hidden_size=4096, intermediate_size=14336,
                                num_hidden_layers=32, num_attention_heads=32, num_key_value_heads=8,
                                max_position_embeddings=32768, rope_theta=1e6,
                                moe=MoEConfig(num_experts=8, top_k=2)),
    "mixtral-tiny": ModelConfig(model_type="mixtral", vocab_size=512, hidden_size=64, intermediate_size=128,
                                num_hidden_layers=2, num_attention_heads=4, num_key_value_heads=2,
                                max_position_embeddings=256, moe=MoEConfig(num_experts=4, top_k=2)),
    "deepseek-moe-16b": ModelConfig(model_type="deepseek", vocab_size=102400, hidden_size=2048,
                                    intermediate_size=10944, num_hidden_layers=28, num_attention_heads=16,
                                    max_position_embeddings=4096,
                                    moe=MoEConfig(num_experts=64, top_k=6, moe_intermediate_size=1408,
                                                  n_shared_experts=2, first_k_dense_replace=1, norm_topk_prob=False)),
    "deepseek-tiny": ModelConfig(model_type="deepseek", vocab_size=512, hidden_size=64, intermediate_size=128,
                                 num_hidden_layers=2, num_attention_heads=4, max_position_embeddings=256,
                                 moe=MoEConfig(num_experts=8, top_k=2, moe_intermediate_size=32, n_shared_experts=1,
                                               first_k_dense_replace=1, norm_topk_prob=False)),
    # ---- DeepSeek-V3: MLA + sigmoid router with group-limited top-k, shared expert, first 3 layers dense
    "deepseek-v3": ModelConfig(model_type="deepseek_v3", vocab_size=129280, hidden_size=7168, intermediate_size=18432,
                               num_hidden_layers=61, num_attention_heads=128, max_position_embeddings=163840,
                               norm_eps=1e-6, rope_theta=10000.0, rope_interleaved=True, q_lora_rank=1536,
                               kv_lora_rank=512, qk_nope_head_dim=128, qk_rope_head_dim=64, v_head_dim=128,
                               moe=MoEConfig(num_experts=256, top_k=8, moe_intermediate_size=2048, n_shared_experts=1,
                                             first_k_dense_replace=3, norm_topk_prob=True, scoring_func="sigmoid",
                                             n_group=8, topk_group=4, routed_scaling_factor=2.5)),
    "deepseek_v3-tiny": ModelConfig(model_type="deepseek_v3", vocab_size=512, hidden_size=64, intermediate_size=128,
                                    num_hidden_layers=3, num_attention_heads=4, max_position_embeddings=256,
                                    norm_eps=1e-6, rope_interleaved=True, q_lora_rank=24, kv_lora_rank=16,
                                    qk_nope_head_dim=16, qk_rope_head_dim=8, v_head_dim=12,
                                    moe=MoEConfig(num_experts=8, top_k=2, moe_intermediate_size=32, n_shared_experts=1,
                                                  first_k_dense_replace=1, norm_topk_prob=True, scoring_func="sigmoid",
                                                  n_group=4, topk_group=2, routed_scaling_factor=2.5)),
    # ---- GPT-2 family (learned positions, LayerNorm, GELU, tied embeddings)
    "gpt2": ModelConfig(model_type="gpt2", vocab_size=50257, hidden_size=768, intermediate_size=3072,
                        num_hidden_layers=12, num_attention_heads=12, max_position_embeddings=1024, norm_type="layer",
                        hidden_act="gelu_new", glu=False, attention_bias=True, mlp_bias=True, pos_type="learned",
                        tie_word_embeddings=True),
    "gpt2-tiny": ModelConfig(model_type="gpt2", vocab_size=512, hidden_size=64, intermediate_size=256,
                             num_hidden_layers=2, num_attention_heads=4, max_position_embeddings=128,
                             norm_type="layer", hidden_act="gelu_new", glu=False, attention_bias=True, mlp_bias=True,
                             pos_type="learned", tie_word_embeddings=True),
    "mistral-7b": ModelConfig(model_type="mistral", vocab_size=32000, hidden_size=4096, intermediate_size=14336,
                              num_hidden_layers=32, num_attention_heads=32, num_key_value_heads=8,
                              max_position_embeddings=32768, sliding_window=4096),
    "qwen2-7b": ModelConfig(model_type="qwen2", vocab_size=152064, hidden_size=3584, intermediate_size=18944,
                            num_hidden_layers=28, num_attention_heads=28, num_key_value_heads=4,
                            max_position_embeddings=32768, rope_theta=1e6, attention_bias=True,
                            attention_out_bias=False, norm_eps=1e-6),
    "qwen3-8b": ModelConfig(model_type="qwen3", vocab_size=151936, hidden_size=4096, intermediate_size=12288,
                            num_hidden_layers=36, num_attention_heads=32, num_key_value_heads=8, head_dim=128,
                            max_position_embeddings=40960, rope_theta=1e6, qk_norm=True, norm_eps=1e-6),
    "bert-base": ModelConfig(model_type="bert", vocab_size=30522, hidden_size=768, intermediate_size=3072,
                             num_hidden_layers=12, num_attention_heads=12, max_position_embeddings=512,
                             norm_type="layer", hidden_act="gelu", glu=False, attention_bias=True, mlp_bias=True,
                             pos_type="learned", causal=False, type_vocab_size=2, post_norm=True, final_norm=False,
                             embed_norm=True, norm_eps=1e-12),
    "opt-125m": ModelConfig(model_type="opt", vocab_size=50272, hidden_size=768, intermediate_size=3072,
                            num_hidden_layers=12, num_attention_heads=12, max_position_embeddings=2048,
                            norm_type="layer", hidden_act="relu", glu=False, attention_bias=True, mlp_bias=True,
                            pos_type="learned", tie_word_embeddings=True),
    "bloom-560m": ModelConfig(model_type="bloom", vocab_size=250880, hidden_size=1024, intermediate_size=4096,
                              num_hidden_layers=24, num_attention_heads=16, norm_type="layer", hidden_act="gelu_new",
                              glu=False, attention_bias=True, mlp_bias=True, pos_type="alibi", embed_norm=True,
                              tie_word_embeddings=True),
    "falcon-7b": ModelConfig(model_type="falcon", vocab_size=65024, hidden_size=4544, intermediate_size=18176,
                             num_hidden_layers=32, num_attention_heads=71, num_key_value_heads=1, norm_type="layer",
                             hidden_act="gelu", glu=False, parallel_block=True),
    "gptj-6b": ModelConfig(model_type="gptj", vocab_size=50400, hidden_size=4096, intermediate_size=16384,
                           num_hidden_layers=28, num_attention_heads=16, max_position_embeddings=2048,
                           norm_type="layer", hidden_act="gelu_new", glu=False, mlp_bias=True, parallel_block=True,
                           rope_interleaved=True, partial_rotary_factor=0.25, lm_head_bias=True),
    "chatglm2-6b": ModelConfig(model_type="chatglm", vocab_size=65024, hidden_size=4096, intermediate_size=13696,
                               num_hidden_layers=28, num_attention_heads=32, num_key_value_heads=2,
                               max_position_embeddings=32768, attention_bias=True, attention_out_bias=False,
                               rope_interleaved=True, partial_rotary_factor=0.5),
    "baichuan-7b": ModelConfig(model_type="baichuan", vocab_size=64000, hidden_size=4096, intermediate_size=11008,
                               num_hidden_layers=32, num_attention_heads=32, max_position_embeddings=4096,
                               norm_eps=1e-6),
    "baichuan2-13b": ModelConfig(model_type="baichuan", vocab_size=125696, hidden_size=5120, intermediate_size=13696,
                                 num_hidden_layers=40, num_attention_heads=40, max_position_embeddings=4096,
                                 pos_type="alibi", norm_eps=1e-6, norm_head=True),
    "baichuan-tiny": ModelConfig(model_type="baichuan", vocab_size=512, hidden_size=64, intermediate_size=128,
                                 num_hidden_layers=2, num_attention_heads=4, max_position_embeddings=256,
                                 pos_type="alibi", norm_head=True),
    "command-r": ModelConfig(model_type="command", vocab_size=256000, hidden_size=8192, intermediate_size=22528,
                             num_hidden_layers=40, num_attention_heads=64, num_key_value_heads=64, norm_type="layer",
                             parallel_block=True, tie_word_embeddings=True, logit_scale=0.0625, rope_theta=8e6,
                             rope_interleaved=True),
}


def _tiny(preset: str, **kw) -> ModelConfig:
    """Test-size variant of a family preset (2 layers, hidden 64, 4 heads, vocab 512) keeping every family switch."""
    base = dict(vocab_size=512, hidden_size=64, intermediate_size=128, num_hidden_layers=2, num_attention_heads=4,
                num_key_value_heads=2, head_dim=None, max_position_embeddings=256)
    base.update(kw)
    return replace(MODEL_ZOO[preset], **base)


MODEL_ZOO.update({
    "mistral-tiny": _tiny("mistral-7b", sliding_window=None),
    "qwen2-tiny": _tiny("qwen2-7b"),
    "qwen3-tiny": _tiny("qwen3-8b", head_dim=16),
    "opt-tiny": _tiny("opt-125m", num_key_value_heads=4),
    "bloom-tiny": _tiny("bloom-560m", num_key_value_heads=4),
    "falcon-tiny": _tiny("falcon-7b", num_key_value_heads=2),
    "gptj-tiny": _tiny("gptj-6b", num_key_value_heads=4, partial_rotary_factor=0.5),
    "chatglm-tiny": _tiny("chatglm2-6b"),
    "command-tiny": _tiny("command-r", num_key_value_heads=4),
    "bert-tiny": _tiny("bert-base", num_key_value_heads=4),
})


def get_config(name: str, **overrides) -> ModelConfig:
    if name not in MODEL_ZOO:
        raise KeyError(f"unknown model preset {name!r}; available: {sorted(MODEL_ZOO)}")
    cfg = MODEL_ZOO[name]
    if not overrides:
        return replace(cfg)
    # derived fields must be re-derived when the shape changes
    if ("hidden_size" in overrides or "num_attention_heads" in overrides) and "head_dim" not in overrides \
            and cfg.head_dim == cfg.hidden_size // cfg.num_attention_heads:
        overrides["head_dim"] = None
    return replace(cfg, **overrides)
