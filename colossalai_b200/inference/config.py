"""Inference configuration.  Parity: reference `colossalai/inference/config.py:53-418` (`InferenceConfig`,
`InputMetaData`, `ModelShardInferenceConfig`, `DiffusionGenerationConfig`, rpc (de)serialisation)."""
from __future__ import annotations

from dataclasses import dataclass, field, fields
from typing import Any, Dict, List, Optional, Union

import torch

__all__ = ["InferenceConfig", "InputMetaData", "ModelShardInferenceConfig", "DiffusionGenerationConfig",
           "GenerationConfig", "RPC_PARAM"]

_DTYPE_MAPPING = {"fp16": torch.float16, "bf16": torch.bfloat16, "fp32": torch.float32}
_ALLOWED_DTYPES = [torch.float16, torch.bfloat16, torch.float32]
_DEFAULT_PROMPT_TEMPLATES = {
    "llama": "[INST] <<SYS>>\nYou are a helpful, respectful and honest assistant.\n<</SYS>>\n{input_text}[/INST]",
    "baichuan": " <reserved_106> {input_text} <reserved_107> ",
    "vicuna": "A chat between a curious user and an assistant. USER: {input_text}\nASSISTANT: ",
}


class RPC_PARAM:
    """Mixin: (de)serialise a dataclass for the RPC control plane."""

    def to_rpc_param(self) -> dict:
        out = {}
        for f in fields(self):
            v = getattr(self, f.name)
            if isinstance(v, torch.dtype):
                v = str(v)
            elif isinstance(v, torch.Tensor):
                v = v.tolist()
            out[f.name] = v
        return out

    @classmethod
    def from_rpc_param(cls, d: dict):
        kw = {}
        for f in fields(cls):
            if f.name in d:
                v = d[f.name]
                if isinstance(v, str) and v.startswith("torch."):
                    v = getattr(torch, v.split(".", 1)[1])
                kw[f.name] = v
        return cls(**kw)


@dataclass
class GenerationConfig:
    max_new_tokens: Optional[int] = None
    max_length: Optional[int] = None
    do_sample: bool = False
    temperature: float = 1.0
    top_k: Optional[int] = None
    top_p: Optional[float] = None
    min_p: Optional[float] = None
    repetition_penalty: float = 1.0
    no_repeat_ngram_size: int = 0
    forced_eos_token_id: Optional[int] = None
    num_beams: int = 1
    eos_token_id: Optional[Union[int, List[int]]] = None
    pad_token_id: Optional[int] = None
    length_penalty: float = 1.0
    early_stopping: bool = False

    def to_dict(self) -> Dict[str, Any]:
        return {f.name: getattr(self, f.name) for f in fields(self)}


@dataclass
class InputMetaData(RPC_PARAM):
    """Per-step metadata handed to the model (flattened, un-padded batch)."""

    block_tables: torch.Tensor = None
    sequence_lengths: torch.Tensor = None
    fd_inter_tensor: Any = None
    batch_size: int = 64
    is_prompts: bool = False
    use_cuda_kernel: bool = False
    use_cuda_graph: bool = False
    kv_seq_len: int = 512
    head_dim: int = 32
    high_precision: bool = False
    dtype: torch.dtype = torch.float32
    use_spec_dec: bool = False
    num_tokens_to_verify: int = 0
    batch_token_ids: Optional[List[List[int]]] = None

    def __repr__(self) -> str:
        return (f"InputMetaData(batch_size={self.batch_size}, is_prompts={self.is_prompts}, "
                f"kv_seq_len={self.kv_seq_len}, use_cuda_graph={self.use_cuda_graph})")


@dataclass
class InferenceConfig(RPC_PARAM):
    """Engine configuration (names follow the reference)."""

    max_batch_size: int = 8
    max_output_len: int = 256
    max_input_len: int = 256
    dtype: Union[str, torch.dtype] = torch.float16
    kv_cache_dtype: Optional[str] = None          # None -> model dtype; "fp8" -> e5m2 storage
    prompt_template: Optional[str] = None
    do_sample: bool = False
    beam_width: int = 1
    prefill_ratio: Optional[float] = 1.2
    pad_input: bool = False
    early_stopping: Optional[bool] = False
    top_k: Optional[int] = 50
    top_p: Optional[float] = 1.0
    temperature: Optional[float] = 1.0
    no_repeat_ngram_size: Optional[int] = 0
    repetition_penalty: Optional[float] = 1.0
    forced_eos_token_id: int = None
    max_n_spec_tokens: int = 5
    glimpse_large_kv: bool = False
    block_size: int = 16
    tp_size: int = 1
    pp_size: int = 1
    micro_batch_size: int = 1
    use_cuda_kernel: bool = True
    high_precision: Optional[bool] = False
    use_cuda_graph: bool = False
    max_context_len_to_capture: int = 512
    enable_streamingllm: bool = False
    start_token_size: int = 4
    generated_token_size: int = 512
    pattern: Optional[str] = None
    patched_parallelism_size: int = 1
    ignore_eos: bool = False
    use_spec_dec: bool = False
    # reuse the cached K/V of full blocks whose tokens (and every token before them) equal a prompt's: the prompt's
    # prefill computes only the rest.  Off by default, like the other cache features.
    enable_prefix_caching: bool = False
    # chunked prefill: no step feeds the model more than this many tokens.  Every decoding sequence feeds its token and
    # prompt chunks fill the rest, so a long prompt no longer stalls the running streams.  None: whole prompts, with
    # prefill and decode in separate steps.
    max_num_batched_tokens: Optional[int] = None

    def __post_init__(self) -> None:
        self.max_context_len_to_capture = self.max_input_len + self.max_output_len
        self._verify_config()

    def _verify_config(self) -> None:
        if isinstance(self.dtype, str):
            assert self.dtype in _DTYPE_MAPPING, f"dtype must be one of {list(_DTYPE_MAPPING)}"
            self.dtype = _DTYPE_MAPPING[self.dtype]
        assert self.dtype in _ALLOWED_DTYPES, f"Expected dtype in {_ALLOWED_DTYPES}, got {self.dtype}"
        if self.kv_cache_dtype:
            assert self.kv_cache_dtype in ("fp8",), f"kv_cache_dtype must be None or 'fp8', got {self.kv_cache_dtype}"
        assert self.block_size in (8, 16, 32, 64, 128), "block_size must be one of 8/16/32/64/128"
        if self.prompt_template is not None:
            if self.prompt_template in _DEFAULT_PROMPT_TEMPLATES:
                self.prompt_template = _DEFAULT_PROMPT_TEMPLATES[self.prompt_template]
            else:
                assert "{input_text}" in self.prompt_template, "custom prompt templates need an {input_text} placeholder"
        if self.enable_streamingllm:
            assert self.start_token_size <= self.block_size, "start_token_size must fit in one block"
            assert self.generated_token_size % self.block_size == 0
            self.start_token_size = self.block_size
        # streamingLLM rewrites block tables and rolls blocks out of the window, so blocks cannot be shared
        assert not (self.enable_prefix_caching and self.enable_streamingllm), \
            "enable_prefix_caching cannot be combined with enable_streamingllm"
        if self.max_num_batched_tokens is not None:
            n = self.max_num_batched_tokens
            # chunks end on block boundaries, and every step has room for one block of prompt after one token per
            # running sequence
            assert n > 0 and n % self.block_size == 0, "max_num_batched_tokens must be a positive multiple of block_size"
            assert n >= self.max_batch_size + self.block_size, \
                "max_num_batched_tokens must be at least max_batch_size + block_size"
            assert not self.enable_streamingllm, "max_num_batched_tokens cannot be combined with enable_streamingllm"
            assert self.beam_width == 1, "max_num_batched_tokens cannot be combined with beam_width > 1"

    def to_generation_config(self, model_config=None) -> GenerationConfig:
        meta = dict(max_length=self.max_input_len + self.max_output_len, max_new_tokens=self.max_output_len)
        for t in ("do_sample", "top_k", "top_p", "temperature", "no_repeat_ngram_size", "repetition_penalty",
                  "forced_eos_token_id", "early_stopping"):
            if getattr(self, t, None) is not None:
                meta[t] = getattr(self, t)
        meta["num_beams"] = self.beam_width
        if model_config is not None:
            for t in ("pad_token_id", "bos_token_id", "eos_token_id"):
                if getattr(model_config, t, None) is not None and t in GenerationConfig.__dataclass_fields__:
                    meta[t] = getattr(model_config, t)
        return GenerationConfig(**{k: v for k, v in meta.items() if k in GenerationConfig.__dataclass_fields__})


@dataclass
class ModelShardInferenceConfig:
    dtype: torch.dtype = None
    use_cuda_kernel: bool = False
    use_spec_dec: bool = False
    use_flash_attn: bool = False
    patched_parallelism_size: int = 1


@dataclass
class DiffusionGenerationConfig:
    prompt_2: Optional[Union[str, List[str]]] = None
    prompt_3: Optional[Union[str, List[str]]] = None
    height: Optional[int] = None
    width: Optional[int] = None
    num_inference_steps: int = None
    timesteps: List[int] = None
    guidance_scale: float = None
    negative_prompt: Optional[Union[str, List[str]]] = None
    num_images_per_prompt: Optional[int] = 1
    generator: Any = None
    latents: Any = None
    output_type: Optional[str] = "pil"
    return_dict: bool = True
    joint_attention_kwargs: Optional[Dict[str, Any]] = None
    clip_skip: Optional[int] = None
    callback_on_step_end: Any = None

    def to_dict(self) -> Dict[str, Any]:
        return {k: v for k, v in self.__dict__.items() if v is not None}
