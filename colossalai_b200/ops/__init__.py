"""Python face of the native op set.  CUDA tensors -> sm_90a kernels; CPU tensors -> PyTorch reference."""
from ._dispatch import force_torch, is_forced_torch, use_native
from .activation import bias_act, get_activation, glu, glu_ref, swiglu
from .attention import attention, attention_ref, attention_with_lse_ref
from .gemm import linear_forward, matmul_nn, matmul_tn
from .norm import layer_norm, layer_norm_ref, rms_norm, rms_norm_ref
from .rope import build_rope_cache, rope_qkv, rope_ref

__all__ = [
    "force_torch", "is_forced_torch", "use_native", "bias_act", "get_activation", "glu", "glu_ref", "swiglu",
    "attention", "attention_ref", "attention_with_lse_ref", "linear_forward", "matmul_nn", "matmul_tn",
    "layer_norm", "layer_norm_ref", "rms_norm", "rms_norm_ref", "build_rope_cache", "rope_qkv", "rope_ref",
]
