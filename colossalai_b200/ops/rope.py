"""Rotary position embedding applied in place to the q/k head ranges of a packed QKV tensor.

Native path: `kernel/csrc/elementwise.cu::rope_kernel`.  Parity: reference `rotary_embedding` CUDA op (N15),
Triton `rotary_embedding`, HF `apply_rotary_pos_emb` call in `shardformer/modeling/llama.py:545`.
"""
from __future__ import annotations

import ctypes
from typing import Optional, Tuple

import torch

from ..kernel import loader
from ._align import VEC_BYTES, rows_aligned
from ._dispatch import use_native
from ._dtypes import code

_lib = None


def _get_lib():
    global _lib
    if _lib is None:
        _lib = loader.load("cb200_elementwise")
    return _lib


def build_rope_cache(max_pos: int, rot_dim: int, base: float = 10000.0, device=None,
                     scaling_factor: float = 1.0, llama3_scaling: Optional[dict] = None) -> Tuple[torch.Tensor, torch.Tensor]:
    """fp32 cos/sin caches of shape [max_pos, rot_dim/2]."""
    inv_freq = 1.0 / (base ** (torch.arange(0, rot_dim, 2, dtype=torch.float32, device=device) / rot_dim))
    if llama3_scaling:
        factor = llama3_scaling.get("factor", 8.0)
        low, high = llama3_scaling.get("low_freq_factor", 1.0), llama3_scaling.get("high_freq_factor", 4.0)
        old = llama3_scaling.get("original_max_position_embeddings", 8192)
        wavelen = 2 * torch.pi / inv_freq
        smooth = (old / wavelen - low) / (high - low)
        scaled = torch.where(wavelen > old / low, inv_freq / factor, inv_freq)
        mid = (1 - smooth) * inv_freq / factor + smooth * inv_freq
        is_mid = (wavelen <= old / low) & (wavelen >= old / high)
        inv_freq = torch.where(is_mid, mid, scaled)
    t = torch.arange(max_pos, dtype=torch.float32, device=device) / scaling_factor
    freqs = torch.outer(t, inv_freq)
    return freqs.cos().contiguous(), freqs.sin().contiguous()


def rope_ref(x: torch.Tensor, positions: Optional[torch.Tensor], cos: torch.Tensor, sin: torch.Tensor,
             rot_dim: Optional[int] = None, interleaved: bool = False, sign: float = 1.0) -> torch.Tensor:
    """x: [T, n_heads, D].  Returns rotated copy."""
    T, _, D = x.shape
    rot = rot_dim or D
    if positions is None:
        positions = torch.arange(T, device=x.device)
    c = cos[positions].unsqueeze(1)  # [T,1,rot/2]
    s = sin[positions].unsqueeze(1) * sign
    xf = x.float()
    xr, xp = xf[..., :rot], xf[..., rot:]
    if not interleaved:
        x1, x2 = xr[..., : rot // 2], xr[..., rot // 2:]
        out = torch.cat([x1 * c - x2 * s, x2 * c + x1 * s], dim=-1)
    else:
        x1, x2 = xr[..., 0::2], xr[..., 1::2]
        out = torch.stack([x1 * c - x2 * s, x2 * c + x1 * s], dim=-1).flatten(-2)
    return torch.cat([out, xp], dim=-1).to(x.dtype)


def _native_rope_(qkv2d: torch.Tensor, positions, cos, sin, n_rot_heads: int, D: int, rot_dim: int, sign: float,
                  interleaved: bool) -> None:
    if not rows_aligned(qkv2d):
        # the kernel rotates 16-byte vectors of each row: rotate an aligned copy with padded rows, then copy back
        vec = VEC_BYTES // qkv2d.element_size()
        T, W = qkv2d.shape
        tmp = torch.empty(T, -(-W // vec) * vec, dtype=qkv2d.dtype, device=qkv2d.device)[:, :W]
        tmp.copy_(qkv2d)
        _native_rope_(tmp, positions, cos, sin, n_rot_heads, D, rot_dim, sign, interleaved)
        qkv2d.copy_(tmp)
        return
    lib = _get_lib()
    loader.check(lib.cb_rope(loader.ptr(qkv2d), loader.ptr(positions), loader.ptr(cos), loader.ptr(sin),
                             ctypes.c_int64(qkv2d.shape[0]), ctypes.c_int64(qkv2d.stride(0)), n_rot_heads, D,
                             rot_dim, ctypes.c_float(sign), int(interleaved), code(qkv2d.dtype),
                             loader.stream_ptr()), "rope")
    loader.launch_counter.add("rope")


class _RopeQKVFn(torch.autograd.Function):
    """Rotates heads [0, n_rot_heads) of every token row of a packed [T, n_heads_total*D] buffer.
    The forward returns a NEW tensor (one extra write) so autograd never sees an in-place op on a saved tensor;
    the backward rotates the incoming gradient in place (it is a fresh buffer)."""

    @staticmethod
    def forward(ctx, qkv, positions, cos, sin, n_rot_heads, D, rot_dim, interleaved):
        out = qkv.clone(memory_format=torch.contiguous_format)
        _native_rope_(out.view(out.shape[0], -1), positions, cos, sin, n_rot_heads, D, rot_dim, 1.0, interleaved)
        ctx.save_for_backward(positions, cos, sin)
        ctx.cfg = (n_rot_heads, D, rot_dim, interleaved)
        return out

    @staticmethod
    def backward(ctx, dout):
        positions, cos, sin = ctx.saved_tensors
        n_rot_heads, D, rot_dim, interleaved = ctx.cfg
        d = dout.contiguous().clone() if not dout.is_contiguous() or dout._base is not None else dout.clone()
        _native_rope_(d.view(d.shape[0], -1), positions, cos, sin, n_rot_heads, D, rot_dim, -1.0, interleaved)
        return d, None, None, None, None, None, None, None


def rope_qkv(qkv: torch.Tensor, positions: Optional[torch.Tensor], cos: torch.Tensor, sin: torch.Tensor,
             n_q_heads: int, n_kv_heads: int, head_dim: int, rot_dim: Optional[int] = None,
             interleaved: bool = False) -> torch.Tensor:
    """qkv: [T, (n_q + 2*n_kv) * D] packed as q heads | k heads | v heads.  Rotates q and k."""
    rot = rot_dim or head_dim
    vec = 4 if qkv.dtype == torch.float32 else 8
    if positions is not None and positions.dtype != torch.int64:
        positions = positions.long()
    if (use_native(qkv) and qkv.dtype in (torch.float32, torch.float16, torch.bfloat16)
            and (rot // 2) % vec == 0 and head_dim % vec == 0):
        if positions is None:
            positions = torch.arange(qkv.shape[0], device=qkv.device)
        return _RopeQKVFn.apply(qkv, positions.contiguous(), cos, sin, n_q_heads + n_kv_heads, head_dim, rot,
                                interleaved)
    T = qkv.shape[0]
    x = qkv.view(T, n_q_heads + 2 * n_kv_heads, head_dim)
    qk = rope_ref(x[:, : n_q_heads + n_kv_heads], positions, cos, sin, rot, interleaved)
    return torch.cat([qk, x[:, n_q_heads + n_kv_heads:]], dim=1).reshape(T, -1)
