"""Norm layers backed by the fused sm_90a kernels (`ops.rms_norm`, `ops.layer_norm`).

Parity: reference `colossalai/shardformer/layer/normalization.py:27-353` (`FusedRMSNorm`, `FusedLayerNorm`,
`RMSNorm`, `LayerNorm` wrappers with `sp_partial_derived` marking).  No apex: the kernels are ours.
"""
from __future__ import annotations

from typing import Optional

import torch
import torch.nn as nn

from ... import ops
from .utils import SeqParallelUtils

__all__ = ["RMSNorm", "LayerNorm", "FusedRMSNorm", "FusedLayerNorm", "BaseLayerNorm"]


class BaseLayerNorm(nn.Module):
    @staticmethod
    def from_native_module(module: nn.Module, sp_partial_derived: bool = False, **kwargs) -> nn.Module:
        raise NotImplementedError


def _mark(module: nn.Module, sp_partial_derived: bool) -> None:
    if sp_partial_derived:
        for p in module.parameters(recurse=False):
            SeqParallelUtils.marked_as_sp_partial_derived_param(p)


class FusedRMSNorm(BaseLayerNorm):
    """y = x / rms(x) * w (optionally fused with a residual add: `forward(x, residual)` -> (y, x + residual))."""

    def __init__(self, hidden_size: int, eps: float = 1e-6, dtype=None, device=None, offset: float = 0.0) -> None:
        super().__init__()
        self.weight = nn.Parameter(torch.ones(hidden_size, dtype=dtype, device=device))
        self.variance_epsilon = eps
        self.eps = eps
        self.offset = offset  # gemma-style (1 + w)
        self.hidden_size = hidden_size

    def reset_parameters(self) -> None:
        nn.init.ones_(self.weight) if self.offset == 0.0 else nn.init.zeros_(self.weight)

    @staticmethod
    def from_native_module(module: nn.Module, sp_partial_derived: bool = False, **kwargs) -> "FusedRMSNorm":
        w = module.weight
        eps = getattr(module, "variance_epsilon", getattr(module, "eps", 1e-6))
        new = FusedRMSNorm(w.shape[0], eps=eps, dtype=w.dtype, device=w.device)
        new.weight = w
        _mark(new, sp_partial_derived)
        return new

    def forward(self, x: torch.Tensor, residual: Optional[torch.Tensor] = None):
        w = self.weight if self.offset == 0.0 else self.weight + self.offset
        if w.dtype != x.dtype:
            w = w.to(x.dtype)
        return ops.rms_norm(x, w, self.eps, residual)

    def extra_repr(self) -> str:
        return f"{self.hidden_size}, eps={self.eps}"


class FusedLayerNorm(BaseLayerNorm):
    def __init__(self, hidden_size: int, eps: float = 1e-5, bias: bool = True, dtype=None, device=None) -> None:
        super().__init__()
        self.weight = nn.Parameter(torch.ones(hidden_size, dtype=dtype, device=device))
        self.bias = nn.Parameter(torch.zeros(hidden_size, dtype=dtype, device=device)) if bias else None
        self.eps = eps
        self.hidden_size = hidden_size
        self.normalized_shape = (hidden_size,)

    def reset_parameters(self) -> None:
        nn.init.ones_(self.weight)
        if self.bias is not None:
            nn.init.zeros_(self.bias)

    @staticmethod
    def from_native_module(module: nn.LayerNorm, sp_partial_derived: bool = False, **kwargs) -> "FusedLayerNorm":
        new = FusedLayerNorm(module.weight.shape[0], eps=module.eps, bias=module.bias is not None,
                             dtype=module.weight.dtype, device=module.weight.device)
        new.weight = module.weight
        if module.bias is not None:
            new.bias = module.bias
        _mark(new, sp_partial_derived)
        return new

    def forward(self, x: torch.Tensor) -> torch.Tensor:
        w, b = self.weight, self.bias
        if w.dtype != x.dtype:
            w = w.to(x.dtype)
            b = None if b is None else b.to(x.dtype)
        return ops.layer_norm(x, w, b, self.eps)

    def extra_repr(self) -> str:
        return f"{self.hidden_size}, eps={self.eps}, bias={self.bias is not None}"


class RMSNorm(FusedRMSNorm):
    """Non-fused name kept for API parity; same module (the fused kernel is always used on CUDA)."""


class LayerNorm(FusedLayerNorm):
    """Non-fused name kept for API parity."""
