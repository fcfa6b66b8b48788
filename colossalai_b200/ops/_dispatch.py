"""Native-vs-reference dispatch policy shared by every op.

Rule: CUDA tensors -> the sm_90a kernel (hard error if its library is missing on a GPU box);
CPU tensors -> the plain PyTorch reference (CPU plumbing tier).  `CB200_FORCE_TORCH=1` forces the reference
path on GPU too (used by the numerics tests and by the "baseline mode" of the benchmarks).
"""
from __future__ import annotations

import os
from contextlib import contextmanager

import torch

_force_torch = os.environ.get("CB200_FORCE_TORCH", "0") == "1"


def use_native(*tensors: torch.Tensor) -> bool:
    if _force_torch:
        return False
    for t in tensors:
        if t is not None:
            return t.is_cuda
    return False


@contextmanager
def force_torch(enabled: bool = True):
    """Context manager: run ops through their PyTorch reference implementation."""
    global _force_torch
    prev = _force_torch
    _force_torch = enabled
    try:
        yield
    finally:
        _force_torch = prev


def is_forced_torch() -> bool:
    return _force_torch
