"""Address alignment of tensors handed to the native kernels.

The memory-bound kernels read and write whole 16-byte vectors (`Vec16` in `kernel/csrc/common.cuh`), and the fp8
dequantiser reads 4-byte words.  A tensor can be contiguous and still start at any element offset: `flat[k:]` of a
flat buffer, a parameter inside a flat ZeRO chunk, or one rank's slice of an fp8 communication buffer.  A vector
access at such an address is a misaligned-address fault, so every native gate checks the tensors its kernel
vector-loads or stores with `is_aligned` / `rows_aligned`, and passes `aligned(t)` instead of `t`: the tensor
itself when it is aligned, otherwise a copy in a fresh block of the caching allocator (those start on 512-byte
boundaries).  The op stays native either way.
"""
from __future__ import annotations

from typing import Optional

import torch

VEC_BYTES = 16


def is_aligned(t: Optional[torch.Tensor], nbytes: int = VEC_BYTES) -> bool:
    """True if `t` is None or its first element starts on an `nbytes` boundary."""
    return t is None or t.data_ptr() % nbytes == 0


def rows_aligned(t: torch.Tensor, nbytes: int = VEC_BYTES) -> bool:
    """True if every row of the 2-D, unit-column-stride `t` starts on an `nbytes` boundary."""
    return is_aligned(t, nbytes) and t.stride(-1) == 1 and (t.stride(0) * t.element_size()) % nbytes == 0


def aligned(t: Optional[torch.Tensor], nbytes: int = VEC_BYTES) -> Optional[torch.Tensor]:
    """`t` if `is_aligned(t, nbytes)`, else a contiguous copy of it at a fresh, aligned address."""
    if is_aligned(t, nbytes):
        return t
    c = t.clone(memory_format=torch.contiguous_format)
    assert is_aligned(c, nbytes), "the allocator returned a misaligned block"
    return c
