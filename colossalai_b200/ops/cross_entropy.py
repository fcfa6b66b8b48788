"""Building blocks of the (vocab-parallel) cross entropy: row max, sum-exp + target logit, softmax gradient.

Native path: `kernel/csrc/cross_entropy.cu`.  Reference path: PyTorch fp32.
Parity: the math of reference `DistCrossEntropy` (`colossalai/shardformer/layer/loss.py:25-127`).
"""
from __future__ import annotations

import ctypes
from typing import Optional

import torch

from ..kernel import loader
from ._align import aligned
from ._dispatch import use_native
from ._dtypes import code

_lib = None


def _get_lib():
    global _lib
    if _lib is None:
        _lib = loader.load("cb200_loss")
    return _lib


def _ok(logits: torch.Tensor) -> bool:
    vec = 4 if logits.dtype == torch.float32 else 8
    return (use_native(logits) and logits.dtype in (torch.float32, torch.float16, torch.bfloat16)
            and logits.shape[-1] % vec == 0 and logits.is_contiguous())


def row_max(logits: torch.Tensor, valid_cols: Optional[int] = None) -> torch.Tensor:
    Vv = logits.shape[-1] if valid_cols is None else valid_cols
    if _ok(logits):
        lib = _get_lib()
        logits = aligned(logits)   # rows are read as 16-byte vectors
        T, V = logits.shape
        out = torch.empty(T, dtype=torch.float32, device=logits.device)
        loader.check(lib.cb_ce_row_max(loader.ptr(logits), loader.ptr(out), T, V, Vv, code(logits.dtype),
                                       loader.stream_ptr()), "ce_row_max")
        loader.launch_counter.add("ce_row_max")
        return out
    return logits[:, :Vv].float().max(dim=-1).values


def sumexp_and_target(logits: torch.Tensor, target: torch.Tensor, gmax: torch.Tensor, vocab_start: int,
                      ignore_index: int, valid_cols: Optional[int] = None) -> torch.Tensor:
    """Returns fp32 [2, T]: row 0 = sum_j exp(x_j - gmax); row 1 = x_target if this rank owns the target else 0."""
    T, V = logits.shape
    Vv = V if valid_cols is None else valid_cols
    if _ok(logits):
        lib = _get_lib()
        logits = aligned(logits)
        out = torch.empty(2, T, dtype=torch.float32, device=logits.device)
        tgt = (target if target.dtype == torch.int64 else target.long()).contiguous()
        loader.check(lib.cb_ce_sumexp_target(loader.ptr(logits), loader.ptr(tgt), loader.ptr(gmax),
                                             loader.ptr(out), T, V, Vv, ctypes.c_int64(vocab_start),
                                             ctypes.c_int64(ignore_index), code(logits.dtype),
                                             loader.stream_ptr()), "ce_sumexp_target")
        loader.launch_counter.add("ce_sumexp_target")
        return out
    xf = logits[:, :Vv].float()
    sumexp = torch.exp(xf - gmax.unsqueeze(-1)).sum(-1)
    local = target - vocab_start
    own = (local >= 0) & (local < Vv) & (target != ignore_index)
    idx = local.clamp(0, Vv - 1)
    tl = xf.gather(-1, idx.unsqueeze(-1)).squeeze(-1)
    tl = torch.where(own, tl, torch.zeros_like(tl))
    return torch.stack([sumexp, tl], 0)


def softmax_grad(logits: torch.Tensor, target: torch.Tensor, gmax: torch.Tensor, sumexp: torch.Tensor,
                 scale: Optional[torch.Tensor], vocab_start: int, ignore_index: int,
                 row_scale: Optional[torch.Tensor] = None, valid_cols: Optional[int] = None) -> torch.Tensor:
    """grad[t, j] = s_t * (softmax(x)[t, j] - 1[j == target_t])  with s_t = scale (scalar tensor) or row_scale[t];
    rows whose target == ignore_index get zero."""
    T, V = logits.shape
    Vv = V if valid_cols is None else valid_cols
    if row_scale is None:
        row_scale = scale.reshape(1).expand(T)
    row_scale = row_scale.float().contiguous()
    if _ok(logits):
        lib = _get_lib()
        logits = aligned(logits)
        out = torch.empty_like(logits)
        tgt = (target if target.dtype == torch.int64 else target.long()).contiguous()
        loader.check(lib.cb_ce_softmax_grad(loader.ptr(logits), loader.ptr(tgt), loader.ptr(gmax),
                                            loader.ptr(sumexp), loader.ptr(row_scale), loader.ptr(out),
                                            T, V, Vv, ctypes.c_int64(vocab_start), ctypes.c_int64(ignore_index),
                                            code(logits.dtype), loader.stream_ptr()), "ce_softmax_grad")
        loader.launch_counter.add("ce_softmax_grad")
        return out
    xf = logits[:, :Vv].float()
    p = torch.exp(xf - gmax.unsqueeze(-1)) / sumexp.unsqueeze(-1)
    local = target - vocab_start
    own = (local >= 0) & (local < Vv)
    idx = local.clamp(0, Vv - 1)
    onehot = torch.zeros_like(p)
    onehot.scatter_(-1, idx.unsqueeze(-1), own.float().unsqueeze(-1))
    g = (p - onehot) * row_scale.unsqueeze(-1)
    g = torch.where((target != ignore_index).unsqueeze(-1), g, torch.zeros_like(g))
    if Vv < V:
        g = torch.cat([g, g.new_zeros(T, V - Vv)], dim=-1)
    return g.to(logits.dtype)
