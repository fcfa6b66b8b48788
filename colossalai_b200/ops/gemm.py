"""Dense GEMM entry points used by every linear layer.

`linear_forward(x, w)` = x @ w^T, `matmul_nn(a, b)` = a @ b, `matmul_tn(a, b)` = a^T @ b (wgrad).
Native path: our wgmma/TMA GEMM (kernel/csrc/gemm_wgmma.cu) for bf16/fp16 on sm_90a when the shape is
tile-aligned; otherwise cuBLAS through torch (plain library GEMM).  Parity: every `F.linear` / `torch.matmul`
call site in the reference's `shardformer/layer/_operation.py:90-737`.
"""
from __future__ import annotations

import os
from typing import Optional

import torch
import torch.nn.functional as F

from ._dispatch import use_native

_native = None
# plain (un-fused) GEMMs: "cublas" = library GEMM through torch (default), "native" = our wgmma kernel.
# The comm-fused GEMMs (parallel/fused.py) always run our main loop - there is no library equivalent.
_BACKEND = os.environ.get("CB200_GEMM_BACKEND", "cublas")


def set_gemm_backend(name: str) -> None:
    global _BACKEND
    assert name in ("cublas", "native")
    _BACKEND = name


def get_gemm_backend() -> str:
    return _BACKEND


def _try_native():
    global _native
    if _BACKEND != "native":
        return False
    if _native is None:
        try:
            from . import gemm_native

            _native = gemm_native if gemm_native.available() else False
        except Exception:
            _native = False
    return _native


def linear_forward(x: torch.Tensor, w: torch.Tensor, bias: Optional[torch.Tensor] = None) -> torch.Tensor:
    """y[..., N] = x[..., K] @ w[N, K]^T (+ bias)."""
    if use_native(x, w):
        n = _try_native()
        if n and n.supported_nt(x, w):
            y = n.gemm_nt(x.reshape(-1, x.shape[-1]), w).view(x.shape[:-1] + (w.shape[0],))
            return y if bias is None else y + bias
    return F.linear(x, w, bias)


def matmul_nn(a: torch.Tensor, b: torch.Tensor) -> torch.Tensor:
    """c[M, N] = a[M, K] @ b[K, N]   (dgrad: dX = dY @ W with W stored [N_out, K_in])."""
    if use_native(a, b):
        n = _try_native()
        if n and n.supported_nn(a, b):
            return n.gemm_nn(a, b)
    return a @ b


def matmul_tn(a: torch.Tensor, b: torch.Tensor, out: Optional[torch.Tensor] = None,
              accumulate: bool = False) -> torch.Tensor:
    """c[N, K] = a[M, N]^T @ b[M, K]   (wgrad: dW = dY^T @ X); optionally accumulate into `out`."""
    if use_native(a, b):
        n = _try_native()
        if n and n.supported_tn(a, b):
            if out is None or n.out_ok(out):
                return n.gemm_tn(a, b, out=out, accumulate=accumulate)
            # an output the epilogue cannot store into (a view at an odd element offset, or with an odd row stride):
            # run the GEMM into a fresh aligned buffer (holding a copy of `out` when accumulating) and write it back
            if accumulate:
                o = out.clone(memory_format=torch.contiguous_format)
            else:
                o = torch.empty(out.shape, dtype=out.dtype, device=out.device)
            n.gemm_tn(a, b, out=o, accumulate=accumulate)
            return out.copy_(o)
    if out is not None and a.is_cuda and out.dtype == a.dtype and out.is_contiguous():
        # library path: accumulate inside the GEMM epilogue (beta = 1) instead of a separate add pass
        if accumulate:
            return out.addmm_(a.t(), b)
        return torch.mm(a.t(), b, out=out)
    c = a.t() @ b
    if out is not None:
        if accumulate:
            out.add_(c)
        else:
            out.copy_(c)
        return out
    return c
