"""SmoothQuant W8A8 linear on the GPU: int8 activations (per token, or one calibrated static scale) times int8
weights (per output channel) on the int8 wgmma GEMM.

`quantize_per_token(x)` / `quantize_static(x, act_scale)` run the int8 mode of the per-row quantiser
(kernel/csrc/quant.cu, `cb_int8_quant_rows`); `w8a8_linear(x, w_q, w_scale, bias, act_scale)` quantises x and runs
`cb_gemm_w8a8` (kernel/csrc/gemm_wgmma.cu): exact int32 sums, then y = (acc * sx) * w_scale + bias rounded once to
x's dtype.  Both are bitwise equal to the PyTorch path of `quantization.smoothquant.W8A8Linear` with an exact integer
GEMM.  Shapes whose output tiles fill at most half the SMs (decode batches) split K across CTAs; the launcher chooses,
and this module only provides the zeroed int32 workspace it asks for.  This module is the only caller of the two
launchers.
"""
from __future__ import annotations

import ctypes
from typing import Optional, Tuple

import torch

from ..kernel import loader
from ._dispatch import use_native
from ._dtypes import code

__all__ = ["supported", "quantize_per_token", "quantize_static", "w8a8_linear", "MAX_K"]

MAX_K = 133143      # 127 * 127 * K must fit in the int32 accumulator
_FLOAT = (torch.float32, torch.float16, torch.bfloat16)
_gemm_lib = None
_quant_lib = None


def _libs():
    global _gemm_lib, _quant_lib
    if _gemm_lib is None:
        _gemm_lib = loader.load("cb200_gemm")
        _gemm_lib.cb_gemm_w8a8_workspace.restype = ctypes.c_longlong
        _quant_lib = loader.load("cb200_quant")
    return _gemm_lib, _quant_lib


def _vec(t: Optional[torch.Tensor], n: int, dtypes, device) -> bool:
    return t is None or (t.dtype in dtypes and t.numel() == n and t.is_contiguous() and t.device == device)


def supported(x: torch.Tensor, w_q: torch.Tensor, w_scale: torch.Tensor, bias: Optional[torch.Tensor] = None,
              act_scale: Optional[torch.Tensor] = None) -> bool:
    """The native path's envelope: an sm_90 GPU; x [..., K] in fp32 / fp16 / bf16 with unit column stride; w_q a
    contiguous int8 [N, K] with a 16-byte aligned base, K a multiple of 16 (the TMA row stride) and at most MAX_K, N even
    (two output columns per store); w_scale fp32 [N]; bias [N] in fp32 / fp16 / bf16 or None; act_scale None (per
    token) or one fp32 element."""
    if not use_native(x) or x.dim() < 1 or x.dtype not in _FLOAT or x.numel() == 0 or x.stride(-1) != 1:
        return False
    if torch.cuda.get_device_capability(x.device)[0] != 9:
        return False
    if w_q.dtype != torch.int8 or w_q.dim() != 2 or not w_q.is_contiguous() or w_q.device != x.device:
        return False
    N, K = w_q.shape
    if x.shape[-1] != K or K % 16 or K > MAX_K or N % 2 or N == 0 or w_q.data_ptr() % 16:
        return False
    return (w_scale is not None and _vec(w_scale, N, (torch.float32,), x.device) and _vec(bias, N, _FLOAT, x.device)
            and _vec(act_scale, 1, (torch.float32,), x.device))


def _quantize(x2: torch.Tensor, act_scale: Optional[torch.Tensor]):
    M, K = x2.shape
    xq = torch.empty(M, K, dtype=torch.int8, device=x2.device)
    sx = torch.empty(M, 1, dtype=torch.float32, device=x2.device) if act_scale is None else act_scale
    rc = _libs()[1].cb_int8_quant_rows(loader.ptr(x2), loader.ptr(xq), M, K, ctypes.c_int64(x2.stride(0)),
                                       loader.ptr(None if act_scale is not None else sx), loader.ptr(act_scale),
                                       code(x2.dtype), loader.stream_ptr())
    loader.check(rc, "int8_quant_rows")
    loader.launch_counter.add("w8a8_quant")
    return xq, sx


def _rows(x: torch.Tensor) -> torch.Tensor:
    x2 = x.reshape(-1, x.shape[-1])
    return x2 if x2.stride(-1) == 1 else x2.contiguous()


def quantize_per_token(x: torch.Tensor) -> Tuple[torch.Tensor, torch.Tensor]:
    """(int8 [M, K], fp32 scales [M, 1]) of x [M, K], bitwise equal to `quantize_activation_per_token` on the GPU."""
    return _quantize(_rows(x), None)


def quantize_static(x: torch.Tensor, act_scale: torch.Tensor) -> torch.Tensor:
    """int8 [M, K] = clamp(round(x / act_scale), -127, 127) with a device fp32 scalar act_scale."""
    return _quantize(_rows(x), act_scale.reshape(1))[0]


def w8a8_linear(x: torch.Tensor, w_q: torch.Tensor, w_scale: torch.Tensor, bias: Optional[torch.Tensor],
                act_scale: Optional[torch.Tensor] = None) -> torch.Tensor:
    """y[..., N] = (int8(x) @ w_q^T) * sx * w_scale + bias in x's dtype; sx per token when act_scale is None, else the
    static scale.  Raises ValueError outside `supported(...)`."""
    if not supported(x, w_q, w_scale, bias, act_scale):
        raise ValueError("w8a8_linear: arguments outside the native envelope (see ops.w8a8.supported)")
    x2 = _rows(x)
    xq, sx = _quantize(x2, None if act_scale is None else act_scale.reshape(1))
    return _gemm(xq, sx, act_scale is None, w_q, w_scale, bias, x.dtype).view(*x.shape[:-1], w_q.shape[0])


def _gemm(xq, sx, per_row, w_q, w_scale, bias, out_dtype) -> torch.Tensor:
    """y [M, N] = (xq @ w_q^T) * sx * w_scale + bias; xq int8 [M, K] contiguous, sx fp32 [M] (per_row) or [1]."""
    M, K = xq.shape
    N = w_q.shape[0]
    gemm, _ = _libs()
    y = torch.empty(M, N, dtype=out_dtype, device=xq.device)
    ws_bytes = int(gemm.cb_gemm_w8a8_workspace(M, N, K))
    ws = torch.zeros((ws_bytes + 3) // 4, dtype=torch.int32, device=xq.device) if ws_bytes else None
    rc = gemm.cb_gemm_w8a8(loader.ptr(xq), loader.ptr(w_q), loader.ptr(y), M, N, K, K, K, N, loader.ptr(sx),
                           int(per_row), loader.ptr(w_scale), loader.ptr(bias),
                           code(bias.dtype) if bias is not None else 0, code(y.dtype), loader.ptr(ws),
                           ctypes.c_longlong(ws_bytes), loader.stream_ptr())
    loader.check(rc, "gemm_w8a8")
    loader.launch_counter.add("gemm_w8a8_splitk" if ws_bytes else "gemm_w8a8")
    return y
