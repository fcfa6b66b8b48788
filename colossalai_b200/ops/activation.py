"""Fused gated activations (SwiGLU / GeGLU) on a packed `[..., 2*I]` gate|up tensor, and bias+activation.

Native path: `kernel/csrc/elementwise.cu`.  Parity: reference `silu_and_mul` (N16), Triton `LlamaActCombine`,
TorchScript `bias_gelu` (`colossalai/kernel/jit/bias_gelu.py`).
"""
from __future__ import annotations

import ctypes
from typing import Optional

import torch
import torch.nn.functional as F

from ..kernel import loader
from ._align import aligned
from ._dispatch import use_native
from ._dtypes import code

_ACT = {"silu": 0, "swiglu": 0, "gelu_tanh": 1, "gelu_new": 1, "gelu_pytorch_tanh": 1, "gelu": 2, "geglu": 2}
_lib = None


def _get_lib():
    global _lib
    if _lib is None:
        _lib = loader.load("cb200_elementwise")
    return _lib


def _act_ref(x: torch.Tensor, act: int) -> torch.Tensor:
    if act == 0:
        return F.silu(x)
    if act == 1:
        return F.gelu(x, approximate="tanh")
    return F.gelu(x)


def glu_ref(gate_up: torch.Tensor, act: str = "silu") -> torch.Tensor:
    g, u = gate_up.float().chunk(2, dim=-1)
    return (_act_ref(g, _ACT[act]) * u).to(gate_up.dtype)


class _GLUFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, gate_up, act, valid_rows=None):
        lib = _get_lib()
        shape = gate_up.shape
        I = shape[-1] // 2
        gu = aligned(gate_up.contiguous().view(-1, 2 * I))
        out = torch.empty(gu.shape[0], I, dtype=gu.dtype, device=gu.device)
        loader.check(lib.cb_glu_fwd_bounded(loader.ptr(gu), loader.ptr(out), ctypes.c_int64(gu.shape[0]), I, act,
                                            code(gu.dtype), loader.ptr(valid_rows), loader.stream_ptr()), "glu_fwd")
        loader.launch_counter.add("glu_fwd")
        ctx.save_for_backward(gu, valid_rows if valid_rows is not None else torch.empty(0))
        ctx.act, ctx.shape = act, shape
        return out.view(shape[:-1] + (I,))

    @staticmethod
    def backward(ctx, dout):
        lib = _get_lib()
        gu, vr = ctx.saved_tensors
        vr = vr if vr.numel() else None
        I = gu.shape[1] // 2
        d = aligned(dout.contiguous().view(-1, I))
        dgu = torch.empty_like(gu)
        loader.check(lib.cb_glu_bwd_bounded(loader.ptr(d), loader.ptr(gu), loader.ptr(dgu), ctypes.c_int64(gu.shape[0]),
                                            I, ctx.act, code(gu.dtype), loader.ptr(vr), loader.stream_ptr()), "glu_bwd")
        loader.launch_counter.add("glu_bwd")
        return dgu.view(ctx.shape), None, None


def glu(gate_up: torch.Tensor, act: str = "silu", valid_rows: Optional[torch.Tensor] = None) -> torch.Tensor:
    """out = act(gate) * up where gate = gate_up[..., :I], up = gate_up[..., I:].
    `valid_rows` (int64 device scalar, optional): only the first `valid_rows` rows are computed (expert-parallel
    receive buffers are over-allocated and the number of rows that arrived is only known on the device); the rest of
    the output is left uninitialised."""
    I = gate_up.shape[-1] // 2
    vec = 4 if gate_up.dtype == torch.float32 else 8
    if use_native(gate_up) and gate_up.dtype in (torch.float32, torch.float16, torch.bfloat16) and I % vec == 0:
        if valid_rows is not None:
            valid_rows = valid_rows.to(device=gate_up.device, dtype=torch.int64).reshape(1).contiguous()
        return _GLUFn.apply(gate_up, _ACT[act], valid_rows)
    return glu_ref(gate_up, act)


def swiglu(gate_up: torch.Tensor) -> torch.Tensor:
    return glu(gate_up, "silu")


class _BiasActFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x, bias, act):
        lib = _get_lib()
        shape = x.shape
        H = shape[-1]
        x2 = aligned(x.contiguous().view(-1, H))
        bias = aligned(bias)
        y = torch.empty_like(x2)
        loader.check(lib.cb_bias_act_fwd(loader.ptr(x2), loader.ptr(bias), loader.ptr(y), ctypes.c_int64(x2.shape[0]),
                                         H, act, code(x.dtype), loader.stream_ptr()), "bias_act_fwd")
        loader.launch_counter.add("bias_act_fwd")
        ctx.save_for_backward(x2, bias)
        ctx.act, ctx.shape = act, shape
        return y.view(shape)

    @staticmethod
    def backward(ctx, dy):
        lib = _get_lib()
        x2, bias = ctx.saved_tensors
        H = x2.shape[1]
        d = aligned(dy.contiguous().view(-1, H))
        dx = torch.empty_like(x2)
        loader.check(lib.cb_bias_act_bwd(loader.ptr(d), loader.ptr(x2), loader.ptr(bias), loader.ptr(dx),
                                         ctypes.c_int64(x2.shape[0]), H, ctx.act, code(x2.dtype),
                                         loader.stream_ptr()), "bias_act_bwd")
        loader.launch_counter.add("bias_act_bwd")
        db = dx.sum(0) if bias is not None else None
        return dx.view(ctx.shape), db, None


def bias_act(x: torch.Tensor, bias: Optional[torch.Tensor], act: str = "gelu") -> torch.Tensor:
    """act(x + bias) fused (bias may be None)."""
    vec = 4 if x.dtype == torch.float32 else 8
    if (use_native(x) and x.dtype in (torch.float32, torch.float16, torch.bfloat16) and x.shape[-1] % vec == 0
            and (bias is None or bias.dtype == x.dtype)):
        return _BiasActFn.apply(x, bias, _ACT[act])
    h = x if bias is None else x + bias
    return _act_ref(h.float(), _ACT[act]).to(x.dtype)


def get_activation(name: str):
    name = name.lower()
    if name in ("silu", "swish"):
        return F.silu
    if name in ("gelu_new", "gelu_tanh", "gelu_pytorch_tanh", "gelu_fast"):
        return lambda x: F.gelu(x, approximate="tanh")
    if name == "gelu":
        return F.gelu
    if name == "relu":
        return F.relu
    if name == "quick_gelu":
        return lambda x: x * torch.sigmoid(1.702 * x)
    raise ValueError(f"unknown activation {name}")
