"""SmoothQuant W8A8 post-training quantisation: migrate activation outliers into the weights with a per-channel
smoothing vector `s = max|X|^alpha / max|W|^(1-alpha)` folded into the preceding norm, then run the linears with int8
weights (per output channel) and int8 activations (per token, dynamic) on the int8 tensor-core GEMM.

Parity: reference `colossalai/legacy/inference/quant/smoothquant/models/{base_model.py:1-480, linear.py:1-190,
llama.py}` (`get_act_scales`, `smooth_ln_fcs`, `W8A8B8O8Linear`, `W8A8BFP32OFP32Linear`, `SmoothLlamaForCausalLM`) —
those wrap torch-int CUTLASS int8 GEMMs.  Here, on an sm_90 GPU, `W8A8Linear` runs two native launches per call
(`ops.w8a8`: the per-token int8 quantiser, then the int8 wgmma GEMM with the scales and bias in its epilogue).  CPU
tensors and shapes outside that envelope run the PyTorch path below (`torch._int_mm` on CUDA, an exact integer
emulation on the CPU), which is also the numerics reference.
"""
from __future__ import annotations

from typing import Dict, Iterable, List, Optional, Sequence

import torch
import torch.nn as nn

from ..ops import w8a8

__all__ = ["get_act_scales", "smooth_ln_fcs", "quantize_weight_per_channel", "quantize_activation_per_token",
           "W8A8Linear", "smooth_and_quantize_model", "int8_matmul"]


@torch.no_grad()
def get_act_scales(model: nn.Module, calibration_batches: Iterable[Dict[str, torch.Tensor]]) -> Dict[str, torch.Tensor]:
    """Per input-channel max|x| seen by every `nn.Linear` over the calibration set."""
    scales: Dict[str, torch.Tensor] = {}

    def hook(name):
        def fn(mod, inp, out):
            x = inp[0].detach().reshape(-1, inp[0].shape[-1]).abs().max(dim=0).values.float()
            scales[name] = torch.maximum(scales[name], x) if name in scales else x
        return fn

    hooks = [m.register_forward_hook(hook(n)) for n, m in model.named_modules() if isinstance(m, nn.Linear)]
    was_training = model.training
    model.eval()
    for batch in calibration_batches:
        model(**batch)
    for h in hooks:
        h.remove()
    model.train(was_training)
    return scales


@torch.no_grad()
def smooth_ln_fcs(ln: nn.Module, fcs: Sequence[nn.Linear], act_scales: torch.Tensor, alpha: float = 0.5) -> torch.Tensor:
    """Divide the norm's affine output by `s`, multiply the input channels of the following linears by `s`:
    the float function is unchanged while activations lose their outlier channels."""
    w_max = torch.stack([fc.weight.abs().max(dim=0).values.float() for fc in fcs]).max(dim=0).values.clamp(min=1e-5)
    s = (act_scales.float().to(w_max.device).pow(alpha) / w_max.pow(1 - alpha)).clamp(min=1e-5)
    ln.weight.div_(s.to(ln.weight.dtype))
    if getattr(ln, "bias", None) is not None:
        ln.bias.div_(s.to(ln.bias.dtype))
    for fc in fcs:
        fc.weight.mul_(s.to(fc.weight.dtype).view(1, -1))
    return s


def quantize_weight_per_channel(w: torch.Tensor):
    """[out, in] -> int8 [out, in], scale [out] (symmetric absmax)."""
    scale = w.abs().amax(dim=1).float().clamp(min=1e-8) / 127.0
    q = torch.clamp(torch.round(w.float() / scale[:, None]), -127, 127).to(torch.int8)
    return q, scale


def quantize_activation_per_token(x: torch.Tensor):
    scale = x.abs().amax(dim=-1, keepdim=True).float().clamp(min=1e-8) / 127.0
    q = torch.clamp(torch.round(x.float() / scale), -127, 127).to(torch.int8)
    return q, scale


def int8_matmul(a: torch.Tensor, b_t: torch.Tensor) -> torch.Tensor:
    """int8 [M, K] x int8 [N, K]^T -> int32 [M, N] (IMMA on CUDA; exact emulation on CPU)."""
    if a.is_cuda and a.shape[0] > 16 and a.shape[0] % 8 == 0 and a.shape[1] % 8 == 0 and b_t.shape[0] % 8 == 0:
        return torch._int_mm(a.contiguous(), b_t.t().contiguous())
    if a.is_cuda:
        return (a.float() @ b_t.float().t()).round().to(torch.int32)      # small-M decode: exact below 2^24
    return a.to(torch.int32) @ b_t.to(torch.int32).t()


class W8A8Linear(nn.Module):
    """y = (int8(x) @ int8(W)^T) * sx * sw + b; activation scales per token (dynamic) or a calibrated static one."""

    def __init__(self, in_features: int, out_features: int, bias: bool = True, act_quant: str = "per_token",
                 static_act_scale: Optional[float] = None) -> None:
        super().__init__()
        self.in_features, self.out_features, self.act_quant = in_features, out_features, act_quant
        self.register_buffer("weight", torch.zeros(out_features, in_features, dtype=torch.int8))
        self.register_buffer("weight_scale", torch.ones(out_features, dtype=torch.float32))
        self.register_buffer("act_scale", torch.tensor(float(static_act_scale or 1.0)))
        self.bias = nn.Parameter(torch.zeros(out_features)) if bias else None

    @classmethod
    def from_float(cls, lin: nn.Linear, act_quant: str = "per_token", act_absmax: Optional[float] = None) -> "W8A8Linear":
        new = cls(lin.in_features, lin.out_features, lin.bias is not None, act_quant,
                  None if act_absmax is None else act_absmax / 127.0)
        q, s = quantize_weight_per_channel(lin.weight.data)
        new.weight, new.weight_scale = q, s
        if lin.bias is not None:
            new.bias.data = lin.bias.data.clone().float()
        return new.to(lin.weight.device)

    def _apply(self, fn, recurse=True):
        # a floating-point cast of the module must not round the quantisation scales: where `fn` changed a scale's
        # dtype, keep the fp32 original on the device `fn` moved it to
        state = {n: self._buffers[n] for n in ("weight_scale", "act_scale")}
        super()._apply(fn, recurse)
        for name, orig in state.items():
            moved = self._buffers[name]
            if moved.dtype != orig.dtype:
                self._buffers[name] = orig.to(device=moved.device)
        return self

    def forward(self, x: torch.Tensor) -> torch.Tensor:
        shape = x.shape
        x2 = x.reshape(-1, shape[-1])
        static = None if self.act_quant == "per_token" else self.act_scale
        # the native GEMM has no backward: a bias that needs a gradient stays on the autograd path below
        bias_grad = self.bias is not None and self.bias.requires_grad and torch.is_grad_enabled()
        if not bias_grad and w8a8.supported(x2, self.weight, self.weight_scale, self.bias, static):
            return w8a8.w8a8_linear(x2, self.weight, self.weight_scale, self.bias, static).reshape(
                *shape[:-1], self.out_features)
        if self.act_quant == "per_token":
            xq, sx = quantize_activation_per_token(x2)
        else:
            sx = self.act_scale
            xq = torch.clamp(torch.round(x2.float() / sx), -127, 127).to(torch.int8)
        acc = int8_matmul(xq, self.weight).float()
        y = acc * sx * self.weight_scale[None, :]
        if self.bias is not None:
            y = y + self.bias.float()
        return y.to(x.dtype).reshape(*shape[:-1], self.out_features)

    def extra_repr(self) -> str:
        return f"in={self.in_features}, out={self.out_features}, act_quant={self.act_quant}"


@torch.no_grad()
def smooth_and_quantize_model(model: nn.Module, calibration_batches: Iterable[Dict[str, torch.Tensor]],
                              alpha: float = 0.5, skip: Iterable[str] = ("lm_head",),
                              act_quant: str = "per_token") -> nn.Module:
    """Our decoder stack: smooth (input_layernorm -> qkv_proj) and (post_attention_layernorm -> gate_up/up proj), then
    swap every linear outside `skip` for `W8A8Linear`."""
    batches = list(calibration_batches)
    scales = get_act_scales(model, batches)
    mods = dict(model.named_modules())
    for name, m in mods.items():
        if hasattr(m, "input_layernorm") and hasattr(m, "self_attn") and hasattr(m.self_attn, "qkv_proj"):
            key = f"{name}.self_attn.qkv_proj"
            if key in scales and isinstance(m.self_attn.qkv_proj, nn.Linear):
                smooth_ln_fcs(m.input_layernorm, [m.self_attn.qkv_proj], scales[key], alpha)
            mlp = getattr(m, "mlp", None)
            first = getattr(mlp, "gate_up_proj", None) or getattr(mlp, "up_proj", None)
            if isinstance(first, nn.Linear) and hasattr(m, "post_attention_layernorm"):
                key = f"{name}.mlp." + ("gate_up_proj" if hasattr(mlp, "gate_up_proj") else "up_proj")
                if key in scales:
                    smooth_ln_fcs(m.post_attention_layernorm, [first], scales[key], alpha)
    static = get_act_scales(model, batches) if act_quant == "static" else {}
    for name, m in list(model.named_modules()):
        if isinstance(m, nn.Linear) and not any(s in name for s in skip):
            absmax = float(static[name].max()) if name in static else None
            new = W8A8Linear.from_float(m, act_quant, absmax)
            parent = model
            *path, leaf = name.split(".")
            for p in path:
                parent = getattr(parent, p)
            setattr(parent, leaf, new)
    return model
