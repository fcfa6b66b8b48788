"""Weight-only int8 / 4-bit (fp4, nf4) quantisation of nn.Linear layers.

The reference delegates to bitsandbytes (`colossalai/quantization/bnb.py:30-330`: quantize_model,
replace_with_bnb_layers, get_keys_to_not_convert, find_tied_parameters).  bitsandbytes is not part of this stack, so the
quantised layers are implemented here: block-wise absmax scaling, 8-bit signed codes or 4-bit codebook indices packed
two per byte.  On the GPU the forward and the input gradient run on `ops/wq_gemm.py`, whose kernel decodes the packed
weight inside the GEMM: no 16-bit copy of a frozen weight is kept for backward, which is what lets QLoRA train a model
whose 16-bit weights would not fit.  The quantisation state (absmax, scales, codebook) stays fp32 whatever dtype the
module is cast to.
"""
from __future__ import annotations

from typing import Dict, List, Optional

import torch
import torch.nn as nn
import torch.nn.functional as F

from .bnb_config import BnbQuantizationConfig

__all__ = ["quantize_model", "replace_with_bnb_layers", "get_keys_to_not_convert", "find_tied_parameters",
           "Linear8bit", "Linear4bit"]

# buffers of the quantisation state that must keep full precision through `module.to(dtype)` / `.half()` / `.bfloat16()`
_FP32_STATE = ("scale", "absmax", "absmax_meta", "code")


class _WeightOnlyLinear(torch.autograd.Function):
    """y = x W^T on a frozen quantised weight.  Only the module (whose buffers are the packed weight) is kept for
    backward; dX = dY W decodes the weight again."""

    @staticmethod
    def forward(ctx, x: torch.Tensor, layer: nn.Module) -> torch.Tensor:
        from ..ops.wq_gemm import wq_linear

        ctx.layer = layer
        return wq_linear(x, layer)

    @staticmethod
    def backward(ctx, dy: torch.Tensor):
        from ..ops.wq_gemm import wq_matmul_nn

        if not ctx.needs_input_grad[0]:
            return None, None
        return wq_matmul_nn(dy.contiguous(), ctx.layer), None


class _QuantLinearBase(nn.Module):
    def _apply(self, fn, recurse=True):
        # a floating-point cast of the module must not round the quantisation state: where `fn` changed a state
        # buffer's dtype, keep the fp32 original on the device `fn` moved it to
        state = {n: self._buffers[n] for n in _FP32_STATE if self._buffers.get(n) is not None}
        super()._apply(fn, recurse)
        for name, orig in state.items():
            moved = self._buffers[name]
            if moved.dtype != orig.dtype:
                self._buffers[name] = orig.to(device=moved.device)
        return self

    def dequantize(self) -> torch.Tensor:
        """The weight in the compute dtype; on the GPU through the native decode kernel, bitwise equal to
        `dequantize_reference()`."""
        from ..ops.wq_gemm import dequantize

        return dequantize(self)

    def forward(self, x: torch.Tensor) -> torch.Tensor:
        y = _WeightOnlyLinear.apply(x.to(self.compute_dtype), self)
        if self.bias is not None:
            y = y + self.bias
        return y.to(x.dtype)

_NF4 = [-1.0, -0.6961928009986877, -0.5250730514526367, -0.39491748809814453, -0.28444138169288635,
        -0.18477343022823334, -0.09105003625154495, 0.0, 0.07958029955625534, 0.16093020141124725,
        0.24611230194568634, 0.33791524171829224, 0.44070982933044434, 0.5626170039176941, 0.7229568362236023, 1.0]
_FP4 = [0.0, 0.0052083333, 0.6666667, 1.0, 0.3333333, 0.5, 0.1666667, 0.25,
        -0.0, -0.0052083333, -0.6666667, -1.0, -0.3333333, -0.5, -0.1666667, -0.25]


class Linear8bit(_QuantLinearBase):
    """Row-wise absmax int8 weights."""

    def __init__(self, linear: nn.Linear, compute_dtype: torch.dtype) -> None:
        super().__init__()
        w = linear.weight.data.float()
        scale = w.abs().amax(dim=1, keepdim=True).clamp_min(1e-8) / 127.0
        self.register_buffer("weight_q", torch.round(w / scale).clamp_(-127, 127).to(torch.int8))
        self.register_buffer("scale", scale.to(torch.float32))
        self.bias = None if linear.bias is None else nn.Parameter(linear.bias.data.to(compute_dtype), False)
        self.in_features, self.out_features, self.compute_dtype = linear.in_features, linear.out_features, compute_dtype

    def dequantize_reference(self) -> torch.Tensor:
        return (self.weight_q.float() * self.scale).to(self.compute_dtype)


class Linear4bit(_QuantLinearBase):
    """Block-wise absmax + 16-entry codebook (nf4 / fp4); optional double quantisation of the absmax vector."""

    def __init__(self, linear: nn.Linear, compute_dtype: torch.dtype, quant_type: str = "nf4", block_size: int = 64,
                 double_quant: bool = False) -> None:
        super().__init__()
        w = linear.weight.data.float().reshape(-1)
        self.shape = tuple(linear.weight.shape)
        pad = (-w.numel()) % block_size
        if pad:
            w = F.pad(w, (0, pad))
        blocks = w.view(-1, block_size)
        absmax = blocks.abs().amax(dim=1).clamp_min(1e-8)
        code = torch.tensor(_NF4 if quant_type == "nf4" else _FP4, dtype=torch.float32, device=w.device)
        normed = blocks / absmax[:, None]
        idx = (normed.unsqueeze(-1) - code).abs().argmin(dim=-1).to(torch.uint8).view(-1)
        self.register_buffer("packed", (idx[0::2] << 4) | idx[1::2])
        self.register_buffer("code", code)
        self.double_quant = double_quant
        if double_quant:
            off = absmax.mean()
            s = (absmax - off).abs().max().clamp_min(1e-8) / 127.0
            self.register_buffer("absmax_q", torch.round((absmax - off) / s).to(torch.int8))
            self.register_buffer("absmax_meta", torch.stack([off, s]))
        else:
            self.register_buffer("absmax", absmax)
        self.block_size, self.numel = block_size, linear.weight.numel()
        self.bias = None if linear.bias is None else nn.Parameter(linear.bias.data.to(compute_dtype), False)
        self.in_features, self.out_features, self.compute_dtype = linear.in_features, linear.out_features, compute_dtype

    def dequantize_reference(self) -> torch.Tensor:
        idx = torch.stack([self.packed >> 4, self.packed & 0xF], dim=1).view(-1).long()
        absmax = (self.absmax_q.float() * self.absmax_meta[1] + self.absmax_meta[0]) if self.double_quant else self.absmax
        w = self.code[idx].view(-1, self.block_size) * absmax[:, None]
        return w.view(-1)[: self.numel].view(self.shape).to(self.compute_dtype)


def find_tied_parameters(model: nn.Module) -> List[List[str]]:
    seen: Dict[int, List[str]] = {}
    for name, p in model.named_parameters(remove_duplicate=False):
        seen.setdefault(id(p), []).append(name)
    return [names for names in seen.values() if len(names) > 1]


def get_keys_to_not_convert(model: nn.Module) -> List[str]:
    """Keep tied weights and the output head in full precision (same rule as the reference, bnb.py:208-258)."""
    tied = [n for g in find_tied_parameters(model) for n in g]
    keep = {n.rsplit(".", 1)[0] for n in tied}
    children = list(model.named_modules())
    linears = [n for n, m in children if isinstance(m, nn.Linear)]
    if linears:
        keep.add(linears[-1])
    for n in ("lm_head", "score", "classifier"):
        if any(c == n or c.endswith("." + n) for c, _ in children):
            keep.add(n)
    return sorted(k for k in keep if k)


def replace_with_bnb_layers(model: nn.Module, bnb_quantization_config: BnbQuantizationConfig,
                            modules_to_not_convert: Optional[List[str]] = None, current_key_name=None) -> nn.Module:
    skip = modules_to_not_convert or []
    cfg = bnb_quantization_config

    def walk(mod: nn.Module, prefix: str) -> int:
        n = 0
        for name, child in list(mod.named_children()):
            full = f"{prefix}.{name}" if prefix else name
            if isinstance(child, nn.Linear) and not any(full == s or full.endswith("." + s) or s in full.split(".")
                                                        for s in skip):
                q = (Linear8bit(child, cfg.torch_dtype) if cfg.load_in_8bit else
                     Linear4bit(child, cfg.bnb_4bit_compute_dtype, cfg.bnb_4bit_quant_type, cfg.block_size,
                                cfg.bnb_4bit_use_double_quant))
                setattr(mod, name, q)
                n += 1
            else:
                n += walk(child, full)
        return n

    if walk(model, "") == 0:
        import warnings

        warnings.warn("No linear modules were found in the model; nothing was quantised.")
    return model


def quantize_model(model: nn.Module, bnb_quantization_config: BnbQuantizationConfig) -> nn.Module:
    cfg = bnb_quantization_config
    skip = list(cfg.skip_modules) if cfg.skip_modules is not None else get_keys_to_not_convert(model)
    keep32 = cfg.keep_in_fp32_modules or []
    skip = skip + keep32
    model = replace_with_bnb_layers(model, cfg, modules_to_not_convert=skip)
    for name, p in model.named_parameters():
        if any(k in name for k in keep32):
            p.data = p.data.float()
        elif p.is_floating_point():
            p.data = p.data.to(cfg.torch_dtype)
    dev = torch.device("cuda", torch.cuda.current_device()) if torch.cuda.is_available() else torch.device("cpu")
    return model.to(dev)
