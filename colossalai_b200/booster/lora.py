"""LoRA adapters (native; the reference wraps `peft`: `booster/plugin/*:enable_lora`, `checkpoint_io/*:
save_lora_as_pretrained`, `Booster.enable_lora` booster.py:243-288).

`LoraConfig(r, lora_alpha, target_modules, lora_dropout)`; `apply_lora` freezes the base model and wraps the targeted
linear layers (plain `nn.Linear`, our TP linears and the quantised `Linear4bit` / `Linear8bit` of QLoRA) with a
low-rank `B @ A` delta; adapters are saved in the peft-compatible layout (`adapter_config.json` + `adapter_model.{bin,safetensors}` with `base_model.model.<name>.lora_A.weight`).
"""
from __future__ import annotations

import json
import math
import os
from dataclasses import asdict, dataclass, field
from typing import Dict, List, Optional, Union

import torch
import torch.nn as nn
import torch.nn.functional as F

__all__ = ["LoraConfig", "LoraLinear", "apply_lora", "save_lora_adapters", "load_lora_adapters", "merge_lora",
           "lora_state_dict", "is_lora_model"]

_DEFAULT_TARGETS = ["q_proj", "k_proj", "v_proj", "qkv_proj", "o_proj", "query_key_value", "c_attn"]


@dataclass
class LoraConfig:
    r: int = 8
    lora_alpha: int = 16
    lora_dropout: float = 0.0
    target_modules: Optional[Union[List[str], str]] = None
    bias: str = "none"
    task_type: Optional[str] = "CAUSAL_LM"
    use_dora: bool = False
    init_lora_weights: bool = True

    def to_dict(self) -> dict:
        d = asdict(self)
        d["peft_type"] = "LORA"
        return d

    @classmethod
    def from_any(cls, cfg) -> "LoraConfig":
        if isinstance(cfg, cls):
            return cfg
        if isinstance(cfg, dict):
            return cls(**{k: v for k, v in cfg.items() if k in cls.__dataclass_fields__})
        kw = {k: getattr(cfg, k) for k in cls.__dataclass_fields__ if hasattr(cfg, k)}   # e.g. a peft.LoraConfig
        return cls(**kw)


class LoraLinear(nn.Module):
    """y = base(x) + (alpha/r) * dropout(x) A^T B^T.  `base` may be any module mapping [..., in] -> [..., out]."""

    def __init__(self, base: nn.Module, in_features: int, out_features: int, cfg: LoraConfig) -> None:
        super().__init__()
        self.base_layer = base
        self.r, self.scaling = cfg.r, cfg.lora_alpha / cfg.r
        w = getattr(base, "weight", None)
        if w is None and _is_quantized(base):
            # a frozen quantised base: adapters in its compute dtype, next to its packed buffers
            dev, dt = next(base.buffers()).device, base.compute_dtype
        else:
            dev = w.device if w is not None else None
            dt = w.dtype if (w is not None and w.is_floating_point()) else torch.float32
        self.lora_A = nn.Linear(in_features, cfg.r, bias=False, device=dev, dtype=dt)
        self.lora_B = nn.Linear(cfg.r, out_features, bias=False, device=dev, dtype=dt)
        self.lora_dropout = nn.Dropout(cfg.lora_dropout) if cfg.lora_dropout > 0 else nn.Identity()
        if cfg.init_lora_weights:
            nn.init.kaiming_uniform_(self.lora_A.weight, a=math.sqrt(5))
            nn.init.zeros_(self.lora_B.weight)
        self.merged = False

    @property
    def weight(self):
        return self.base_layer.weight

    @property
    def bias(self):
        return getattr(self.base_layer, "bias", None)

    def forward(self, x: torch.Tensor, *args, **kwargs):
        out = self.base_layer(x, *args, **kwargs)
        if self.merged:
            return out
        delta = self.lora_B(self.lora_A(self.lora_dropout(x))) * self.scaling
        if isinstance(out, tuple):
            return (out[0] + delta.to(out[0].dtype),) + out[1:]
        return out + delta.to(out.dtype)

    def merge(self) -> None:
        if _is_quantized(self.base_layer):
            raise NotImplementedError(
                f"cannot merge a LoRA adapter into a quantised {type(self.base_layer).__name__}: its weight is packed "
                "and frozen; load the unquantised base model and merge the saved adapters into it instead")
        if not self.merged and isinstance(self.base_layer, nn.Linear):
            self.base_layer.weight.data += (self.lora_B.weight @ self.lora_A.weight).to(self.base_layer.weight.dtype) \
                * self.scaling
            self.merged = True


def _is_quantized(m: nn.Module) -> bool:
    from ..quantization.bnb import Linear4bit, Linear8bit

    return isinstance(m, (Linear4bit, Linear8bit))


def _linear_dims(m: nn.Module):
    if isinstance(m, nn.Linear) or _is_quantized(m):
        return m.in_features, m.out_features
    w = getattr(m, "weight", None)
    if w is not None and w.dim() == 2 and hasattr(m, "forward") and type(m).__name__.startswith(("Linear1D", "Linear")):
        return w.shape[1], w.shape[0]
    return None


def is_lora_model(model: nn.Module) -> bool:
    return any(isinstance(m, LoraLinear) for m in model.modules())


def apply_lora(model: nn.Module, lora_config=None, pretrained_dir: Optional[str] = None) -> nn.Module:
    """Freeze `model`, wrap target linears, optionally load adapters from `pretrained_dir`."""
    if lora_config is None:
        assert pretrained_dir is not None, "either lora_config or pretrained_dir is required"
        with open(os.path.join(pretrained_dir, "adapter_config.json")) as f:
            lora_config = json.load(f)
    cfg = LoraConfig.from_any(lora_config)
    targets = cfg.target_modules or _DEFAULT_TARGETS
    if isinstance(targets, str):
        targets = [targets]
    for p in model.parameters():
        p.requires_grad_(False)
    n = 0
    for parent_name, parent in list(model.named_modules()):
        for child_name, child in list(parent.named_children()):
            if isinstance(child, LoraLinear) or child_name not in targets and not any(
                    (f"{parent_name}.{child_name}").endswith(t) for t in targets):
                continue
            dims = _linear_dims(child)
            if dims is None:
                continue
            setattr(parent, child_name, LoraLinear(child, dims[0], dims[1], cfg))
            n += 1
    if n == 0:
        raise ValueError(f"LoRA: no module matched target_modules={targets}")
    model._lora_config = cfg
    if pretrained_dir is not None:
        load_lora_adapters(model, pretrained_dir)
    return model


def lora_state_dict(model: nn.Module, prefix: str = "base_model.model.") -> Dict[str, torch.Tensor]:
    out = {}
    for name, m in model.named_modules():
        if isinstance(m, LoraLinear):
            out[f"{prefix}{name}.lora_A.weight"] = m.lora_A.weight.detach().cpu()
            out[f"{prefix}{name}.lora_B.weight"] = m.lora_B.weight.detach().cpu()
    return out


def save_lora_adapters(model: nn.Module, checkpoint: str, use_safetensors: bool = False,
                       state_dict: Optional[dict] = None) -> None:
    from ..interface import ModelWrapper

    if isinstance(model, ModelWrapper):
        model = model.unwrap()
    os.makedirs(checkpoint, exist_ok=True)
    sd = state_dict if state_dict is not None else lora_state_dict(model)
    cfg = getattr(model, "_lora_config", LoraConfig())
    with open(os.path.join(checkpoint, "adapter_config.json"), "w") as f:
        json.dump(cfg.to_dict(), f, indent=2)
    if use_safetensors:
        try:
            from safetensors.torch import save_file

            save_file({k: v.contiguous() for k, v in sd.items()}, os.path.join(checkpoint, "adapter_model.safetensors"))
            return
        except ImportError:
            pass
    torch.save(sd, os.path.join(checkpoint, "adapter_model.bin"))


def load_lora_adapters(model: nn.Module, checkpoint: str, prefix: str = "base_model.model.") -> None:
    st = os.path.join(checkpoint, "adapter_model.safetensors")
    if os.path.exists(st):
        from safetensors.torch import load_file

        sd = load_file(st)
    else:
        sd = torch.load(os.path.join(checkpoint, "adapter_model.bin"), map_location="cpu", weights_only=True)
    mods = dict(model.named_modules())
    for k, v in sd.items():
        name = k[len(prefix):] if k.startswith(prefix) else k
        mod_name, which, _ = name.rsplit(".", 2)
        which = which.split(".")[0]
        m = mods[mod_name]
        getattr(m, which).weight.data.copy_(v.to(getattr(m, which).weight.dtype))


def merge_lora(model: nn.Module, unload: bool = False) -> nn.Module:
    """Fold every adapter into its base weight; with `unload` the `LoraLinear` wrappers are replaced by the plain
    (now merged) base layers — peft's `merge_and_unload`."""
    for m in model.modules():
        if isinstance(m, LoraLinear):
            m.merge()
    if unload:
        for parent in list(model.modules()):
            for name, child in list(parent.named_children()):
                if isinstance(child, LoraLinear):
                    setattr(parent, name, child.base_layer)
    return model
