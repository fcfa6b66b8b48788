"""FusedLAMB: two-stage multi-tensor LAMB with global grad-norm clipping.
Parity: reference `colossalai/nn/optimizer/fused_lamb.py:82`."""
from __future__ import annotations

import torch

from ...ops import multi_tensor as mt
from ...ops._dispatch import use_native
from .lamb import Lamb

__all__ = ["FusedLAMB"]


class FusedLAMB(torch.optim.Optimizer):
    def __init__(self, params, lr=1e-3, bias_correction=True, betas=(0.9, 0.999), eps=1e-6, weight_decay=0.01,
                 amsgrad=False, adam_w_mode=True, grad_averaging=True, set_grad_none=True, max_grad_norm=1.0,
                 use_nvlamb=False) -> None:
        if amsgrad:
            raise RuntimeError("FusedLAMB does not support the AMSGrad variant.")
        super().__init__(params, dict(lr=lr, bias_correction=bias_correction, betas=betas, eps=eps,
                                      weight_decay=weight_decay, grad_averaging=grad_averaging,
                                      max_grad_norm=max_grad_norm))
        self.adam_w_mode = adam_w_mode
        self.set_grad_none = set_grad_none
        self.use_nvlamb = use_nvlamb

    def zero_grad(self, set_to_none: bool = False):
        super().zero_grad(set_to_none=set_to_none or self.set_grad_none)

    @torch.no_grad()
    def step(self, closure=None):
        loss = closure() if closure is not None else None
        grads_all = [p.grad for g in self.param_groups for p in g["params"] if p.grad is not None]
        if not grads_all:
            return loss
        native = use_native(grads_all[0]) and all(g.is_contiguous() for g in grads_all)
        if native:
            gnorm = mt.norm_sq(mt.TensorTable(grads_all, grads_all), "grad")[0].sqrt()
        else:
            gnorm = torch.stack([g.float().pow(2).sum() for g in grads_all]).sum().sqrt()
        max_norm = self.defaults["max_grad_norm"]
        clip = (gnorm / max_norm).clamp(min=1.0) if max_norm and max_norm > 0 else torch.ones_like(gnorm)
        inv_scale = float(1.0 / clip.item())
        for group in self.param_groups:
            group["step"] = group.get("step", 0) + 1
            b1, b2 = group["betas"]
            ps, gs, ms, vs = [], [], [], []
            for p in group["params"]:
                if p.grad is None:
                    continue
                st = self.state[p]
                if len(st) == 0:
                    st["exp_avg"] = torch.zeros_like(p, dtype=torch.float32)
                    st["exp_avg_sq"] = torch.zeros_like(p, dtype=torch.float32)
                ps.append(p.data)
                gs.append(p.grad.data)
                ms.append(st["exp_avg"])
                vs.append(st["exp_avg_sq"])
            if not ps:
                continue
            # the trust ratio applies only with nvlamb or a non-zero weight decay (reference stage 2); otherwise a
            # group (typically biases and norms, weight_decay=0) steps with the plain learning rate
            trust = bool(self.use_nvlamb or group["weight_decay"] != 0)
            if native:
                mt.lamb(mt.TensorTable(ps, gs, ms, vs), group["lr"], b1, b2, group["eps"], group["weight_decay"],
                        group["step"], self.adam_w_mode, group["bias_correction"], group["grad_averaging"], inv_scale,
                        trust_ratio=trust)
            else:
                bc1 = 1 - b1 ** group["step"] if group["bias_correction"] else 1.0
                bc2 = 1 - b2 ** group["step"] if group["bias_correction"] else 1.0
                b3 = 1 - b1 if group["grad_averaging"] else 1.0
                for p, g, m, v in zip(ps, gs, ms, vs):
                    gf, pf = g.float() * inv_scale, p.float()
                    if not self.adam_w_mode:
                        gf = gf + group["weight_decay"] * pf
                    m.mul_(b1).add_(gf, alpha=b3)
                    v.mul_(b2).addcmul_(gf, gf, value=1 - b2)
                    u = (m / bc1) / ((v / bc2).sqrt() + group["eps"])
                    if self.adam_w_mode:
                        u = u + group["weight_decay"] * pf
                    ratio = 1.0
                    if trust:
                        pn, un = pf.norm(), u.norm()
                        ratio = torch.where((pn > 0) & (un > 0), pn / un, torch.ones_like(pn))
                    p.copy_(pf - group["lr"] * ratio * u)
        return loss
