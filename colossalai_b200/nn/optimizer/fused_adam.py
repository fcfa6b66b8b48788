"""FusedAdam: one multi-tensor launch per param group (sm_90a kernel; torch `_foreach` reference on CPU).
Parity: reference `colossalai/nn/optimizer/fused_adam.py` (multi_tensor_adam, adamw_mode, div_scale)."""
from __future__ import annotations

from typing import Dict, List, Optional

import torch

from ...ops import multi_tensor as mt
from ...ops._dispatch import use_native

__all__ = ["FusedAdam", "adam_reference_step"]


def adam_reference_step(params: List[torch.Tensor], grads: List[torch.Tensor], exp_avgs: List[torch.Tensor],
                        exp_avg_sqs: List[torch.Tensor], lr: float, beta1: float, beta2: float, eps: float,
                        weight_decay: float, step: int, adamw: bool, bias_correction: bool, inv_scale: float = 1.0,
                        lp_copies: Optional[List[Optional[torch.Tensor]]] = None) -> None:
    """Plain PyTorch Adam/AdamW on lists (the CPU tier and the numerics oracle of the fused kernel)."""
    bc1 = 1 - beta1 ** step if bias_correction else 1.0
    bc2 = 1 - beta2 ** step if bias_correction else 1.0
    for i, (p, g, m, v) in enumerate(zip(params, grads, exp_avgs, exp_avg_sqs)):
        gf = g.float() * inv_scale
        pf = p.float()
        if not adamw and weight_decay != 0:
            gf = gf + weight_decay * pf
        m.mul_(beta1).add_(gf, alpha=1 - beta1)
        v.mul_(beta2).addcmul_(gf, gf, value=1 - beta2)
        upd = (m / bc1) / ((v / bc2).sqrt() + eps)
        if adamw and weight_decay != 0:
            upd = upd + weight_decay * pf
        pf = pf - lr * upd
        p.copy_(pf)
        if lp_copies is not None and lp_copies[i] is not None:
            lp_copies[i].copy_(pf)


class FusedAdam(torch.optim.Optimizer):
    def __init__(self, params, lr: float = 1e-3, bias_correction: bool = True, betas=(0.9, 0.999), eps: float = 1e-8,
                 adamw_mode: bool = True, weight_decay: float = 0.0, amsgrad: bool = False,
                 set_grad_none: bool = True) -> None:
        if amsgrad:
            raise RuntimeError("FusedAdam does not support the AMSGrad variant")
        defaults = dict(lr=lr, bias_correction=bias_correction, betas=betas, eps=eps, weight_decay=weight_decay)
        super().__init__(params, defaults)
        self.adamw_mode = adamw_mode
        self.set_grad_none = set_grad_none
        self._tables: Dict[tuple, mt.TensorTable] = {}

    def zero_grad(self, set_to_none: bool = False) -> None:
        if set_to_none or self.set_grad_none:
            for group in self.param_groups:
                for p in group["params"]:
                    p.grad = None
        else:
            super().zero_grad(set_to_none=False)

    def _table(self, params, grads, ms, vs) -> mt.TensorTable:
        key = mt.TensorTable.key_of(params, grads, ms, vs)
        tbl = self._tables.get(key)
        if tbl is None:
            if len(self._tables) > 16:
                self._tables.clear()
            tbl = mt.TensorTable(params, grads, ms, vs, keepalive=True)
            self._tables[key] = tbl
        return tbl

    @torch.no_grad()
    def step(self, closure=None, div_scale: float = -1.0, grads=None, output_params=None, scale=None,
             grad_norms=None, inv_scale_dev: Optional[torch.Tensor] = None, noop_flag: Optional[torch.Tensor] = None):
        loss = closure() if closure is not None else None
        inv_scale = 1.0 / div_scale if div_scale > 0 else 1.0
        for group in self.param_groups:
            ps, gs, ms, vs = [], [], [], []
            staged = []         # (param, contiguous copy stepped in its place): written back after the step
            group["step"] = group.get("step", 0) + 1
            beta1, beta2 = group["betas"]
            for p in group["params"]:
                if p.grad is None:
                    continue
                if p.grad.is_sparse:
                    raise RuntimeError("FusedAdam does not support sparse gradients")
                st = self.state[p]
                if len(st) == 0:
                    st["exp_avg"] = torch.zeros_like(p, dtype=torch.float32, memory_format=torch.contiguous_format)
                    st["exp_avg_sq"] = torch.zeros_like(p, dtype=torch.float32, memory_format=torch.contiguous_format)
                if p.data.is_contiguous():
                    ps.append(p.data)
                else:
                    ps.append(p.data.contiguous())
                    staged.append((p, ps[-1]))
                gs.append(p.grad.data if p.grad.data.is_contiguous() else p.grad.data.contiguous())
                ms.append(st["exp_avg"])
                vs.append(st["exp_avg_sq"])
            if not ps:
                continue
            if use_native(ps[0]):
                # the staging copies are new tensors every step: a cached table would pin them
                tbl = mt.TensorTable(ps, gs, ms, vs) if staged else self._table(ps, gs, ms, vs)
                mt.adam(tbl, group["lr"], beta1, beta2, group["eps"], group["weight_decay"], group["step"],
                        self.adamw_mode, group["bias_correction"], inv_scale, noop_flag, inv_scale_dev)
            else:
                adam_reference_step(ps, gs, ms, vs, group["lr"], beta1, beta2, group["eps"], group["weight_decay"],
                                    group["step"], self.adamw_mode, group["bias_correction"], inv_scale)
            for p, c in staged:
                p.data.copy_(c)
        return loss
