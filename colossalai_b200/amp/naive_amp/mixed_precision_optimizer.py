"""Mixed-precision optimizer: low-precision working params, fp32 master copy + moments.

Parity: reference `colossalai/amp/naive_amp/mixed_precision_optimizer.py:37-224` (master weights, unscale + clip,
overflow skip, `update_master_params`).  H100-first fast path: when the wrapped optimizer is an Adam-family optimizer
of ours and everything is on the GPU, ONE fused kernel launch per param group reads the bf16 grad, applies the
device-resident unscale x clip coefficient, updates the fp32 master + moments and writes the bf16 working copy —
no separate unscale pass, no grad fp32 materialisation, no master->working copy pass, no host sync for the norm.
"""
from __future__ import annotations

import math
from typing import Dict, List, Optional, Tuple

import torch
import torch.distributed as dist
from torch import Tensor, inf
from torch.nn import Module, Parameter
from torch.optim import Optimizer

from ...interface import OptimizerWrapper
from ...ops import multi_tensor as mt
from ...ops._dispatch import use_native
from .mixed_precision_mixin import BF16MixedPrecisionMixin, FP16MixedPrecisionMixin

__all__ = ["MixedPrecisionOptimizer", "NaiveFP16MixedPrecisionMixin"]


class NaiveFP16MixedPrecisionMixin(FP16MixedPrecisionMixin):
    def __init__(self, working_params: List[Parameter], **kw) -> None:
        super().__init__(**kw)
        self.params = working_params

    def check_local_overflow(self) -> bool:
        for p in self.params:
            if p.grad is not None and not torch.isfinite(p.grad).all():
                return True
        return False


def _is_fused_adam(optim: Optimizer) -> bool:
    from ...nn.optimizer.cpu_adam import CPUAdam
    from ...nn.optimizer.fused_adam import FusedAdam

    return isinstance(optim, (FusedAdam, CPUAdam)) or isinstance(optim, (torch.optim.AdamW, torch.optim.Adam))


class MixedPrecisionOptimizer(OptimizerWrapper):
    def __init__(self, optim: Optimizer, model: Module, precision: str = "fp16", initial_scale: float = 2**16,
                 min_scale: float = 1, growth_factor: float = 2, backoff_factor: float = 0.5,
                 growth_interval: int = 1000, hysteresis: int = 2, max_scale: float = 2**32, max_norm: float = 0.0,
                 fused: bool = True) -> None:
        super().__init__(optim)
        if precision == "fp16":
            working = [p for g in self.optim.param_groups for p in g["params"]]
            self.mixed_precision = NaiveFP16MixedPrecisionMixin(
                working, initial_scale=initial_scale, min_scale=min_scale, growth_factor=growth_factor,
                backoff_factor=backoff_factor, growth_interval=growth_interval, hysteresis=hysteresis,
                max_scale=max_scale)
        elif precision == "bf16":
            self.mixed_precision = BF16MixedPrecisionMixin()
        else:
            raise ValueError(f"unsupported precision: {precision}")
        self.max_norm = max_norm
        self.working_to_master_map: Dict[Parameter, Tensor] = {}
        self.master_to_working_map: Dict[Tensor, Parameter] = {}
        self._current_grad_norm: Optional[float] = None
        # fp32 master copies replace low-precision params inside the wrapped optimizer
        for group in self.optim.param_groups:
            master_params = []
            for p in group["params"]:
                if p.requires_grad:
                    master_p = p
                    if p.dtype != torch.float32:
                        master_p = p.detach().clone().float()
                        master_p.requires_grad_(False)
                        for a in ("dist_shard", "shard_fn", "gather_fn", "dist_global_shape", "ep_group",
                                  "moe_dp_group", "partial_derived"):
                            if hasattr(p, a):
                                setattr(master_p, a, getattr(p, a))
                        self.working_to_master_map[p] = master_p
                        self.master_to_working_map[master_p] = p
                    master_params.append(master_p)
            group["params"] = master_params
        self._use_fused = fused and _is_fused_adam(self.optim)
        self._tables: Dict[int, mt.TensorTable] = {}
        self._moments: Dict[Tensor, Tuple[Tensor, Tensor]] = {}
        self._step_count = 0

    # ------------------------------------------------------------------ backward
    def backward(self, loss: Tensor, inputs=None, retain_graph: bool = False, **kwargs) -> None:
        loss = self.mixed_precision.pre_backward(loss)
        loss.backward(inputs=inputs, retain_graph=retain_graph, **kwargs)

    def backward_by_grad(self, tensor: Tensor, grad: Tensor, inputs: Tensor = None, retain_graph: bool = False):
        grad = self.mixed_precision.pre_backward_by_grad(tensor, grad)
        torch.autograd.backward(tensors=tensor, grad_tensors=grad, inputs=inputs, retain_graph=retain_graph)

    def zero_grad(self, *args, **kwargs) -> None:
        for p in self.working_to_master_map.keys():
            p.grad = None
        self.mixed_precision.pre_zero_grad()
        return super().zero_grad(*args, **kwargs)

    # ------------------------------------------------------------------ grad norm (overridden by hybrid optimizers)
    def _working_params_with_grad(self) -> List[Parameter]:
        out = []
        for group in self.optim.param_groups:
            for mp in group["params"]:
                wp = self.master_to_working_map.get(mp, mp)
                if wp.grad is not None:
                    out.append(wp)
        return out

    def _local_grad_norm_sq(self, params: List[Parameter]) -> Tensor:
        """Sum of squared gradient entries of `params` as a device tensor [1] (no host sync)."""
        if not params:
            dev = "cuda" if torch.cuda.is_available() else "cpu"
            return torch.zeros(1, device=dev)
        grads = [p.grad for p in params]
        if use_native(grads[0]) and all(g.is_contiguous() for g in grads):
            return mt.norm_sq(mt.TensorTable(grads, grads), "grad")[0]
        return torch.stack([g.float().pow(2).sum() for g in grads]).sum().reshape(1)

    def _compute_grad_norm_sq(self, params: List[Parameter]) -> Tensor:
        """Global squared grad norm.  Base class: single group of replicated params."""
        return self._local_grad_norm_sq(params)

    # ------------------------------------------------------------------ step
    def _moments_for(self, mp: Tensor) -> Tuple[Tensor, Tensor]:
        st = self.optim.state[mp]
        if "exp_avg" not in st:
            st["exp_avg"] = torch.zeros_like(mp, dtype=torch.float32)
            st["exp_avg_sq"] = torch.zeros_like(mp, dtype=torch.float32)
            st["step"] = torch.tensor(0.0) if isinstance(self.optim, (torch.optim.AdamW, torch.optim.Adam)) else 0
        return st["exp_avg"], st["exp_avg_sq"]

    def _fused_step(self, div_scale: float, clip_coef_dev: Optional[Tensor]) -> None:
        self._step_count += 1
        adamw = getattr(self.optim, "adamw_mode", isinstance(self.optim, torch.optim.AdamW))
        for gi, group in enumerate(self.optim.param_groups):
            ps, gs, ms, vs, lps = [], [], [], [], []
            for mp in group["params"]:
                wp = self.master_to_working_map.get(mp, mp)
                if wp.grad is None:
                    continue
                m, v = self._moments_for(mp)
                ps.append(mp.data)
                gs.append(wp.grad.data if wp.grad.is_contiguous() else wp.grad.data.contiguous())
                ms.append(m)
                vs.append(v)
                lps.append(wp.data if wp is not mp else None)
            if not ps:
                continue
            group["step"] = group.get("step", 0) + 1
            # gradients are fresh allocations every step -> the descriptor table is rebuilt (cheap: one small H2D)
            tbl = mt.TensorTable(ps, gs, ms, vs, lps)
            beta1, beta2 = group["betas"]
            mt.adam(tbl, group["lr"], beta1, beta2, group["eps"], group["weight_decay"], group["step"], adamw,
                    group.get("bias_correction", True), inv_scale=1.0 / div_scale, inv_scale_dev=clip_coef_dev)

    def step(self, *args, **kwargs):
        if self.mixed_precision.should_skip_step():
            self.zero_grad()
            return
        working = self._working_params_with_grad()
        div_scale = self.mixed_precision.get_grad_div_scale()
        clip_coef_dev = None
        if self.max_norm > 0.0:
            norm_sq = self._compute_grad_norm_sq(working)
            total_norm = norm_sq.sqrt() / div_scale
            self._grad_norm_dev = total_norm
            # coefficient stays on the device: min(1, max_norm / (norm + eps))
            clip_coef_dev = (self.max_norm / (total_norm + 1e-6)).clamp(max=1.0).float().reshape(1)
        on_gpu = bool(working) and use_native(working[0].grad)
        if self._use_fused and on_gpu:
            self._fused_step(div_scale, clip_coef_dev)
            return
        # ---- generic path: master.grad = working.grad (fp32), unscale+clip, inner step, copy back
        for group in self.optim.param_groups:
            for mp in group["params"]:
                wp = self.master_to_working_map.get(mp)
                if wp is not None and wp.grad is not None:
                    mp.grad = wp.grad.data.float()
                    wp.grad = None
        coef = 1.0 / div_scale
        if clip_coef_dev is not None:
            coef = coef * clip_coef_dev.to(torch.float32)
        for group in self.optim.param_groups:
            for mp in group["params"]:
                if mp.grad is not None and (clip_coef_dev is not None or div_scale != 1.0):
                    mp.grad.mul_(coef.to(mp.grad.device) if torch.is_tensor(coef) else coef)
        self.optim.step(*args, **kwargs)
        for group in self.optim.param_groups:
            for mp in group["params"]:
                wp = self.master_to_working_map.get(mp)
                if wp is not None:
                    wp.data.copy_(mp.data)
                    mp.grad = None

    def get_grad_norm(self, norm_type=2.0, **kwargs) -> Optional[float]:
        g = getattr(self, "_grad_norm_dev", None)
        return None if g is None else float(g.item())

    def update_master_params(self, model: Module) -> None:
        for p in model.parameters():
            if p in self.working_to_master_map:
                self.working_to_master_map[p].data.copy_(p.data)

    def get_working_to_master_map(self) -> Dict[int, Tensor]:
        return {id(w): m for w, m in self.working_to_master_map.items()}

    def get_master_to_working_map(self) -> Dict[int, Tensor]:
        return {id(m): w for m, w in self.master_to_working_map.items()}
