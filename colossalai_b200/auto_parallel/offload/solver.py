"""Parameter offload planning + runtime: pick which layers keep their parameters in host memory so the model fits a
device budget, and stream them in ahead of use.

* `SynGreedySolver`  — offload the layers with the best (bytes freed / stall time) ratio until the peak fits; every
  offloaded layer is fetched synchronously right before it runs.
* `AsynGreedySolver` — same selection, but each fetch is issued `prefetch_distance` layers early on a copy stream so the
  transfer hides under the compute of the layers in between; selection accounts for the hidden part.

`memory_optimize(model, budget)` applies a plan with forward pre/post hooks (fetch / release), pinned host copies and a
side CUDA stream.  The default host-link bandwidth is 50 GB/s (PCIe Gen5 x16 class).

Parity: reference `colossalai/auto_parallel/offload/{solver.py:1-520 (SynGreedySolver, AsynGreedySolver),
amp_optimizer.py, base_offload_module.py, runtime.py (pre-fwd / post-bwd upload-offload ops), mem_optimize.py:1-60}`.
"""
from __future__ import annotations

from dataclasses import dataclass, field
from typing import Dict, List, Optional, Sequence

import torch
import torch.nn as nn

__all__ = ["OffloadPlan", "SynGreedySolver", "AsynGreedySolver", "memory_optimize"]


@dataclass
class LayerCost:
    name: str
    param_bytes: float
    compute_s: float


@dataclass
class OffloadPlan:
    offloaded: List[str] = field(default_factory=list)
    prefetch_at: Dict[str, Optional[str]] = field(default_factory=dict)   # layer -> layer whose pre-hook starts the fetch
    peak_param_bytes: float = 0.0
    est_stall_s: float = 0.0


class SynGreedySolver:
    asynchronous = False

    def __init__(self, layers: Sequence[LayerCost], budget_bytes: float, bandwidth: float = 50e9,
                 prefetch_distance: int = 1) -> None:
        self.layers, self.budget, self.bw = list(layers), float(budget_bytes), float(bandwidth)
        self.distance = max(1, prefetch_distance)

    def _stall(self, idx: int) -> float:
        """Exposed transfer time if layer `idx` is offloaded."""
        t = self.layers[idx].param_bytes / self.bw
        if not self.asynchronous:
            return t
        hidden = sum(l.compute_s for l in self.layers[max(0, idx - self.distance):idx])
        return max(0.0, t - hidden)

    def _peak(self, off: set) -> float:
        """Resident bytes: all kept layers + the largest window of simultaneously live offloaded layers."""
        resident = sum(l.param_bytes for i, l in enumerate(self.layers) if i not in off)
        window = 0.0
        for i in range(len(self.layers)):
            live = sum(self.layers[j].param_bytes for j in range(i, min(len(self.layers), i + (
                self.distance + 1 if self.asynchronous else 1))) if j in off)
            window = max(window, live)
        return resident + window

    def solve(self) -> OffloadPlan:
        off: set = set()
        order = sorted(range(len(self.layers)),
                       key=lambda i: -(self.layers[i].param_bytes / (self._stall(i) + 1e-9)))
        for i in order:
            if self._peak(off) <= self.budget:
                break
            off.add(i)
        if self._peak(off) > self.budget:
            raise RuntimeError(f"offload: even with every layer on the host the peak is {self._peak(off):.3g} B "
                               f"> budget {self.budget:.3g} B")
        plan = OffloadPlan(peak_param_bytes=self._peak(off))
        for i in sorted(off):
            name = self.layers[i].name
            plan.offloaded.append(name)
            j = max(0, i - self.distance) if self.asynchronous else i
            plan.prefetch_at[name] = self.layers[j].name
            plan.est_stall_s += self._stall(i)
        return plan


class AsynGreedySolver(SynGreedySolver):
    asynchronous = True


class _OffloadRuntime:
    """Holds the pinned host copies and does the fetch / release; on CPU-only hosts the copies are plain tensors and the
    'device' is the CPU (the hook order and accounting are still exercised)."""

    def __init__(self, device: torch.device) -> None:
        self.device = device
        self.stream = torch.cuda.Stream() if device.type == "cuda" else None
        self.host: Dict[nn.Parameter, torch.Tensor] = {}
        self.events: Dict[str, "torch.cuda.Event"] = {}
        self.resident_log: List[str] = []

    def offload(self, mod: nn.Module) -> None:
        for p in mod.parameters(recurse=True):
            h = p.data.detach().to("cpu")
            if self.device.type == "cuda":
                h = h.pin_memory()
            self.host[p] = h
            p.data = torch.empty(0, dtype=p.dtype, device=self.device)

    def fetch(self, name: str, mod: nn.Module, asynchronous: bool) -> None:
        if any(p in self.host and p.data.numel() == 0 for p in mod.parameters()):
            if self.stream is not None and asynchronous:
                with torch.cuda.stream(self.stream):
                    for p in mod.parameters():
                        if p in self.host and p.data.numel() == 0:
                            p.data = self.host[p].to(self.device, non_blocking=True)
                    ev = torch.cuda.Event()
                    ev.record(self.stream)
                    self.events[name] = ev
            else:
                for p in mod.parameters():
                    if p in self.host and p.data.numel() == 0:
                        p.data = self.host[p].to(self.device)
            self.resident_log.append(f"fetch:{name}")

    def wait(self, name: str) -> None:
        ev = self.events.pop(name, None)
        if ev is not None:
            torch.cuda.current_stream().wait_event(ev)

    def release(self, name: str, mod: nn.Module) -> None:
        for p in mod.parameters():
            if p in self.host:
                if p.grad is None and not torch.is_grad_enabled():
                    pass
                p.data = torch.empty(0, dtype=p.dtype, device=self.device)
        self.resident_log.append(f"release:{name}")


def memory_optimize(model: nn.Module, budget_bytes: float, layers: Optional[Sequence[str]] = None,
                    solver_name: str = "asyn", bandwidth: float = 50e9, prefetch_distance: int = 1,
                    flops_per_s: float = 1.0e15):
    """Plan + install hooks.  `layers`: names of the sequentially executed blocks (default: the children of the
    longest `nn.ModuleList`).  Inference / forward-only release is exact; during training parameters are kept
    resident from their forward to their backward (released by a full-backward hook)."""
    named = dict(model.named_modules())
    if layers is None:
        lists = [(n, m) for n, m in named.items() if isinstance(m, (nn.ModuleList, nn.Sequential)) and len(m) > 0]
        assert lists, "pass `layers=` for models without a ModuleList of blocks"
        base, ml = max(lists, key=lambda kv: len(kv[1]))
        layers = [f"{base}.{i}" if base else str(i) for i in range(len(ml))]
    costs = []
    for n in layers:
        m = named[n]
        pb = float(sum(p.numel() * p.element_size() for p in m.parameters()))
        costs.append(LayerCost(n, pb, 2.0 * sum(p.numel() for p in m.parameters()) / flops_per_s))
    fixed = float(sum(p.numel() * p.element_size() for p in model.parameters())) - sum(c.param_bytes for c in costs)
    cls = AsynGreedySolver if solver_name.startswith("asyn") else SynGreedySolver
    plan = cls(costs, budget_bytes - fixed, bandwidth, prefetch_distance).solve()
    dev = next(model.parameters()).device
    rt = _OffloadRuntime(dev)
    off = set(plan.offloaded)
    starters: Dict[str, List[str]] = {}
    for name, at in plan.prefetch_at.items():
        starters.setdefault(at, []).append(name)
    for n in layers:
        m = named[n]
        if n in off:
            rt.offload(m)

        def pre(mod, args, n=n):
            for tgt in starters.get(n, []):
                rt.fetch(tgt, named[tgt], asynchronous=cls.asynchronous and tgt != n)
            if n in off:
                rt.fetch(n, mod, asynchronous=False)       # no-op when the prefetch already ran
                rt.wait(n)

        def post(mod, args, out, n=n):
            if n in off and not (torch.is_grad_enabled() and any(p.requires_grad for p in mod.parameters())):
                rt.release(n, mod)

        m.register_forward_pre_hook(pre)
        m.register_forward_hook(post)
        if n in off:
            def bwd_pre(mod, gout, n=n):
                rt.fetch(n, mod, asynchronous=False)

            def bwd_post(mod, gin, gout, n=n):
                rt.release(n, mod)

            m.register_full_backward_pre_hook(bwd_pre)
            m.register_full_backward_hook(bwd_post)
    model._offload_runtime, model._offload_plan = rt, plan
    return model, plan
