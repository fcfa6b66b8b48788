"""Sparse Mixture-of-Experts block with expert parallelism (Mixtral / DeepSeekMoE / DeepSeek-V3 routing).

Parity: reference `EPMixtralSparseMoeBlock` (`colossalai/shardformer/modeling/mixtral.py:54-208`), `EPDeepseekMoE`
(`deepseek.py:63-230`), `EpDeepseekV3MoE` (`deepseek_v3.py:26`).  Differences (H100-first):
  * expert weights are batched tensors `[E_local, 2I, H]` / `[E_local, H, I]` driven by ONE grouped GEMM per
    projection instead of a python loop of small GEMMs;
  * dispatch/combine go through `colossalai_b200.moe` which has two backends: `nccl` (sorted tokens + uneven
    all-to-all; sizes exchanged on device, one host sync for the split sizes) and `fused` (router top-k -> direct
    remote row stores into per-expert symmetric buffers, no host sync);
  * load-balancing aux loss and router z-loss are accumulated on the module (`aux_loss`).
"""
from __future__ import annotations

import math
from typing import Optional, Tuple

import torch
import torch.nn as nn
import torch.nn.functional as F

from .. import ops
from ..parallel import comm
from ..tensor.moe_tensor import set_moe_tensor_ep_group
from .config import ModelConfig

__all__ = ["SparseMoE", "Router", "GroupedExperts"]


class Router(nn.Module):
    def __init__(self, cfg: ModelConfig) -> None:
        super().__init__()
        self.cfg = cfg
        m = cfg.moe
        self.gate = nn.Linear(cfg.hidden_size, m.num_experts, bias=False)
        if m.scoring_func == "sigmoid":
            self.e_score_correction_bias = nn.Parameter(torch.zeros(m.num_experts), requires_grad=False)

    def forward(self, x: torch.Tensor) -> Tuple[torch.Tensor, torch.Tensor, torch.Tensor]:
        """x [T, H] -> (topk weights [T, k] fp32, topk expert ids [T, k] int64, router logits [T, E] fp32)."""
        m = self.cfg.moe
        logits = F.linear(x.float(), self.gate.weight.float())
        if m.scoring_func == "softmax":
            scores = logits.softmax(dim=-1)
            w, idx = scores.topk(m.top_k, dim=-1)
        else:  # DeepSeek-V3 sigmoid scoring + group-limited top-k
            scores = logits.sigmoid()
            choice = scores + self.e_score_correction_bias
            if m.n_group > 1:
                T = x.shape[0]
                g = choice.view(T, m.n_group, -1)
                group_scores = g.topk(2, dim=-1)[0].sum(-1)
                gidx = group_scores.topk(m.topk_group, dim=-1)[1]
                gmask = torch.zeros_like(group_scores).scatter_(1, gidx, 1.0)
                choice = (g * gmask.unsqueeze(-1)).view(T, -1).masked_fill(
                    (gmask.unsqueeze(-1).expand_as(g) == 0).reshape(T, -1), float("-inf"))
            idx = choice.topk(m.top_k, dim=-1)[1]
            w = scores.gather(1, idx)
        if m.norm_topk_prob:
            w = w / (w.sum(-1, keepdim=True) + 1e-20)
        w = w * m.routed_scaling_factor
        return w, idx, logits


class GroupedExperts(nn.Module):
    """E_local experts stored as batched weights; forward runs on tokens grouped (sorted) by local expert."""

    def __init__(self, cfg: ModelConfig, num_local_experts: int, intermediate: int) -> None:
        super().__init__()
        self.cfg, self.num_local_experts, self.intermediate = cfg, num_local_experts, intermediate
        H = cfg.hidden_size
        up_out = 2 * intermediate if cfg.glu else intermediate
        self.w_up = nn.Parameter(torch.empty(num_local_experts, up_out, H))      # gate|up fused
        self.w_down = nn.Parameter(torch.empty(num_local_experts, H, intermediate))
        nn.init.normal_(self.w_up, std=cfg.initializer_range)        # (on meta: recorded by the lazy-init log only)
        nn.init.normal_(self.w_down, std=cfg.initializer_range)

    def forward(self, x_sorted: torch.Tensor, counts: torch.Tensor) -> torch.Tensor:
        """x_sorted [N, H] rows grouped by local expert; counts [E_local] rows per expert."""
        from ..moe.grouped_gemm import grouped_linear

        h = grouped_linear(x_sorted, self.w_up, counts)
        # rows past sum(counts) are padding of an over-allocated receive buffer: the activation skips them (the count
        # stays on the device)
        h = ops.glu(h, self.cfg.hidden_act, valid_rows=counts.sum()) if self.cfg.glu \
            else ops.get_activation(self.cfg.hidden_act)(h)
        return grouped_linear(h, self.w_down, counts)


class SparseMoE(nn.Module):
    def __init__(self, cfg: ModelConfig) -> None:
        super().__init__()
        self.cfg = cfg
        m = cfg.moe
        self.num_experts, self.top_k = m.num_experts, m.top_k
        inter = m.moe_intermediate_size or cfg.intermediate_size
        self.router = Router(cfg)
        self.experts = GroupedExperts(cfg, m.num_experts, inter)
        if m.n_shared_experts > 0:
            from .transformer import MLP

            self.shared_experts = MLP(cfg, intermediate_size=inter * m.n_shared_experts)
        self.shard_config = None
        self.ep_group = None
        self.ep_size, self.ep_rank = 1, 0
        self.aux_loss: Optional[torch.Tensor] = None

    # called by the policy
    def setup_parallel(self, shard_config) -> None:
        ep_group = shard_config.ep_group
        self.ep_group = ep_group
        # no ep group configured = experts are replicated (plain data / tensor parallel run), NOT "the world"
        self.ep_size = comm.group_size(ep_group) if ep_group is not None else 1
        self.ep_rank = comm.group_rank(ep_group) if ep_group is not None else 0
        if self.ep_size > 1:
            assert self.num_experts % self.ep_size == 0
            n_local = self.num_experts // self.ep_size
            s = self.ep_rank * n_local
            ex = self.experts
            if ex.w_up.shape[0] == self.num_experts:   # slice the held experts
                if ex.w_up.device.type == "meta":
                    up = torch.empty((n_local,) + tuple(ex.w_up.shape[1:]), device="meta", dtype=ex.w_up.dtype)
                    down = torch.empty((n_local,) + tuple(ex.w_down.shape[1:]), device="meta", dtype=ex.w_down.dtype)
                    from ..lazy import copy_lazy_ops

                    new_up, new_down = nn.Parameter(up), nn.Parameter(down)
                    copy_lazy_ops(ex.w_up, new_up)
                    copy_lazy_ops(ex.w_down, new_down)
                    ex.w_up, ex.w_down = new_up, new_down
                else:
                    ex.w_up = nn.Parameter(ex.w_up.data[s:s + n_local].clone())
                    ex.w_down = nn.Parameter(ex.w_down.data[s:s + n_local].clone())
                ex.num_local_experts = n_local
        # Megatron-style sequence parallelism: the block sees only this rank's sequence shard, so the gradients of its
        # replicated (non-TP, non-EP) parameters are partial sums -> all-reduced over the tp group with the norm grads
        sp_mode = getattr(shard_config, "sp_mode", None)
        if sp_mode in ("split_gather", "ring") and getattr(shard_config, "sequence_parallel_size", 1) > 1:
            from ..tensor.d_tensor import is_distributed_tensor

            for name, p in self.named_parameters():
                if is_distributed_tensor(p) or (self.ep_size > 1 and name.startswith("experts.")):
                    continue
                p.partial_derived = True
        for p in self.experts.parameters():
            set_moe_tensor_ep_group(p, ep_group, getattr(shard_config, "moe_dp_group", None))
            if self.ep_size > 1:
                from ..tensor.d_tensor.api import mark_sharded

                mark_sharded(p, 0, ep_group)      # checkpoint IO gathers / re-shards experts like any other shard

    def _aux(self, logits: torch.Tensor, idx: torch.Tensor) -> torch.Tensor:
        m = self.cfg.moe
        T, E = logits.shape
        probs = logits.softmax(-1) if m.scoring_func == "softmax" else logits.sigmoid()
        frac_tokens = torch.zeros(E, device=logits.device, dtype=torch.float32)
        frac_tokens.scatter_add_(0, idx.reshape(-1), torch.ones(idx.numel(), device=logits.device))
        frac_tokens = frac_tokens / max(idx.numel(), 1)
        aux = E * (frac_tokens * probs.mean(0)).sum() * m.router_aux_loss_coef
        if m.router_z_loss_coef > 0:
            aux = aux + m.router_z_loss_coef * torch.logsumexp(logits, -1).pow(2).mean()
        return aux

    def forward(self, x: torch.Tensor) -> torch.Tensor:
        from ..moe import dispatch_combine

        shape = x.shape
        x2 = x.reshape(-1, shape[-1])
        w, idx, logits = self.router(x2)
        if self.training:
            self.aux_loss = self._aux(logits, idx)
        out = dispatch_combine.moe_forward(x2, w, idx, self.experts, self.num_experts, self.ep_group)
        if hasattr(self, "shared_experts"):
            out = out + self.shared_experts(x2)
        return out.reshape(shape)
