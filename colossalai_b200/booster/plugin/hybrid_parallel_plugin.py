"""HybridParallelPlugin: TP x PP x SP x DP(ZeRO) on one named device mesh.

Parity: reference `colossalai/booster/plugin/hybrid_parallel_plugin.py:59-1529` (`HybridParallelModule`,
`HybridParallel{Naive,AMP,Zero}Optimizer`, `HybridParallelPlugin.__init__/configure/execute_pipeline`, grad-norm
reduction over tp/pp, tied-embedding / SP-partial / DP gradient syncs, dataloader with DistributedSampler over dp).
Additions: `comm_backend="fused"` routes TP/SP linears through the fused compute+collective kernels; the AMP
optimizer runs the single-launch fused Adam (see amp/naive_amp/mixed_precision_optimizer.py).
"""
from __future__ import annotations

import ctypes
import random
from contextlib import contextmanager, nullcontext
from functools import partial
from types import MethodType
from typing import Any, Callable, Dict, Iterator, List, Optional, OrderedDict, Tuple, Union

import numpy as np
import torch
import torch.distributed as dist
import torch.nn as nn
from torch import Tensor, inf
from torch.distributed import ProcessGroup
from torch.nn import Module
from torch.optim import Optimizer
from torch.optim.lr_scheduler import _LRScheduler as LRScheduler
from torch.utils.data import DataLoader
from torch.utils.data.distributed import DistributedSampler

from ...accelerator import get_accelerator
from ...amp.naive_amp.mixed_precision_optimizer import MixedPrecisionOptimizer
from ...checkpoint_io import CheckpointIO
from ...cluster import DeviceMesh
from ...interface import AMPModelMixin, ModelWrapper, OptimizerWrapper
from ...logging import get_dist_logger
from ...parallel import comm
from ...pipeline.stage_manager import PipelineStageManager
from ...shardformer import GradientCheckpointConfig, ShardConfig, ShardFormer
from ...shardformer.layer._operation import set_comm_backend
from ...shardformer.layer.utils import SeqParallelUtils
from ...shardformer.policies.base_policy import Policy
from ...tensor.d_tensor import is_distributed_tensor
from ...tensor.moe_tensor import get_ep_group, is_moe_tensor
from .plugin_base import PipelinePluginBase, _seed_worker

__all__ = ["HybridParallelPlugin", "HybridParallelModule", "HybridParallelNaiveOptimizer",
           "HybridParallelAMPOptimizer", "HybridParallelZeroOptimizer", "get_param_info"]

PRECISION_TORCH_TYPE = {"fp16": torch.float16, "fp32": torch.float32, "bf16": torch.bfloat16}
SUPPORT_SP_MODE = ["split_gather", "ring", "all_to_all", "ring_attn"]


def _convert_floating_point(x, dtype: torch.dtype = torch.float16):
    if isinstance(x, torch.Tensor) and torch.is_floating_point(x):
        return x.to(dtype)
    return x


def _tree_map(fn, obj):
    if isinstance(obj, dict):
        return {k: _tree_map(fn, v) for k, v in obj.items()}
    if isinstance(obj, (list, tuple)):
        return type(obj)(_tree_map(fn, v) for v in obj)
    return fn(obj)


def _bucketed_all_reduce(grads: List[Tensor], group: ProcessGroup, average_by: int, bucket_bytes: int = 64 << 20):
    """Flatten -> all_reduce -> unflatten in buckets (keeps launch count and NCCL latency low)."""
    if not grads:
        return
    by_dtype: Dict[torch.dtype, List[Tensor]] = {}
    for g in grads:
        by_dtype.setdefault(g.dtype, []).append(g)
    for dtype, gs in by_dtype.items():
        bucket, size = [], 0
        def flush():
            nonlocal bucket, size
            if not bucket:
                return
            flat = torch.cat([g.reshape(-1) for g in bucket])
            if average_by > 1:
                flat.div_(average_by)
            dist.all_reduce(flat, group=group)
            off = 0
            for g in bucket:
                n = g.numel()
                g.copy_(flat[off:off + n].view_as(g))
                off += n
            bucket, size = [], 0
        for g in gs:
            bucket.append(g)
            size += g.numel() * g.element_size()
            if size >= bucket_bytes:
                flush()
        flush()


class HybridParallelModule(ModelWrapper, AMPModelMixin):
    def __init__(self, module: Module, precision: str, shard_config: ShardConfig, dp_group: ProcessGroup,
                 tp_group: ProcessGroup, sp_group: ProcessGroup, use_ddp: bool, ddp_config: dict,
                 custom_policy: Policy, overlap_allgather: bool = False, use_fp8: bool = False,
                 inplace_wgrad: bool = False) -> None:
        self.stage_manager = shard_config.pipeline_stage_manager
        self.shard_config = shard_config
        self.dp_group, self.tp_group, self.sp_group = dp_group, tp_group, sp_group
        self.use_ddp = use_ddp
        self.require_grad_sync = True
        self.overlap_allgather = overlap_allgather
        self.use_fp8 = use_fp8
        shardformer = ShardFormer(shard_config)
        if custom_policy is not None:
            assert isinstance(custom_policy, object)
        module, self.shared_params = shardformer.optimize(module, policy=custom_policy)
        # tied parameters across pipeline stages: a group per tie
        self.shared_param_process_groups = []
        for shared in self.shared_params:
            if len(shared) > 0:
                self.shared_param_process_groups.append(
                    self.stage_manager.init_process_group_by_stages(list(shared.keys())))
        # precision + device
        self.mixed_precision = None
        if precision in ("fp16", "bf16"):
            self.mixed_precision = PRECISION_TORCH_TYPE[precision]
            module = module.to(self.mixed_precision)
        module = module.to(get_accelerator().get_current_device())
        self.dp_size = comm.group_size(dp_group) if dp_group is not None else 1
        super().__init__(module)
        if use_fp8:
            from ...quantization.fp8_hook import convert_linear_to_fp8

            convert_linear_to_fp8(self.module)
        elif inplace_wgrad:
            self._enable_inplace_wgrad()

    def _enable_inplace_wgrad(self) -> None:
        """Gradient accumulation inside the wgrad GEMM epilogue (`grad += dY^T X` with beta = 1): plain `nn.Linear`s
        are routed through our autograd function, every 2-D linear weight is flagged (see `_accumulate_wgrad`)."""
        from ...shardformer.layer._operation import linear_with_grad_accum

        def fwd(mod, x):
            return linear_with_grad_accum(x, mod.weight, mod.bias)

        for m in self.module.modules():
            w = getattr(m, "weight", None)
            if not isinstance(w, nn.Parameter) or w.dim() != 2 or isinstance(m, nn.Embedding):
                continue
            if type(m) is nn.Linear:
                m.forward = MethodType(fwd, m)
            w._cb200_inplace_wgrad = True

    # ------------------------------------------------------------------ grad syncs
    def sync_shared_params(self) -> None:
        for shared, group in zip(self.shared_params, self.shared_param_process_groups):
            if self.stage_manager.stage in shared:
                p = shared[self.stage_manager.stage]
                if p.grad is not None:
                    dist.all_reduce(p.grad, group=group)

    @contextmanager
    def no_sync(self):
        old = self.require_grad_sync
        self.require_grad_sync = False
        try:
            yield
        finally:
            self.require_grad_sync = old

    def sync_dp_grads(self) -> None:
        """Average gradients over the data-parallel group (dense params) — bucketed all-reduce."""
        if self.dp_group is None or self.dp_size == 1 or not self.require_grad_sync:
            return
        grads = [p.grad for p in self.module.parameters() if p.grad is not None and not is_moe_tensor(p)]
        _bucketed_all_reduce(grads, self.dp_group, self.dp_size)
        moe_dp_group = getattr(self, "moe_dp_group", None)
        if moe_dp_group is not None and comm.group_size(moe_dp_group) > 1:
            mg = [p.grad for p in self.module.parameters() if p.grad is not None and is_moe_tensor(p)]
            _bucketed_all_reduce(mg, moe_dp_group, comm.group_size(moe_dp_group))

    def sync_sp_grads(self, grads: Optional[List[Tensor]] = None) -> None:
        """all_to_all / ring_attn: params are replicated over sp -> grads are averaged with dp (handled by using the
        dp x sp group as `dp_group`).  split_gather / ring: all-reduce the sp-partial (norm / bias) grads over tp."""
        sc = self.shard_config
        if sc.sp_mode in ("split_gather", "ring") and sc.sequence_parallel_size > 1 and self.require_grad_sync:
            if grads is not None:
                SeqParallelUtils.allreduce_partial_data_grad(process_group=self.tp_group, grads=grads)
            else:
                SeqParallelUtils.allreduce_partial_data_grad(process_group=self.tp_group, model=self.module)

    def forward(self, *args, **kwargs):
        if self.mixed_precision is not None:
            cast = partial(_convert_floating_point, dtype=self.mixed_precision)
            args = _tree_map(cast, args)
            kwargs = _tree_map(cast, kwargs)
        return super().forward(*args, **kwargs)

    def unwrap(self, unwrap_peft: bool = True):
        return self.module


def get_param_info(optim: Optimizer, model: Optional[Module] = None) -> Dict:
    """Snapshot param ids/shapes before boosting (checkpoint IO needs the original layout to re-shard states).  With
    `model`, also the NAME of every optimizer parameter per group: sharding replaces the parameter tensors, and the
    names are what ties a user's param groups (decay / no-decay, per-layer lr, ...) to the new tensors."""
    if optim is None:
        return {}
    info = {"param_groups": [], "param2id": {}, "id2param": {}, "param2shape": {}}
    if model is not None:
        inner = model.unwrap() if isinstance(model, ModelWrapper) else model
        name_of = {id(p): n for n, p in inner.named_parameters()}
        if all(id(p) in name_of for g in optim.param_groups for p in g["params"]):
            info["group_names"] = [[name_of[id(p)] for p in g["params"]] for g in optim.param_groups]
            # tied parameters: every alias path -> the canonical name (a pipeline stage may only keep the alias, e.g. the
            # last stage owns `lm_head.weight` of a model whose head is tied to the embedding)
            info["alias_of"] = {n: name_of[id(p)] for n, p in inner.named_parameters(remove_duplicate=False)}
    start = 0
    for group in optim.param_groups:
        packed = {k: v for k, v in group.items() if k != "params"}
        packed["params"] = []
        for pid, p in enumerate(group["params"], start):
            packed["params"].append(pid)
            info["param2id"][id(p)] = pid
            info["id2param"][pid] = id(p)
            info["param2shape"][id(p)] = tuple(p.shape)
        info["param_groups"].append(packed)
        start += len(group["params"])
    return info


def _reassign_params(optim: Optimizer, model: Module, param_info: Optional[Dict] = None) -> None:
    """After sharding, model parameters are NEW tensors: point the optimizer at them, group by group."""
    names = (param_info or {}).get("group_names")
    if names is not None and len(names) == len(optim.param_groups):
        inner = model.unwrap() if isinstance(model, ModelWrapper) else model
        new = {n: p for n, p in inner.named_parameters() if p is not None}
        taken = set()
        for g, ns in zip(optim.param_groups, names):
            g["params"] = [new[n] for n in ns if n in new and new[n].requires_grad]     # PP stages drop some names
            taken.update(id(p) for p in g["params"])
        # aliases of tied parameters that survive on this stage under their other name join their partner's group;
        # parameters the user deliberately left out of the optimizer stay out
        alias_of = (param_info or {}).get("alias_of", {})
        group_of = {n: gi for gi, ns in enumerate(names) for n in ns}
        for n, p in new.items():
            if id(p) in taken or not p.requires_grad:
                continue
            canon = alias_of.get(n)
            if canon is not None and canon in group_of:
                optim.param_groups[group_of[canon]]["params"].append(p)
                taken.add(id(p))
        optim.state.clear()
        return
    model_params = set(id(p) for p in model.parameters())
    new_groups = []
    # rebuild in model order; every group's hyper-params are preserved, params matched by position in the model
    all_params = [p for p in model.parameters() if p.requires_grad]
    if len(optim.param_groups) == 1:
        optim.param_groups[0]["params"] = all_params
    else:
        # multiple groups: keep membership by original index order
        counts = [len(g["params"]) for g in optim.param_groups]
        if sum(counts) == len(all_params):
            off = 0
            for g, c in zip(optim.param_groups, counts):
                g["params"] = all_params[off:off + c]
                off += c
        else:
            # PP dropped some params: keep only params still in the model
            for g in optim.param_groups:
                g["params"] = [p for p in g["params"] if id(p) in model_params]
            known = set(id(p) for g in optim.param_groups for p in g["params"])
            rest = [p for p in all_params if id(p) not in known]
            if rest:
                optim.param_groups[0]["params"].extend(rest)
    optim.state.clear()


class _HybridNormMixin:
    """Grad-norm over a (tp, pp)-sharded model: TP-sharded params are summed over tp, replicated params counted
    once; then summed over pp (reference `hybrid_parallel_plugin.py:380-456`)."""

    tp_pg: Optional[ProcessGroup]
    pp_pg: Optional[ProcessGroup]
    tp_size: int
    pp_size: int
    shared_params: List

    def _hybrid_norm_sq(self, params: List[nn.Parameter], local_norm_fn) -> Tensor:
        sharded, replicated = [], []
        shared_ids = set()
        if getattr(self, "stage_manager", None) is not None:
            for shared in self.shared_params:
                # count a tied param only on its first stage
                stages = sorted(shared.keys())
                for s in stages[1:]:
                    shared_ids.add(id(shared[s]))
        moe = []
        for p in params:
            if id(p) in shared_ids:
                continue
            if is_moe_tensor(p):
                moe.append(p)       # expert-parallel shards: summed over the ep group
                continue
            (sharded if (self.tp_size > 1 and is_distributed_tensor(p)) else replicated).append(p)
        n_sh = local_norm_fn(sharded)
        n_rep = local_norm_fn(replicated)
        if self.tp_size > 1:
            dist.all_reduce(n_sh, group=self.tp_pg)
        total = n_sh + n_rep
        if moe:
            n_moe = local_norm_fn(moe)
            ep_group = get_ep_group(moe[0])
            if ep_group is not None and comm.group_size(ep_group) > 1:
                dist.all_reduce(n_moe, group=ep_group)
            total = total + n_moe
        if self.pp_size > 1:
            dist.all_reduce(total, group=self.pp_pg)
        return total


class HybridParallelNaiveOptimizer(OptimizerWrapper, _HybridNormMixin):
    """fp32 training (no master copy)."""

    def __init__(self, optim: Optimizer, model: HybridParallelModule, use_pipeline: bool, param_info: Dict,
                 max_norm: float = 0, tp_process_group: Optional[ProcessGroup] = None,
                 pp_process_group: Optional[ProcessGroup] = None) -> None:
        self.param_info = param_info
        _reassign_params(optim, model, param_info)
        self.model = model
        self.stage_manager = model.stage_manager
        self.shared_params = model.shared_params
        self.max_norm = max_norm
        self.tp_pg, self.pp_pg = tp_process_group, pp_process_group
        self.tp_size = comm.group_size(tp_process_group) if tp_process_group is not None else 1
        self.pp_size = comm.group_size(pp_process_group) if pp_process_group is not None else 1
        super().__init__(optim)

    def backward(self, loss: Tensor, inputs=None, retain_graph: bool = False, **kwargs):
        super().backward(loss, inputs=inputs, retain_graph=retain_graph, **kwargs)
        if self.model.require_grad_sync:
            self.model.sync_sp_grads()

    def backward_by_grad(self, tensor: Tensor, grad: Tensor, inputs=None, retain_graph: bool = False):
        super().backward_by_grad(tensor, grad, inputs=inputs, retain_graph=retain_graph)
        if self.model.require_grad_sync:
            self.model.sync_sp_grads()

    def step(self, *args, **kwargs):
        if self.max_norm > 0:
            params = [p for g in self.optim.param_groups for p in g["params"] if p.grad is not None]
            norm_sq = self._hybrid_norm_sq(
                params, lambda ps: (torch.stack([p.grad.float().pow(2).sum() for p in ps]).sum().reshape(1)
                                    if ps else torch.zeros(1, device=get_accelerator().get_current_device())))
            total = norm_sq.sqrt()
            self._current_grad_norm = float(total.item())
            coef = (self.max_norm / (total + 1e-6)).clamp(max=1.0)
            for p in params:
                p.grad.mul_(coef.to(p.grad.dtype))
        self.optim.step(*args, **kwargs)

    def update_master_params(self, model: Module):
        pass

    def get_working_to_master_map(self):
        return None

    def get_master_to_working_map(self):
        return None


class HybridParallelAMPOptimizer(MixedPrecisionOptimizer, _HybridNormMixin):
    """bf16/fp16 working params + fp32 master (fused single-launch Adam)."""

    def __init__(self, optim: Optimizer, model: HybridParallelModule, use_pipeline: bool, param_info: Dict,
                 precision: str = "fp16", initial_scale: float = 2**16, min_scale: float = 1,
                 growth_factor: float = 2, backoff_factor: float = 0.5, growth_interval: int = 1000,
                 hysteresis: int = 2, max_scale: float = 2**32, max_norm: float = 0,
                 tp_process_group: Optional[ProcessGroup] = None, pp_process_group: Optional[ProcessGroup] = None) -> None:
        self.model = model
        self.param_info = param_info
        self.stage_manager = model.stage_manager
        self.shared_params = model.shared_params
        self.tp_pg, self.pp_pg = tp_process_group, pp_process_group
        self.tp_size = comm.group_size(tp_process_group) if tp_process_group is not None else 1
        self.pp_size = comm.group_size(pp_process_group) if pp_process_group is not None else 1
        _reassign_params(optim, model, param_info)
        super().__init__(optim, model, precision=precision, initial_scale=initial_scale, min_scale=min_scale,
                         growth_factor=growth_factor, backoff_factor=backoff_factor, growth_interval=growth_interval,
                         hysteresis=hysteresis, max_scale=max_scale, max_norm=max_norm)

    def backward(self, loss: Tensor, inputs=None, retain_graph: bool = False, **kwargs):
        super().backward(loss, inputs=inputs, retain_graph=retain_graph, **kwargs)
        if self.model.require_grad_sync:
            self.model.sync_sp_grads()

    def backward_by_grad(self, tensor: Tensor, grad: Tensor, inputs=None, retain_graph: bool = False):
        super().backward_by_grad(tensor, grad, inputs=inputs, retain_graph=retain_graph)
        if self.model.require_grad_sync:
            self.model.sync_sp_grads()

    def _compute_grad_norm_sq(self, params: List[nn.Parameter]) -> Tensor:
        return self._hybrid_norm_sq(params, self._local_grad_norm_sq)


class HybridParallelPlugin(PipelinePluginBase):
    """
    >>> plugin = HybridParallelPlugin(tp_size=8, pp_size=1, enable_sequence_parallelism=True,
    ...                               sequence_parallelism_mode="split_gather", precision="bf16", comm_backend="fused")
    >>> booster = Booster(plugin=plugin)
    >>> model, optimizer, criterion, dataloader, _ = booster.boost(model, optimizer, criterion, dataloader)
    """

    materializes_lazy_models = True      # ShardFormer materialises lazily built models after sharding

    def __init__(self, tp_size: int, pp_size: int, sp_size: int = None, precision: str = "fp16", zero_stage: int = 0,
                 enable_all_optimization: bool = False, enable_fused_normalization: bool = False,
                 enable_flash_attention: bool = False, enable_jit_fused: bool = False,
                 enable_sequence_parallelism: bool = False, sequence_parallelism_mode: str = None,
                 parallel_output: bool = True, num_microbatches: Optional[int] = None,
                 microbatch_size: Optional[int] = None, initial_scale: float = 2**16, min_scale: float = 1,
                 growth_factor: float = 2, backoff_factor: float = 0.5, growth_interval: int = 1000,
                 hysteresis: int = 2, max_scale: float = 2**32, max_norm: float = 0, broadcast_buffers: bool = True,
                 ddp_bucket_cap_mb: int = 25, find_unused_parameters: bool = False, check_reduction: bool = False,
                 gradient_as_bucket_view: bool = False, static_graph: bool = False, zero_bucket_size_in_m: int = 12,
                 cpu_offload: bool = False, offload_optim_frac: float = 1.0,
                 communication_dtype: Optional[torch.dtype] = None,
                 overlap_communication: bool = True, custom_policy: Policy = None, pp_style: str = "1f1b",
                 num_model_chunks: int = 1, scheduler_nodes: List = None, num_layers_per_stage: Optional[List[int]] = None,
                 gradient_checkpoint_config: Optional[GradientCheckpointConfig] = None,
                 enable_metadata_cache: bool = True, make_vocab_size_divisible_by: int = 64, dp_outside: bool = True,
                 overlap_p2p: bool = True, overlap_allgather: bool = False, fp8_communication: bool = False,
                 use_fp8: bool = False, inner_ring_size: int = None, comm_backend: str = "nccl") -> None:
        super().__init__()
        self.logger = get_dist_logger()
        assert dist.is_initialized(), "call colossalai_b200.launch* before creating a plugin"
        world = dist.get_world_size()
        assert world % (tp_size * pp_size) == 0, (
            f"world size {world} is not divisible by tp_size {tp_size} * pp_size {pp_size}")
        assert precision in PRECISION_TORCH_TYPE, f"precision must be one of {list(PRECISION_TORCH_TYPE)}"
        if enable_sequence_parallelism:
            self.sequence_parallelism_mode = sequence_parallelism_mode or "all_to_all"
            assert self.sequence_parallelism_mode in SUPPORT_SP_MODE, (
                f"Sequence parallelism mode {self.sequence_parallelism_mode} is not in the supported list {SUPPORT_SP_MODE}")
            if self.sequence_parallelism_mode in ("split_gather", "ring"):
                assert tp_size > 1, (
                    f"Sequence parallelism mode {self.sequence_parallelism_mode} must be enabled when using tensor parallelism")
                if sp_size not in (None, 1, tp_size):
                    self.logger.warning(f"sp_size is forced to the tp group for mode {self.sequence_parallelism_mode}",
                                        ranks=[0])
                self.sp_size = 1
                self.dp_size = world // (tp_size * pp_size)
            else:
                self.sp_size = 1 if sp_size is None else sp_size
                self.dp_size = world // (self.sp_size * pp_size * tp_size)
                if self.sequence_parallelism_mode == "ring_attn":
                    enable_flash_attention = True
        else:
            self.sequence_parallelism_mode = None
            self.dp_size = world // (tp_size * pp_size)
            assert sp_size is None or sp_size == 1, (
                f"You should not set sp_size when sequence parallelism is not enabled.")
            self.sp_size = 1
        assert self.dp_size * tp_size * pp_size * self.sp_size == world, (
            f"dp {self.dp_size} x pp {pp_size} x tp {tp_size} x sp {self.sp_size} != world {world}")
        self.tp_size, self.pp_size = tp_size, pp_size
        self.precision, self.zero_stage = precision, zero_stage
        self.cpu_offload = cpu_offload
        # with cpu_offload: fraction of the optimizer state kept in pinned host memory (tiering between HBM and
        # DRAM that composes with TP x PP - the reference only has Gemini's tiering without PP, or all-or-nothing ZeRO
        # offload: `hybrid_parallel_plugin.py:666-719`)
        self.offload_optim_frac = offload_optim_frac
        self.enable_all_optimization = enable_all_optimization
        self.enable_fused_normalization = enable_fused_normalization
        self.enable_flash_attention = enable_flash_attention
        self.enable_jit_fused = enable_jit_fused
        self.enable_sequence_parallelism = enable_sequence_parallelism
        self.use_fp8, self.fp8_communication = use_fp8, fp8_communication
        self.custom_policy = custom_policy
        self.comm_backend = comm_backend
        self.pp_style = pp_style
        # ---- mesh.  order: ring_attn puts sp outside tp; dp_outside toggles dp vs pp outermost
        if self.sequence_parallelism_mode == "ring_attn":
            order = ("dp", "pp", "sp", "tp") if dp_outside else ("pp", "dp", "sp", "tp")
        else:
            order = ("dp", "pp", "tp", "sp") if dp_outside else ("pp", "dp", "tp", "sp")
        sizes = dict(dp=self.dp_size, pp=pp_size, tp=tp_size, sp=self.sp_size)
        self.pg_mesh = DeviceMesh(**{k: sizes[k] for k in order})
        self.dp_axis, self.pp_axis = self.pg_mesh.axis("dp"), self.pg_mesh.axis("pp")
        self.tp_axis, self.sp_axis = self.pg_mesh.axis("tp"), self.pg_mesh.axis("sp")
        # ---- pipeline
        self.stage_manager = None
        self.scheduler = None
        self.schedule = None
        assert zero_stage in (0, 1, 2)
        if pp_size > 1:
            assert pp_style in ("1f1b", "interleaved", "zbv"), "Unsupported pipeline parallelism style"
            assert pp_style in ("interleaved", "zbv") or num_model_chunks == 1, (
                "num_model_chunks must be 1 when using 1f1b")
            assert pp_style != "zbv" or num_model_chunks == 2, "num_model_chunks must be 2 when using zero bubble pipeline"
            assert num_microbatches is not None or microbatch_size is not None, (
                "num_microbatches or microbatch_size must be specified when using pipeline parallelism")
            assert zero_stage <= 1, "To avoid prohibitive gradient synchronization costs, zero stage must be 0 or 1 when using pipeline parallelism"
            if pp_style == "zbv":
                self.logger.warning("zero-bubble V schedule: weight gradients are deferred (dX/dW split)", ranks=[0])
            self.stage_manager = PipelineStageManager(
                self.pg_mesh, pipeline_axis=self.pp_axis, enable_interleave=pp_style in ("interleaved", "zbv"),
                use_zbv=pp_style == "zbv", num_model_chunks=num_model_chunks, num_layers_per_stage=num_layers_per_stage)
            from ...pipeline.schedule import InterleavedSchedule, OneForwardOneBackwardSchedule, ZeroBubbleVPipeScheduler

            if pp_style == "interleaved":
                assert num_model_chunks > 1, "number of model chunks must be > 1 when using interleaved"
                self.scheduler = InterleavedSchedule(
                    stage_manager=self.stage_manager, num_model_chunks=num_model_chunks,
                    num_microbatch=num_microbatches, microbatch_size=microbatch_size,
                    enable_metadata_cache=enable_metadata_cache, overlap_p2p=overlap_p2p,
                    fp8_communication=fp8_communication)
            elif pp_style == "1f1b":
                self.scheduler = OneForwardOneBackwardSchedule(
                    stage_manager=self.stage_manager, num_microbatches=num_microbatches,
                    microbatch_size=microbatch_size, enable_metadata_cache=enable_metadata_cache,
                    fp8_communication=fp8_communication)
            else:
                self.scheduler = ZeroBubbleVPipeScheduler(
                    stage_manager=self.stage_manager, schedule=scheduler_nodes, num_model_chunks=num_model_chunks,
                    num_microbatch=num_microbatches, microbatch_size=microbatch_size,
                    enable_metadata_cache=enable_metadata_cache, overlap_p2p=overlap_p2p)
            self.schedule = self.scheduler
        # ---- groups
        self.tp_group = self.pg_mesh.group("tp")
        self.dp_group = self.pg_mesh.group("dp")
        self.pp_group = self.pg_mesh.group("pp")
        if self.enable_sequence_parallelism and self.sequence_parallelism_mode in ("split_gather", "ring"):
            self.sp_group = self.tp_group
        else:
            self.sp_group = self.pg_mesh.group("sp")
        # params are replicated over sp in all_to_all / ring_attn -> their grads are averaged over dp x sp
        if self.enable_sequence_parallelism and self.sequence_parallelism_mode in ("all_to_all", "ring_attn") \
                and self.sp_size > 1:
            self.mixed_dp_group = self.pg_mesh.group("dp", "sp")
            self.dp_size_for_grads = self.dp_size * self.sp_size
        else:
            self.mixed_dp_group = self.dp_group
            self.dp_size_for_grads = self.dp_size
        self.use_fp8 = use_fp8
        self.shard_config = ShardConfig(
            tensor_parallel_process_group=self.tp_group, sequence_parallel_process_group=self.sp_group,
            pipeline_stage_manager=self.stage_manager, enable_tensor_parallelism=self.tp_size > 1,
            enable_all_optimization=self.enable_all_optimization,
            enable_fused_normalization=self.enable_fused_normalization,
            enable_flash_attention=self.enable_flash_attention, enable_jit_fused=self.enable_jit_fused,
            enable_sequence_parallelism=enable_sequence_parallelism,
            sequence_parallelism_mode=self.sequence_parallelism_mode, parallel_output=parallel_output,
            make_vocab_size_divisible_by=make_vocab_size_divisible_by,
            gradient_checkpoint_config=gradient_checkpoint_config, fp8_communication=fp8_communication,
            inner_ring_size=inner_ring_size, pg_mesh=self.pg_mesh, sp_axis=self.sp_axis,
            comm_backend=comm_backend, use_zbv=(pp_style == "zbv" and pp_size > 1))
        self.amp_config = dict(initial_scale=initial_scale, growth_factor=growth_factor,
                               backoff_factor=backoff_factor, growth_interval=growth_interval, hysteresis=hysteresis,
                               min_scale=min_scale, max_scale=max_scale)
        self.ddp_config = dict(broadcast_buffers=broadcast_buffers, bucket_cap_mb=ddp_bucket_cap_mb,
                               find_unused_parameters=find_unused_parameters, check_reduction=check_reduction,
                               gradient_as_bucket_view=gradient_as_bucket_view, static_graph=static_graph)
        self.zero_config = dict(reduce_bucket_size=zero_bucket_size_in_m * 1024 * 1024,
                                communication_dtype=communication_dtype, overlap_communication=overlap_communication,
                                cpu_offload=cpu_offload, offload_optim_frac=offload_optim_frac,
                                partition_grad=(self.zero_stage == 2), forced_dtype=PRECISION_TORCH_TYPE[precision],
                                overlap_allgather=overlap_allgather, fp8_communication=fp8_communication)
        self.max_norm = max_norm
        set_comm_backend(comm_backend)

    def __del__(self):
        try:
            self.pg_mesh.destroy_mesh_process_groups()
        except Exception:
            pass

    # ------------------------------------------------------------------ capability introspection
    @property
    def enable_pipeline_parallelism(self) -> bool:
        return self.pp_size > 1

    def supported_devices(self) -> List[str]:
        return ["cuda", "cpu"]

    def supported_precisions(self) -> List[str]:
        return ["fp16", "bf16", "fp32"]

    def control_device(self) -> bool:
        return True

    def control_precision(self) -> bool:
        return True

    def support_no_sync(self) -> bool:
        return True

    def support_lora(self) -> bool:
        return True

    def control_checkpoint_io(self) -> bool:
        return True

    # ------------------------------------------------------------------ configure
    def configure(self, model: Module, optimizer: Optional[Optimizer] = None, criterion: Optional[Callable] = None,
                  dataloader: Optional[DataLoader] = None, lr_scheduler: Optional[LRScheduler] = None):
        param_info = get_param_info(optimizer, model)
        zbv = self.pp_style == "zbv" and self.pp_size > 1
        if not isinstance(model, ModelWrapper):
            use_ddp = False   # gradient averaging over dp is done explicitly (bucketed) so it composes with PP/SP
            model = HybridParallelModule(model, precision=self.precision, shard_config=self.shard_config,
                                         dp_group=self.mixed_dp_group, tp_group=self.tp_group, sp_group=self.sp_group,
                                         use_ddp=use_ddp, ddp_config=self.ddp_config, custom_policy=self.custom_policy,
                                         overlap_allgather=self.zero_config["overlap_allgather"], use_fp8=self.use_fp8,
                                         inplace_wgrad=(self.zero_stage == 0))
            model.dp_size = self.dp_size_for_grads
        if optimizer is not None and not isinstance(optimizer, OptimizerWrapper):
            from ...nn.optimizer import cast_to_distributed

            optimizer = cast_to_distributed(optimizer)
            if self.zero_stage == 0:
                if self.precision in ("fp16", "bf16"):
                    optimizer = HybridParallelAMPOptimizer(
                        optimizer, model, use_pipeline=self.enable_pipeline_parallelism, param_info=param_info,
                        precision=self.precision, max_norm=self.max_norm, pp_process_group=self.pp_group,
                        tp_process_group=self.tp_group, **self.amp_config)
                else:
                    optimizer = HybridParallelNaiveOptimizer(
                        optimizer, model, use_pipeline=self.enable_pipeline_parallelism, param_info=param_info,
                        max_norm=self.max_norm, pp_process_group=self.pp_group, tp_process_group=self.tp_group)
            else:
                from .hybrid_zero import HybridParallelZeroOptimizer

                zero_dp_size = dist.get_world_size(self.mixed_dp_group)
                if zero_dp_size == 1:
                    self.logger.warning("ZeRO with data-parallel size 1 has no sharding effect", ranks=[0])
                assert self.precision != "fp32", "Please set precision to 'fp16' or 'bf16' when using ZeRO."
                optimizer = HybridParallelZeroOptimizer(
                    optimizer, model, use_pipeline=self.enable_pipeline_parallelism, param_info=param_info,
                    dp_process_group=self.mixed_dp_group, tp_process_group=self.tp_group,
                    pp_process_group=self.pp_group, verbose=False, clip_grad_norm=self.max_norm,
                    **self.zero_config, **self.amp_config)
            if hasattr(optimizer.optim, "setup_distributed"):
                optimizer.optim.setup_distributed(tp_group=self.tp_group, dp_group=self.mixed_dp_group,
                                                  shard_to_working_param=getattr(optimizer, "get_master_to_working_map", lambda: {})() or {},
                                                  padding_map=None, is_zero=self.zero_stage > 0)
        if optimizer is not None and hasattr(model, "bind_optimizer"):
            model.bind_optimizer(optimizer)          # load_model() must refresh the optimizer's fp32 masters
        return model, optimizer, criterion, dataloader, lr_scheduler

    # ------------------------------------------------------------------ training step helpers
    def execute_pipeline(self, data_iter: Iterator, model: HybridParallelModule, criterion: Callable,
                         optimizer: Optional[OptimizerWrapper] = None, return_loss: bool = True,
                         return_outputs: bool = False) -> dict:
        assert self.enable_pipeline_parallelism, "pipeline parallelism is not enabled"
        if return_outputs:
            self.logger.warning("return_outputs may lead to significant extra memory consumption.", ranks=[0])
        # defer DP / shared-param / SP grad syncs to after the last micro-batch
        ctx = optimizer.no_sync() if (optimizer is not None and hasattr(optimizer, "no_sync") and self.zero_stage > 0) \
            else model.no_sync()
        with ctx, model._hook_context() if hasattr(model, "_hook_context") else nullcontext():
            outputs = self.scheduler.forward_backward_step(model, data_iter, criterion, optimizer,
                                                           return_loss=return_loss, return_outputs=return_outputs)
        if not torch.is_grad_enabled() or optimizer is None:
            return outputs
        model.sync_shared_params()
        model.sync_sp_grads()
        if self.zero_stage > 0 and hasattr(optimizer, "sync_grad"):
            optimizer.sync_grad()
        else:
            model.sync_dp_grads()
        return outputs

    def backward_and_sync(self, loss: Tensor, model: HybridParallelModule, optimizer: OptimizerWrapper) -> None:
        """Non-PP path used by `Booster.backward`: backward + sp/dp grad syncs."""
        optimizer.backward(loss)
        if self.zero_stage == 0 and model.require_grad_sync:
            model.sync_dp_grads()

    def prepare_dataloader(self, dataset, batch_size, shuffle=False, seed=1024, drop_last=False, pin_memory=False,
                           num_workers=0, distributed_sampler_cls=None, **kwargs):
        _kwargs = kwargs.copy()
        cls = distributed_sampler_cls or DistributedSampler
        sampler = cls(dataset, num_replicas=self.dp_size, rank=self.pg_mesh.axis_rank("dp"), shuffle=shuffle)
        return DataLoader(dataset, batch_size=batch_size, sampler=sampler, worker_init_fn=_seed_worker(seed),
                          drop_last=drop_last, pin_memory=pin_memory, num_workers=num_workers, **_kwargs)

    def get_checkpoint_io(self) -> CheckpointIO:
        from ...checkpoint_io.hybrid_parallel_checkpoint_io import HybridParallelCheckpointIO

        return HybridParallelCheckpointIO(self.mixed_dp_group, self.pp_group, self.tp_group, self.sp_group,
                                          self.zero_stage)

    def no_sync(self, model: Module, optimizer: OptimizerWrapper) -> Iterator[None]:
        assert self.zero_stage != 2, "ZERO2 is not compatible with no_sync function, please run gradient accumulation with gradient synchronization allowed."
        return optimizer.no_sync() if (self.zero_stage > 0 and hasattr(optimizer, "no_sync")) else model.no_sync()

    def enable_lora(self, model: Module, pretrained_dir: Optional[str] = None, lora_config: Optional[Dict] = None,
                    bnb_quantization_config=None, quantize: bool = False) -> Module:
        from ..lora import apply_lora

        assert self.tp_size == 1, "LoRA is not supported together with tensor parallelism yet"
        return apply_lora(model, lora_config, pretrained_dir)
