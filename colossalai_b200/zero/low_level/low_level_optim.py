"""ZeRO stage 1 / 2 optimizer on flat, bucketed buffers.

Parity: reference `colossalai/zero/low_level/low_level_optim.py:74-1034` (+ `bookkeeping/{bucket_store,gradient_store,
tensor_bucket}.py`): fp32 master shards per rank, gradient reduction overlapped with backward on a side comm stream,
ZeRO-1 (grads kept until the sync point, `no_sync` accumulation) vs ZeRO-2 (reduce-scatter as soon as a bucket is
complete and free the full bucket), unscale + clip with hybrid-aware norm, updated working params all-gathered,
several dp groups (`pg_to_param_list`, used for MoE expert params), cpu_offload of master/optimizer states.

H100-first layout: the working parameters of a bucket are *views of one flat buffer*; every rank owns a contiguous 1/dp
slice of each bucket.  So a bucket needs exactly one `reduce_scatter_tensor` (grads) and one `all_gather_into_tensor`
(updated params) with no flatten / unflatten copies, and the fused Adam kernel updates master shard + moments and writes
the low-precision slice in one launch.
"""
from __future__ import annotations

from contextlib import contextmanager
from typing import Dict, Iterator, List, Optional, Tuple

import torch
import torch.distributed as dist
import torch.nn as nn
from torch import Tensor
from torch.distributed import ProcessGroup
from torch.optim import Optimizer

from ...accelerator import get_accelerator
from ...amp.naive_amp.mixed_precision_mixin import BF16MixedPrecisionMixin, FP16MixedPrecisionMixin
from ...interface import OptimizerWrapper
from ...logging import get_dist_logger
from ...ops import multi_tensor as mt
from ...ops._dispatch import use_native
from ...parallel import comm

__all__ = ["LowLevelZeroOptimizer", "LowLevelZeroFP16MixedPrecisionMixin"]


class LowLevelZeroFP16MixedPrecisionMixin(FP16MixedPrecisionMixin):
    def __init__(self, owner: "LowLevelZeroOptimizer", **kw) -> None:
        super().__init__(**kw)
        self.owner = owner

    def check_local_overflow(self) -> bool:
        for b in self.owner.buckets:
            if b.grad_shard is not None and not torch.isfinite(b.grad_shard).all():
                return True
        return False


class _Bucket:
    """A contiguous group of working params sharing dtype, param group and data-parallel group."""

    def __init__(self, params: List[nn.Parameter], group_id: int, pg: ProcessGroup, align: int = 64) -> None:
        self.params = params
        self.group_id = group_id
        self.pg = pg
        self.ws, self.rank = comm.group_size(pg), comm.group_rank(pg)
        self.dtype = params[0].dtype
        self.device = params[0].device
        offs, n = [], 0
        for p in params:
            offs.append(n)
            n += p.numel()
        mult = self.ws * align
        self.numel = n
        self.padded = ((n + mult - 1) // mult) * mult
        self.offsets = offs
        self.shard_size = self.padded // self.ws
        # flat working storage; params become views
        self.flat = torch.zeros(self.padded, dtype=self.dtype, device=self.device)
        for p, o in zip(params, offs):
            self.flat[o:o + p.numel()].copy_(p.data.reshape(-1))
            p.data = self.flat[o:o + p.numel()].view(p.shape)
        self.grad_full: Optional[Tensor] = None      # [padded] accumulated local gradients (comm dtype)
        self.grad_shard: Optional[Tensor] = None     # [shard_size] reduced gradient shard
        self.n_ready = 0
        self.reduced = False
        self.work = None
        self.touched = [False] * len(params)         # which params received a gradient since the last step

    @property
    def my_slice(self) -> slice:
        return slice(self.rank * self.shard_size, (self.rank + 1) * self.shard_size)

    def working_shard(self) -> Tensor:
        return self.flat[self.my_slice]


class LowLevelZeroOptimizer(OptimizerWrapper):
    def __init__(self, optimizer: Optimizer, pg_to_param_list: Optional[Dict[ProcessGroup, List[nn.Parameter]]] = None,
                 initial_scale: float = 2**16, min_scale: float = 1, growth_factor: float = 2.0,
                 backoff_factor: float = 0.5, growth_interval: int = 2000, hysteresis: int = 2,
                 max_scale: float = 2**24, clip_grad_norm: float = 0.0, verbose: bool = False,
                 reduce_bucket_size: int = 1024 * 1024, communication_dtype: Optional[torch.dtype] = None,
                 overlap_communication: bool = False, partition_grad: bool = False, cpu_offload: bool = False,
                 dp_process_group: Optional[ProcessGroup] = None, extra_dp_group: Optional[ProcessGroup] = None,
                 forced_dtype: Optional[torch.dtype] = None, master_weights: bool = True,
                 overlap_allgather: bool = False, fp8_communication: bool = False, backward_context=None,
                 offload_optim_frac: float = 1.0, skip_untouched_params: bool = False) -> None:
        super().__init__(optim=optimizer)
        # flat buckets step a parameter that received no gradient with a ZERO gradient (moments decay, momentum moves
        # it, weight decay applies).  `skip_untouched_params=True` gives `torch.optim` / reference semantics instead -
        # such a parameter and its moments are left exactly as they were - for one small all-reduce and host read per
        # step (the ranks must agree on what "received no gradient anywhere" means), hence opt-in.  (Adam's bias
        # correction still uses the bucket's step count: a flat state has one counter, not one per parameter.)
        self._skip_untouched = bool(skip_untouched_params)
        # cpu_offload: fraction of the optimizer state (fp32 master + moments, by element count) that lives in pinned
        # host memory and is stepped by the AVX-512 CPU Adam; the rest stays in HBM on the fused multi-tensor path.
        # 1.0 = everything (the reference's `cpu_offload=True`), smaller values tier the state between HBM and DRAM.
        self._offload_frac = float(offload_optim_frac)
        self._offload_numel_seen = 0
        self._offload_total = sum(p.numel() for g in optimizer.param_groups for p in g["params"] if p.requires_grad)
        self._offload_stream = None
        self._dtype = self.optim.param_groups[0]["params"][0].dtype
        self._logger = get_dist_logger()
        self._verbose = verbose
        self._partition_grads = partition_grad
        self._cpu_offload = cpu_offload
        self._master_weights = master_weights
        self._overlap_communication = overlap_communication and torch.cuda.is_available()
        self._overlap_allgather = overlap_allgather
        self._fp8_communication = fp8_communication
        self._reduce_bucket_size = max(int(reduce_bucket_size), 1)
        self._communication_dtype = communication_dtype
        self._clip_grad_norm = clip_grad_norm
        self._backward_context = backward_context
        self.require_grad_sync = True
        self.dp_pg = dp_process_group
        self.extra_dp_group = extra_dp_group
        if forced_dtype is not None:
            for group in self.optim.param_groups:
                for p in group["params"]:
                    p.data = p.data.to(forced_dtype)
            self._dtype = forced_dtype
        # which dp group reduces which param (dense vs expert params)
        if pg_to_param_list is None:
            all_params = [p for g in self.optim.param_groups for p in g["params"]]
            pg_to_param_list = {dp_process_group: all_params}
        self.param_to_pg: Dict[int, ProcessGroup] = {}
        for pg, plist in pg_to_param_list.items():
            for p in plist:
                self.param_to_pg[id(p)] = pg
        self.pg_to_param_list = pg_to_param_list
        self._comm_stream = torch.cuda.Stream() if self._overlap_communication else None
        # ---- build buckets per (param group, dtype, pg)
        self.buckets: List[_Bucket] = []
        self._param_bucket: Dict[int, Tuple[_Bucket, int]] = {}
        self._master_of_bucket: Dict[int, Tensor] = {}
        for gid, group in enumerate(self.optim.param_groups):
            by_key: Dict[Tuple, List[nn.Parameter]] = {}
            for p in group["params"]:
                if not p.requires_grad:
                    continue
                pg = self.param_to_pg.get(id(p), dp_process_group)
                by_key.setdefault((p.dtype, id(pg)), []).append(p)
            master_params = []
            for (dtype, _), plist in by_key.items():
                pg = self.param_to_pg.get(id(plist[0]), dp_process_group)
                # gradients become ready in reverse order of use: bucket in reverse so buckets complete one by one
                cur, cur_n = [], 0
                for p in reversed(plist):
                    if cur and cur_n + p.numel() > self._reduce_bucket_size:
                        master_params.append(self._register_bucket(_Bucket(cur, gid, pg)))
                        cur, cur_n = [], 0
                    cur.append(p)
                    cur_n += p.numel()
                if cur:
                    master_params.append(self._register_bucket(_Bucket(cur, gid, pg)))
            group["params"] = master_params
        # hooks
        self._hooks = []
        for b in self.buckets:
            for idx, p in enumerate(b.params):
                self._hooks.append(p.register_post_accumulate_grad_hook(self._make_hook(b, idx)))
        if self._dtype == torch.float16:
            self.mixed_precision_mixin = LowLevelZeroFP16MixedPrecisionMixin(
                self, initial_scale=initial_scale, min_scale=min_scale, growth_factor=growth_factor,
                backoff_factor=backoff_factor, growth_interval=growth_interval, hysteresis=hysteresis,
                max_scale=max_scale)
        elif self._dtype == torch.bfloat16:
            self.mixed_precision_mixin = BF16MixedPrecisionMixin()
        else:
            self.mixed_precision_mixin = None
        self._tables: Dict = {}
        self._current_grad_norm: Optional[float] = None

    # ------------------------------------------------------------------ construction helpers
    def _register_bucket(self, b: _Bucket) -> nn.Parameter:
        self.buckets.append(b)
        for i, p in enumerate(b.params):
            self._param_bucket[id(p)] = (b, i)
        shard = b.working_shard()
        if self._master_weights or shard.dtype != torch.float32:
            master = shard.detach().clone().float()
        else:
            master = shard.detach()
        b.offloaded = False
        if self._cpu_offload and self._offload_numel_seen < self._offload_frac * self._offload_total:
            master = master.cpu().pin_memory() if torch.cuda.is_available() else master.cpu()
            b.offloaded = True
        self._offload_numel_seen += b.numel
        mp = nn.Parameter(master, requires_grad=True)
        b.master = mp
        self._master_of_bucket[id(b)] = mp
        return mp

    @property
    def dtype(self):
        return self._dtype

    @property
    def num_param_groups(self) -> int:
        return len(self.optim.param_groups)

    # ------------------------------------------------------------------ gradient path
    def _comm_dtype(self, b: _Bucket) -> torch.dtype:
        return self._communication_dtype or b.dtype

    def _make_hook(self, b: _Bucket, idx: int):
        def hook(p: nn.Parameter):
            g = p.grad
            if g is None:
                return
            if b.grad_full is None:
                b.grad_full = torch.zeros(b.padded, dtype=self._comm_dtype(b), device=b.device)
            o = b.offsets[idx]
            b.grad_full[o:o + p.numel()].add_(g.reshape(-1).to(b.grad_full.dtype))
            p.grad = None
            b.touched[idx] = True
            b.n_ready += 1
            if b.n_ready == len(b.params):
                b.n_ready = 0
                if self.require_grad_sync and self._partition_grads:
                    self._reduce_bucket(b)       # ZeRO-2: reduce as soon as complete, free the full buffer
                elif self.require_grad_sync and self._overlap_communication:
                    self._reduce_bucket(b)       # ZeRO-1 + overlap: same, overlapped with the rest of backward

        return hook

    def _reduce_bucket(self, b: _Bucket) -> None:
        if b.grad_full is None:
            return
        ws = b.ws
        full = b.grad_full
        stream = self._comm_stream
        if stream is not None:
            stream.wait_stream(torch.cuda.current_stream())
            ctx = torch.cuda.stream(stream)
        else:
            from contextlib import nullcontext

            ctx = nullcontext()
        with ctx:
            # allocated on the stream that writes and consumes it (a temporary allocated on the compute stream could be
            # handed out again there while the comm stream still reads it)
            shard = torch.empty(b.shard_size, dtype=full.dtype, device=full.device)
            if ws > 1:
                full.div_(ws)
                if self._fp8_communication:
                    from ...quantization.fp8 import reduce_scatter_fp8

                    reduce_scatter_fp8(shard, list(full.chunk(ws)), group=b.pg)
                else:
                    dist.reduce_scatter_tensor(shard, full, group=b.pg)
                if self.extra_dp_group is not None and comm.group_size(self.extra_dp_group) > 1:
                    shard.div_(comm.group_size(self.extra_dp_group))
                    dist.all_reduce(shard, group=self.extra_dp_group)
            else:
                shard.copy_(full)
            if b.grad_shard is None:
                b.grad_shard = shard
            else:
                b.grad_shard.add_(shard)
            if stream is not None:
                full.record_stream(stream)
        b.grad_full = None
        b.reduced = True

    def sync_grad(self) -> None:
        """Reduce every bucket that still holds un-reduced local gradients (end of accumulation / PP step)."""
        for b in self.buckets:
            if b.grad_full is not None:
                self._reduce_bucket(b)

    _sync_grad = sync_grad

    @contextmanager
    def no_sync(self) -> Iterator[None]:
        old = self.require_grad_sync
        self.require_grad_sync = False
        try:
            yield
        finally:
            self.require_grad_sync = old

    def backward(self, loss: Tensor, inputs=None, retain_graph: bool = False, **kw) -> None:
        assert not (self._partition_grads and not self.require_grad_sync), (
            "ZeRO2(partition_grads) and no_sync are not compatible")
        if self.mixed_precision_mixin is not None:
            loss = self.mixed_precision_mixin.pre_backward(loss)
        ctx = self._backward_context() if self._backward_context is not None else None
        if ctx is not None:
            with ctx:
                loss.backward(inputs=inputs, retain_graph=retain_graph)
        else:
            loss.backward(inputs=inputs, retain_graph=retain_graph)
        if self.require_grad_sync:
            self.sync_grad()

    def backward_by_grad(self, tensor, grad, inputs: Tensor = None, retain_graph: bool = False) -> None:
        assert not (self._partition_grads and not self.require_grad_sync)
        if self.mixed_precision_mixin is not None:
            grad = self.mixed_precision_mixin.pre_backward_by_grad(tensor, grad)
        torch.autograd.backward(tensor, grad, inputs=inputs, retain_graph=retain_graph)
        if self.require_grad_sync:
            self.sync_grad()

    def zero_grad(self, set_to_none: bool = True) -> None:
        if self.mixed_precision_mixin is not None:
            self.mixed_precision_mixin.pre_zero_grad()
        for b in self.buckets:
            b.grad_shard = None
            b.grad_full = None
            b.n_ready = 0
            b.touched = [False] * len(b.params)
            for p in b.params:
                p.grad = None
            b.master.grad = None

    # ------------------------------------------------------------------ step
    def _local_norm_sq(self, buckets: List[_Bucket]) -> Tensor:
        dev = get_accelerator().get_current_device()
        shards = [b.grad_shard for b in buckets if b.grad_shard is not None]
        if not shards:
            return torch.zeros(1, device=dev)
        return torch.stack([s.float().pow(2).sum() for s in shards]).sum().reshape(1).to(dev)

    def _compute_grad_norm_sq(self) -> Tensor:
        """Squared global grad norm; each dp group contributes the sum over its shards."""
        total = None
        by_pg: Dict[int, List[_Bucket]] = {}
        for b in self.buckets:
            by_pg.setdefault(id(b.pg), []).append(b)
        for _, bs in by_pg.items():
            n = self._local_norm_sq(bs)
            if bs[0].ws > 1:
                dist.all_reduce(n, group=bs[0].pg)
            total = n if total is None else total + n
        return total if total is not None else torch.zeros(1)

    def step(self, closure=None):
        assert closure is None, "closure is not supported by gemini/zero optimizers"
        if self._comm_stream is not None:
            torch.cuda.current_stream().wait_stream(self._comm_stream)
        if self.mixed_precision_mixin is not None and self.mixed_precision_mixin.should_skip_step():
            if self._verbose:
                self._logger.info("Found overflow. Skip step")
            self.zero_grad()
            return
        div_scale = self.mixed_precision_mixin.get_grad_div_scale() if self.mixed_precision_mixin is not None else 1.0
        clip_coef = None
        if self._clip_grad_norm > 0.0:
            norm = self._compute_grad_norm_sq().sqrt() / div_scale
            self._grad_norm_dev = norm
            clip_coef = (self._clip_grad_norm / (norm + 1e-6)).clamp(max=1.0).float().reshape(1)
        live = [b for b in self.buckets if b.grad_shard is not None]
        self._stepped_groups = set()
        kept = self._snapshot_untouched(live) if self._skip_untouched else []
        fused = (live and use_native(live[0].grad_shard) and self._is_adam())
        if fused and self._cpu_offload:
            # tiered optimizer state: HBM-resident buckets on the fused GPU kernel (asynchronous), host-resident
            # buckets through the pipelined D2H -> CPU Adam -> H2D path, which overlaps with it
            on_gpu = [b for b in live if not b.offloaded]
            if on_gpu:
                self._fused_adam(on_gpu, div_scale, clip_coef)
            self._offload_adam([b for b in live if b.offloaded], div_scale, clip_coef)
        elif fused:
            self._fused_adam(live, div_scale, clip_coef)
        else:
            coef = 1.0 / div_scale
            for b in live:
                g = b.grad_shard.to(b.master.device).float()
                if clip_coef is not None:
                    g = g * (coef * clip_coef.to(g.device))
                elif coef != 1.0:
                    g = g * coef
                b.master.grad = g
            self.optim.step()
            for b in live:
                b.working_shard().copy_(b.master.data.to(b.device))
                b.master.grad = None
        for b, lo, hi, saved in kept:                  # parameters without a gradient anywhere: as if never stepped
            st = self.optim.state[b.master]
            b.master.data[lo:hi].copy_(saved[0])
            for key, v in st.items():
                if torch.is_tensor(v) and v.shape == b.master.data.shape:
                    # a state created by this very step (first step of the bucket) had no value before: zero
                    v[lo:hi].copy_(saved[1][key]) if key in saved[1] else v[lo:hi].zero_()
            b.working_shard()[lo:hi].copy_(b.master.data[lo:hi].to(b.device))
        for b in self.buckets:
            b.grad_shard = None
            b.touched = [False] * len(b.params)
        # all-gather the updated working params (one collective per bucket, straight into param storage)
        for b in self.buckets:
            if b.ws > 1:
                if self._fp8_communication:
                    from ...quantization.fp8 import all_gather_fp8

                    all_gather_fp8(list(b.flat.chunk(b.ws)), b.working_shard().clone(), group=b.pg)
                else:
                    dist.all_gather_into_tensor(b.flat, b.working_shard().clone(), group=b.pg)

    def _snapshot_untouched(self, live: List[_Bucket]):
        """[(bucket, lo, hi, (master, exp_avg, exp_avg_sq) copies)] for the part of this rank's shard that belongs to
        parameters no rank produced a gradient for in this step."""
        out = []
        for b in live:
            flags = torch.tensor([int(t) for t in b.touched], dtype=torch.int32, device=b.device)
            if b.ws > 1:
                dist.all_reduce(flags, op=dist.ReduceOp.MAX, group=b.pg)
            start = b.rank * b.shard_size
            for idx, hit in enumerate(flags.tolist()):
                if hit:
                    continue
                lo = max(b.offsets[idx], start) - start
                hi = min(b.offsets[idx] + b.params[idx].numel(), start + b.shard_size) - start
                if lo >= hi:
                    continue
                st = self.optim.state[b.master]
                states = {k: v[lo:hi].clone() for k, v in st.items()
                          if torch.is_tensor(v) and v.shape == b.master.data.shape}     # moments / momentum buffers
                out.append((b, lo, hi, (b.master.data[lo:hi].clone(), states)))
        return out

    def _bump_step(self, gid: int, group: dict) -> None:
        """Advance a param group's Adam step counter once per optimizer step (both state tiers share it)."""
        if gid not in self._stepped_groups:
            group["step"] = group.get("step", 0) + 1
            self._stepped_groups.add(gid)

    def _is_adam(self) -> bool:
        from ...nn.optimizer.cpu_adam import CPUAdam
        from ...nn.optimizer.fused_adam import FusedAdam

        return isinstance(self.optim, (FusedAdam, CPUAdam, torch.optim.AdamW, torch.optim.Adam))

    def _fused_adam(self, live: List[_Bucket], div_scale: float, clip_coef: Optional[Tensor]) -> None:
        adamw = getattr(self.optim, "adamw_mode", isinstance(self.optim, torch.optim.AdamW))
        for gid, group in enumerate(self.optim.param_groups):
            bs = [b for b in live if b.group_id == gid]
            if not bs:
                continue
            ps, gs, ms, vs, lps = [], [], [], [], []
            for b in bs:
                st = self.optim.state[b.master]
                if "exp_avg" not in st:
                    st["exp_avg"] = torch.zeros_like(b.master.data)
                    st["exp_avg_sq"] = torch.zeros_like(b.master.data)
                    st["step"] = 0
                ps.append(b.master.data)
                gs.append(b.grad_shard)
                ms.append(st["exp_avg"])
                vs.append(st["exp_avg_sq"])
                lps.append(b.working_shard() if b.working_shard().data_ptr() != b.master.data.data_ptr() else None)
            self._bump_step(gid, group)
            tbl = mt.TensorTable(ps, gs, ms, vs, lps)     # grad shards are fresh tensors every step
            beta1, beta2 = group["betas"]
            mt.adam(tbl, group["lr"], beta1, beta2, group["eps"], group["weight_decay"], group["step"], adamw,
                    group.get("bias_correction", True), inv_scale=1.0 / div_scale, inv_scale_dev=clip_coef)

    def _offload_adam(self, live: List[_Bucket], div_scale: float, clip_coef: Optional[Tensor]) -> None:
        """Adam on host-resident optimizer state, pipelined over buckets:
            copy stream : D2H grad shard(b0) | D2H(b1) | D2H(b2) ...        H2D bf16 params(b0) | H2D(b1) ...
            host (OpenMP): . . . . . . . . . | AdamW(b0) | AdamW(b1) | ...
        All D2H copies are queued up front into pinned staging buffers; the host steps bucket i as soon as its copy has
        landed (event), writing the updated low-precision working copy into a pinned buffer whose H2D copy is queued
        at once - so PCIe traffic in both directions overlaps the CPU arithmetic.  (Reference: ZeRO `cpu_offload` of
        `HybridParallelPlugin`, `hybrid_parallel_plugin.py:666-719`, which copies, steps and copies back serially.)"""
        if not live:
            return
        from ...nn.optimizer.cpu_adam import cpu_adam_step

        if self._offload_stream is None:
            self._offload_stream = torch.cuda.Stream()
        st_copy = self._offload_stream
        st_copy.wait_stream(torch.cuda.current_stream())
        inv = 1.0 / div_scale
        if clip_coef is not None:
            inv *= float(clip_coef.item())            # the only host sync of the step (the global norm is a scalar)
        events = []
        with torch.cuda.stream(st_copy):
            for b in live:
                if getattr(b, "host_grad", None) is None or b.host_grad.dtype != b.grad_shard.dtype:
                    b.host_grad = torch.empty(b.shard_size, dtype=b.grad_shard.dtype).pin_memory()
                    b.host_lp = torch.empty(b.shard_size, dtype=b.flat.dtype).pin_memory()
                b.host_grad.copy_(b.grad_shard, non_blocking=True)
                b.grad_shard.record_stream(st_copy)
                ev = torch.cuda.Event()
                ev.record(st_copy)
                events.append(ev)
        adamw = getattr(self.optim, "adamw_mode", isinstance(self.optim, torch.optim.AdamW))
        for b, ev in zip(live, events):
            group = self.optim.param_groups[b.group_id]
            self._bump_step(b.group_id, group)
            stt = self.optim.state[b.master]
            if "exp_avg" not in stt:
                stt["exp_avg"] = torch.zeros_like(b.master.data)
                stt["exp_avg_sq"] = torch.zeros_like(b.master.data)
            beta1, beta2 = group["betas"]
            ev.synchronize()
            same = b.flat.dtype == torch.float32
            cpu_adam_step(b.master.data, b.host_grad, stt["exp_avg"], stt["exp_avg_sq"], group["lr"], beta1, beta2,
                          group["eps"], group["weight_decay"], group["step"], group.get("bias_correction", True), adamw,
                          inv_scale=inv, lp=None if same else b.host_lp)
            with torch.cuda.stream(st_copy):
                b.working_shard().copy_(b.master.data if same else b.host_lp, non_blocking=True)
        torch.cuda.current_stream().wait_stream(st_copy)

    def get_grad_norm(self, norm_type=2.0, **kwargs) -> Optional[float]:
        g = getattr(self, "_grad_norm_dev", None)
        return None if g is None else float(g.item())

    # ------------------------------------------------------------------ checkpoint helpers
    def _gather_full(self, b: _Bucket, shard: Tensor) -> Tensor:
        if b.ws == 1:
            return shard.to(b.device)
        out = torch.empty(b.padded, dtype=shard.dtype, device=b.device)
        dist.all_gather_into_tensor(out, shard.to(b.device).contiguous(), group=b.pg)
        return out

    def state_dict(self) -> Dict:
        """Full (un-sharded) optimizer state keyed by working-param index, gathered over the dp group."""
        state: Dict[int, Dict] = {}
        pid = 0
        groups = []
        for gid, group in enumerate(self.optim.param_groups):
            ids = []
            for b in [bb for bb in self.buckets if bb.group_id == gid]:
                st = self.optim.state.get(b.master, {})
                fulls = {k: self._gather_full(b, v) for k, v in st.items() if torch.is_tensor(v) and v.dim() > 0
                         and v.numel() == b.shard_size}
                scalars = {k: v for k, v in st.items() if k not in fulls}
                for p, o in zip(b.params, b.offsets):
                    entry = {k: f[o:o + p.numel()].view(p.shape).cpu() for k, f in fulls.items()}
                    entry.update(scalars)
                    state[pid] = entry
                    ids.append(pid)
                    pid += 1
            groups.append({**{k: v for k, v in group.items() if k != "params"}, "params": ids})
        return {"state": state, "param_groups": groups}

    def load_state_dict(self, state_dict: Dict) -> None:
        pid = 0
        for gid, group in enumerate(self.optim.param_groups):
            for b in [bb for bb in self.buckets if bb.group_id == gid]:
                st = self.optim.state.setdefault(b.master, {})
                acc: Dict[str, Tensor] = {}
                for p, o in zip(b.params, b.offsets):
                    entry = state_dict["state"].get(pid, {})
                    for k, v in entry.items():
                        if torch.is_tensor(v) and v.dim() > 0:
                            if k not in acc:
                                acc[k] = torch.zeros(b.padded, dtype=v.dtype)
                            acc[k][o:o + p.numel()] = v.reshape(-1)
                        else:
                            st[k] = v
                    pid += 1
                for k, full in acc.items():
                    st[k] = full[b.my_slice].to(b.master.device).clone()
            saved = state_dict["param_groups"][gid]
            for k, v in saved.items():
                if k != "params":
                    group[k] = v

    @torch.no_grad()
    def update_master_params(self, model: Optional[nn.Module] = None) -> None:
        """Refresh the fp32 master shards from the working parameters (after weights were loaded into the model);
        reference: `LowLevelZeroOptimizer.update_master_params`, called by the checkpoint IO after `load_model`."""
        for b in self.buckets:
            if b.master.data.data_ptr() != b.working_shard().data_ptr():
                b.master.data.copy_(b.working_shard().detach().to(b.master.device).float())

    def working_params_in_state_order(self) -> List[nn.Parameter]:
        """Working parameters in the order `state_dict()` / `load_state_dict()` number them."""
        out: List[nn.Parameter] = []
        for gid, _ in enumerate(self.optim.param_groups):
            for b in [bb for bb in self.buckets if bb.group_id == gid]:
                out.extend(b.params)
        return out

    def get_working_to_master_map(self) -> Dict[int, Tensor]:
        return {id(p): b.master for b in self.buckets for p in b.params}

    def get_master_to_working_map(self) -> Dict[int, Tensor]:
        return {id(b.master): b.flat for b in self.buckets}

    def get_param_master_slice(self, p: nn.Parameter) -> Tuple[Tensor, int, int]:
        """(master shard tensor, start, end) of the part of `p` this rank owns (may be empty)."""
        b, i = self._param_bucket[id(p)]
        o = b.offsets[i]
        s, e = max(o, b.my_slice.start), min(o + p.numel(), b.my_slice.stop)
        return b.master.data, s - b.my_slice.start, max(e, s) - b.my_slice.start

    def get_partitioned_gradients_by_param_id(self, group_id: int, param_id: int) -> List[Tensor]:
        for b in self.buckets:
            for p, o in zip(b.params, b.offsets):
                if id(p) == param_id and b.grad_shard is not None:
                    s, e = max(o, b.my_slice.start), min(o + p.numel(), b.my_slice.stop)
                    if e > s:
                        return [b.grad_shard[s - b.my_slice.start:e - b.my_slice.start]]
        return []
