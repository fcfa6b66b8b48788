"""GeminiOptimizer: optimizer over chunked fp32 master shards.

Parity: reference `colossalai/zero/gemini/gemini_optimizer.py:70-874`: optimizer params are views into the fp32 master
shard of each chunk (per original parameter, so per-group hyper-parameters keep working); gradients come from the
reduced gradient shards; loss-scale / overflow / clipping use chunk l2 norms reduced over the zero (and tp) group;
`HybridAdam` runs the AVX-512 kernel on host-resident shards and the multi-tensor sm_90a kernel on device-resident
ones; afterwards the low-precision working shards are refreshed from the master shards.
"""
from __future__ import annotations

import math
from typing import Dict, Iterator, List, Optional, Set, Tuple

import torch
import torch.distributed as dist
import torch.nn as nn
from torch.distributed import ProcessGroup
from torch.optim import Optimizer

from ...accelerator import get_accelerator
from ...amp.naive_amp.mixed_precision_mixin import BF16MixedPrecisionMixin, FP16MixedPrecisionMixin
from ...interface import OptimizerWrapper
from ...logging import get_dist_logger
from .chunk import Chunk, ChunkManager
from .gemini_ddp import GeminiDDP

__all__ = ["GeminiOptimizer", "GeminiAdamOptimizer", "GeminiFP16MixedPrecisionMixin"]


class GeminiFP16MixedPrecisionMixin(FP16MixedPrecisionMixin):
    def __init__(self, module: GeminiDDP, **kw) -> None:
        super().__init__(**kw)
        self.module = module

    def check_local_overflow(self) -> bool:
        return self.module.overflow_counter.item() > 0

    def pre_zero_grad(self) -> None:
        self.module.overflow_counter.zero_()


class GeminiOptimizer(OptimizerWrapper):
    def __init__(self, optim: Optimizer, module: GeminiDDP, gpu_margin_mem_ratio: float = 0.0,
                 initial_scale: float = 2**32, min_scale: float = 1, growth_factor: float = 2,
                 backoff_factor: float = 0.5, growth_interval: int = 1000, hysteresis: int = 2,
                 max_scale: float = 2**32, max_norm: float = 0.0, norm_type: float = 2.0,
                 tp_group: ProcessGroup = None, params_info=None, verbose: bool = False, **defaults) -> None:
        super().__init__(optim)
        assert isinstance(module, GeminiDDP)
        assert norm_type == 2.0, "Gemini only supports L2 norm now"
        self.module = module
        self.gemini_manager = module.gemini_manager
        self.chunk_manager: ChunkManager = self.gemini_manager.chunk_manager
        self.param_to_range: Dict[nn.Parameter, Tuple[int, int]] = {}
        self.param_to_chunk16: Dict[nn.Parameter, Chunk] = {}
        self.chunk16_set: Set[Chunk] = set()
        self.clipping_flag = max_norm > 0.0
        self.max_norm = max_norm
        self.tp_group = tp_group
        self.tp_size = dist.get_world_size(tp_group) if tp_group is not None else 1
        self.params_info = params_info
        self.verbose = verbose
        self._logger = get_dist_logger()
        self.gpu_margin_mem_ratio = float(gpu_margin_mem_ratio)
        # ---- replace optimizer params by views of the fp32 master shards
        working2master = dict(zip(module.fp16_params, module.fp32_params)) if module.fp32_params else {}
        self.id_to_real_params: Dict[int, nn.Parameter] = {}
        self.id_to_fake_params: Dict[int, nn.Parameter] = {}
        self._fake_info: List[Tuple[nn.Parameter, nn.Parameter, Chunk, int, int]] = []
        model_params = {id(p): p for p in module.fp16_params}
        for group in self.optim.param_groups:
            fake = []
            for p in group["params"]:
                if id(p) not in model_params:
                    continue
                c16 = self.chunk_manager.get_chunk(p)
                info = c16.tensors_info[p]
                s, e = max(info.offset, c16.shard_begin), min(info.end, c16.shard_end)
                if e <= s:
                    continue           # this rank holds no part of the parameter
                self.chunk16_set.add(c16)
                self.param_to_chunk16[p] = c16
                self.param_to_range[p] = (s, e)
                master = working2master.get(p)
                if master is not None:
                    c32 = self.chunk_manager.get_chunk(master)
                    base = c32.cuda_global_chunk if c32.is_gathered else \
                        (c32.cuda_shard if c32.cuda_shard is not None else c32.cpu_shard)
                    off = 0 if c32.is_gathered else c32.shard_begin
                else:   # no master weights: optimise the working shard directly
                    base = c16.cuda_global_chunk if c16.is_gathered else \
                        (c16.cuda_shard if c16.cuda_shard is not None else c16.cpu_shard)
                    off = 0 if c16.is_gathered else c16.shard_begin
                fp = nn.Parameter(base[s - off:e - off], requires_grad=True)
                try:
                    fp.grad_dtype = None      # low-precision gradient shards are consumed directly by the kernels
                except Exception:
                    pass
                self.id_to_real_params[id(fp)] = p
                self.id_to_fake_params[id(p)] = fp
                self._fake_info.append((fp, p, c16, s, e))
                fake.append(fp)
            group["params"] = fake
        self.optim.state.clear()
        if module.mixed_precision is torch.float16:
            self.mix_precision_mixin = GeminiFP16MixedPrecisionMixin(
                module, initial_scale=initial_scale, min_scale=min_scale, growth_factor=growth_factor,
                backoff_factor=backoff_factor, growth_interval=growth_interval, hysteresis=hysteresis,
                max_scale=max_scale)
        else:
            self.mix_precision_mixin = BF16MixedPrecisionMixin()

    # ------------------------------------------------------------------ grads
    def _grad_shard(self, c16: Chunk) -> Optional[torch.Tensor]:
        g = c16.grad_chunk
        if g is None:
            return None
        if g.is_gathered:
            return g.cuda_global_chunk
        return g.cuda_shard if g.cuda_shard is not None else g.cpu_shard

    def _set_grad_ptr(self) -> None:
        for fp, p, c16, s, e in self._fake_info:
            g = self._grad_shard(c16)
            if g is None:
                fp.grad = None
                continue
            off = 0 if c16.grad_chunk.is_gathered else c16.shard_begin
            gs = g[s - off:e - off]
            if gs.device != fp.device:
                gs = gs.to(fp.device)
            try:
                fp.grad = gs
            except RuntimeError:
                fp.grad = gs.to(fp.dtype)

    def _clear_grads(self) -> None:
        for fp, *_ in self._fake_info:
            fp.grad = None
        for c in self.chunk16_set:
            c.grad_chunk = None

    def _calc_global_norm(self) -> float:
        dev = get_accelerator().get_current_device()
        t = torch.zeros(1, dtype=torch.float64, device=dev)
        for c in self.chunk16_set:
            g = c.grad_chunk
            if g is not None and g.l2_norm is not None:
                t += g.l2_norm.to(device=dev, dtype=torch.float64) if torch.is_tensor(g.l2_norm) else g.l2_norm
        if dist.is_initialized():
            dist.all_reduce(t, group=self.module.zero_group)
            if self.tp_size > 1:
                dist.all_reduce(t, group=self.tp_group)
        return math.sqrt(t.item())

    def _get_combined_scale(self):
        div_scale = self.mix_precision_mixin.get_grad_div_scale()
        if self.clipping_flag:
            total_norm = self._calc_global_norm() / div_scale
            self._current_grad_norm = total_norm
            clip = (total_norm + 1e-6) / self.max_norm
            if clip > 1:
                div_scale = clip * div_scale
        return -1 if div_scale == 1.0 else div_scale

    # ------------------------------------------------------------------ API
    def zero_grad(self, *args, **kwargs):
        self.mix_precision_mixin.pre_zero_grad()
        self._clear_grads()
        self.module.accumulating_grads = False
        return self.optim.zero_grad(set_to_none=True)

    def step(self, *args, **kwargs):
        if self.mix_precision_mixin.should_skip_step():
            if self.verbose:
                self._logger.info("Found overflow. Skip step")
            self._clear_grads()
            self.zero_grad()
            return
        self._set_grad_ptr()
        combined = self._get_combined_scale()
        try:
            ret = self.optim.step(div_scale=combined, *args, **kwargs)
        except TypeError:
            if combined != -1:
                for fp, *_ in self._fake_info:
                    if fp.grad is not None:
                        fp.grad = fp.grad.float() / combined
            else:
                for fp, *_ in self._fake_info:
                    if fp.grad is not None and fp.grad.dtype != fp.dtype:
                        fp.grad = fp.grad.to(fp.dtype)
            ret = self.optim.step(*args, **kwargs)
        self._update_fp16_params()
        self._clear_grads()
        self.module.overflow_counter.zero_()
        self.module.accumulating_grads = False
        return ret

    def _update_fp16_params(self) -> None:
        for c16 in self.chunk16_set:
            if c16.paired_chunk is not None:
                c16.optim_update()

    def clip_grad_norm(self, model: torch.nn.Module, max_norm: float, norm_type: float = 2.0):
        raise NotImplementedError("pass max_norm to GeminiPlugin / GeminiOptimizer instead")

    def backward(self, loss: torch.Tensor, inputs=None, retain_graph: bool = False, **kw):
        loss = self.mix_precision_mixin.pre_backward(loss)
        self.module.backward(loss)

    def backward_by_grad(self, tensor: torch.Tensor, grad: torch.Tensor, inputs=None, retain_graph: bool = False):
        grad = self.mix_precision_mixin.pre_backward_by_grad(tensor, grad)
        self.module.backward_by_grad(tensor, grad)

    # ------------------------------------------------------------------ checkpoint
    def _agreed_state_layout(self):
        """(tensor keys -> dtype, scalar template) agreed over the zero group.  A rank whose chunk shards hold only
        padding (tiny models, uneven tails) has no optimizer state at all, so the key list cannot be read locally —
        every rank must still join the same sequence of collectives."""
        tkeys: Dict[str, torch.dtype] = {}
        scalars: Dict = {}
        for st in self.optim.state.values():
            for k, v in st.items():
                if torch.is_tensor(v) and v.dim() > 0:
                    tkeys.setdefault(k, v.dtype)
                elif k not in scalars:
                    scalars[k] = v.cpu() if torch.is_tensor(v) else v
        # (`chunk16_set` only lists chunks this rank owns state for - ask the chunk manager, every rank has every chunk)
        params = self.module.fp16_params
        pg = self.chunk_manager.get_chunk(params[0]).torch_pg if params else None
        ws = dist.get_world_size(pg) if dist.is_initialized() else 1       # pg None = the default (world) group
        if ws > 1:
            box = [None] * ws
            dist.all_gather_object(box, (tkeys, scalars), group=pg)
            merged_t: Dict[str, torch.dtype] = {}
            merged_s: Dict = {}
            for t, sc in box:
                for k, v in t.items():
                    merged_t.setdefault(k, v)
                for k, v in sc.items():
                    merged_s.setdefault(k, v)
            tkeys, scalars = merged_t, merged_s
        return dict(sorted(tkeys.items())), scalars

    def state_dict(self, only_rank_0: bool = True) -> dict:
        """Gathered state keyed by the ORIGINAL parameter order.  Collective over the zero group: for every parameter
        and every tensor state key each rank contributes its slice (or zeros) to one all-reduce."""
        order = {id(p): i for i, p in enumerate(self.module.fp16_params)}
        by_param = {id(p): (fp, p, c, s, e) for fp, p, c, s, e in self._fake_info}
        tkeys, scalars = self._agreed_state_layout()
        state: Dict[int, Dict] = {}
        dev = get_accelerator().get_current_device()
        for p in self.module.fp16_params:
            c16 = self.chunk_manager.get_chunk(p)
            info = c16.tensors_info[p]
            ent = by_param.get(id(p))
            st = self.optim.state.get(ent[0], {}) if ent is not None else {}
            out: Dict = {}
            for k, dt in tkeys.items():
                full = torch.zeros(info.end - info.offset, dtype=dt, device=dev)
                if ent is not None and k in st:
                    s, e = ent[3], ent[4]
                    full[s - info.offset:e - info.offset] = st[k].to(dev).reshape(-1)
                if c16.pg_size > 1 and not c16.keep_gathered:
                    dist.all_reduce(full, group=c16.torch_pg)
                out[k] = full.view(info.shape).cpu()
            for k, v in scalars.items():
                own = st.get(k, v)
                out[k] = own.cpu() if torch.is_tensor(own) else own
            state[order[id(p)]] = out
        groups = []
        for g in self.optim.param_groups:
            groups.append({**{k: v for k, v in g.items() if k != "params"},
                           "params": [order[id(self.id_to_real_params[id(fp)])] for fp in g["params"]]})
        return {"state": state, "param_groups": groups}

    def load_state_dict(self, state_dict: dict):
        order = {id(p): i for i, p in enumerate(self.module.fp16_params)}
        for fp, p, c16, s, e in self._fake_info:
            info = c16.tensors_info[p]
            src = state_dict["state"].get(order[id(p)], {})
            st = {}
            for k, v in src.items():
                if torch.is_tensor(v) and v.dim() > 0 and v.numel() == info.end - info.offset:
                    st[k] = v.reshape(-1)[s - info.offset:e - info.offset].to(fp.device).clone()
                else:
                    st[k] = v
            self.optim.state[fp] = st
        for g, saved in zip(self.optim.param_groups, state_dict["param_groups"]):
            for k, v in saved.items():
                if k != "params":
                    g[k] = v

    def state_shard(self, prefix: str = "", max_shard_size: int = 1024, only_rank_0: bool = True,
                    pinned_state_dicts=None) -> Iterator[Tuple[Dict, int]]:
        from ...checkpoint_io.utils import StateDictSharder

        sharder = StateDictSharder(max_shard_size)
        for pid, st in self.state_dict(only_rank_0)["state"].items():
            block, size = sharder.append_optim_state(pid, st)
            if block is not None:
                yield block, size
        yield sharder.current_block, sharder.current_block_size

    def get_working_to_master_map(self):
        return None

    def get_master_to_working_map(self):
        return None


class GeminiAdamOptimizer(GeminiOptimizer):
    def __init__(self, model: torch.nn.Module, **defaults) -> None:
        from ...nn.optimizer import HybridAdam

        optimizer = HybridAdam(model.parameters(), **{k: v for k, v in defaults.items()
                                                      if k in ("lr", "betas", "eps", "weight_decay", "adamw_mode")})
        super().__init__(optimizer, model, **{k: v for k, v in defaults.items()
                                              if k not in ("lr", "betas", "eps", "weight_decay", "adamw_mode")})
