"""LowLevelZeroPlugin: pure data-parallel ZeRO-1/2.
Parity: reference `colossalai/booster/plugin/low_level_zero_plugin.py:368-632`."""
from __future__ import annotations

from contextlib import nullcontext
from functools import partial
from typing import Callable, Dict, Iterator, List, Optional, Tuple

import torch
import torch.distributed as dist
import torch.nn as nn
from torch.optim import Optimizer
from torch.optim.lr_scheduler import _LRScheduler as LRScheduler
from torch.utils.data import DataLoader

from ...accelerator import get_accelerator
from ...checkpoint_io import CheckpointIO, GeneralCheckpointIO
from ...cluster import DeviceMesh
from ...interface import AMPModelMixin, ModelWrapper, OptimizerWrapper
from ...logging import get_dist_logger
from ...zero.low_level import LowLevelZeroOptimizer
from .hybrid_parallel_plugin import _convert_floating_point, _tree_map
from .plugin_base import DPPluginBase

__all__ = ["LowLevelZeroPlugin", "LowLevelZeroModel", "LowLevelZeroCheckpointIO"]

SUPPORTED_PRECISION = ["fp16", "bf16", "fp32"]


class LowLevelZeroModel(ModelWrapper, AMPModelMixin):
    def __init__(self, module: nn.Module, precision: str, overlap_allgather: bool = False, cast_inputs: bool = True,
                 use_fp8: bool = False) -> None:
        super().__init__(module)
        self.dtype = {"fp16": torch.float16, "bf16": torch.bfloat16}.get(precision)
        if self.dtype is not None:
            module = module.to(self.dtype)
        module = module.to(get_accelerator().get_current_device())
        self.module = module
        self.convert_fn = partial(_convert_floating_point, dtype=self.dtype) if (self.dtype is not None and cast_inputs) \
            else None
        self.overlap_allgather = overlap_allgather
        if use_fp8:
            from ...quantization.fp8_hook import convert_linear_to_fp8

            convert_linear_to_fp8(self.module)

    def update_master_params(self) -> None:
        """Called by the checkpoint IO after weights were loaded: the optimizer's fp32 master shards follow."""
        opt = getattr(self, "_zero_optimizer", None)
        opt = opt() if opt is not None else None
        if opt is not None:
            opt.update_master_params(self.module)

    def forward(self, *args, **kwargs):
        if self.convert_fn is not None:
            args = _tree_map(self.convert_fn, args)
            kwargs = _tree_map(self.convert_fn, kwargs)
        return super().forward(*args, **kwargs)


class LowLevelZeroCheckpointIO(GeneralCheckpointIO):
    """Model = plain state dict (params are replicated); optimizer = state gathered over dp, written by rank 0."""

    def save_unsharded_optimizer(self, optimizer: OptimizerWrapper, checkpoint: str, gather_dtensor: bool,
                                 use_async: bool = False):
        assert isinstance(optimizer, LowLevelZeroOptimizer), "Please boost the optimizer before saving!"
        sd = optimizer.state_dict()
        if dist.get_rank() == 0:
            torch.save(sd, checkpoint)
        dist.barrier()

    def save_sharded_optimizer(self, optimizer: OptimizerWrapper, checkpoint: str, gather_dtensor: bool = False,
                               prefix: str = None, size_per_shard: int = 1024, use_async: bool = False):
        import os
        from pathlib import Path

        from ...checkpoint_io.index_file import CheckpointIndexFile
        from ...checkpoint_io.utils import (get_optimizer_base_filenames, save_param_groups, save_state_dict_shards,
                                            shard_optimizer_checkpoint)

        assert isinstance(optimizer, LowLevelZeroOptimizer), "Please boost the optimizer before saving!"
        sd = optimizer.state_dict()
        if dist.get_rank() == 0:
            Path(checkpoint).mkdir(parents=True, exist_ok=True)
            states_name, save_index_file, param_group_file = get_optimizer_base_filenames(prefix)
            index_file = CheckpointIndexFile(checkpoint)
            index_file.append_meta_data("param_groups", param_group_file)
            save_param_groups(sd, os.path.join(checkpoint, param_group_file))
            total = save_state_dict_shards(shard_optimizer_checkpoint(sd, size_per_shard), checkpoint, index_file,
                                           states_name, True)
            index_file.append_meta_data("total_size", total)
            index_file.write_index_file(save_index_file)
        dist.barrier()

    def load_unsharded_optimizer(self, optimizer: OptimizerWrapper, checkpoint: str, low_cpu_mem_mode: bool = True,
                                 num_threads: int = 1):
        from ...checkpoint_io.utils import load_state_dict

        optimizer.load_state_dict(load_state_dict(checkpoint))

    def load_sharded_optimizer(self, optimizer: OptimizerWrapper, index_file_path: str, prefix: str = "",
                               low_cpu_mem_mode: bool = True, num_threads: int = 1):
        from pathlib import Path

        from ...checkpoint_io.index_file import CheckpointIndexFile
        from ...checkpoint_io.utils import load_shard_state_dict

        idx = CheckpointIndexFile.from_file(index_file_path)
        groups = torch.load(idx.get_param_group_filename(), weights_only=False)
        state = {}
        for fn in idx.get_checkpoint_filenames():
            state.update(load_shard_state_dict(Path(fn)))
        optimizer.load_state_dict({"state": state, "param_groups": groups})

    def load_unsharded_model(self, model, checkpoint, strict=True, low_cpu_mem_mode=True, num_threads=1):
        super().load_unsharded_model(model, checkpoint, strict, low_cpu_mem_mode, num_threads)
        if hasattr(model, "update_master_params"):
            model.update_master_params()

    def load_sharded_model(self, model, checkpoint_index_file, strict=False, use_safetensors=False,
                           load_sub_module=True, low_cpu_mem_mode=True, num_threads=1):
        super().load_sharded_model(model, checkpoint_index_file, strict, use_safetensors, load_sub_module,
                                   low_cpu_mem_mode, num_threads)
        if hasattr(model, "update_master_params"):      # the fp32 master shards must follow the loaded weights
            model.update_master_params()

    def save_unsharded_model(self, model, checkpoint, gather_dtensor, use_safetensors, use_async=False):
        if dist.get_rank() == 0:
            super().save_unsharded_model(model, checkpoint, gather_dtensor, use_safetensors, use_async)
        dist.barrier()

    def save_sharded_model(self, model, checkpoint_path, gather_dtensor=False, prefix=None, max_shard_size=1024,
                           use_safetensors=False, use_async=False):
        if dist.get_rank() == 0:
            super().save_sharded_model(model, checkpoint_path, gather_dtensor, prefix, max_shard_size,
                                       use_safetensors, use_async)
        dist.barrier()


class LowLevelZeroPlugin(DPPluginBase):
    """
    >>> plugin = LowLevelZeroPlugin(stage=2, precision="bf16", max_norm=1.0)
    >>> model, optimizer, *_ = Booster(plugin=plugin).boost(model, optimizer)
    """

    def __init__(self, stage: int = 1, precision: str = "fp16", initial_scale: float = 2**32, min_scale: float = 1,
                 growth_factor: float = 2, backoff_factor: float = 0.5, growth_interval: int = 1000,
                 hysteresis: int = 2, max_scale: float = 2**32, max_norm: float = 0.0, norm_type: float = 2.0,
                 reduce_bucket_size_in_m: int = 12, communication_dtype: Optional[torch.dtype] = None,
                 overlap_communication: bool = True, overlap_allgather: bool = False, cpu_offload: bool = False, offload_optim_frac: float = 1.0,
                 master_weights: bool = True, skip_untouched_params: bool = False, verbose: bool = False,
                 cast_inputs: bool = True,
                 fp8_communication: bool = False, use_fp8: bool = False, extra_dp_size: int = 1) -> None:
        super().__init__()
        assert stage in (1, 2), "LowLevelZeroPlugin only supports stage 1/2 training"
        assert precision in SUPPORTED_PRECISION, "LowLevelZeroPlugin only supports amp training"
        assert norm_type == 2.0, "LowLevelZeroPlugin only supports norm_type=2.0 now"
        self.stage, self.precision = stage, precision
        self.extra_dp_size = extra_dp_size
        if extra_dp_size > 1:
            assert dist.get_world_size() % extra_dp_size == 0
            inner = dist.get_world_size() // extra_dp_size
            self.pg_mesh = DeviceMesh(extra_dp=extra_dp_size, dp=inner)
            self.dp_group = self.pg_mesh.group("dp")
            self.extra_dp_group = self.pg_mesh.group("extra_dp")
        else:
            self.pg_mesh, self.dp_group, self.extra_dp_group = None, None, None
        self.zero_optim_kwargs = dict(
            initial_scale=initial_scale, min_scale=min_scale, growth_factor=growth_factor,
            backoff_factor=backoff_factor, growth_interval=growth_interval, hysteresis=hysteresis,
            max_scale=max_scale, clip_grad_norm=max_norm, reduce_bucket_size=reduce_bucket_size_in_m * 1024 * 1024,
            communication_dtype=communication_dtype, overlap_communication=overlap_communication,
            partition_grad=(stage == 2), cpu_offload=cpu_offload, offload_optim_frac=offload_optim_frac,
            master_weights=master_weights, skip_untouched_params=skip_untouched_params,
            overlap_allgather=overlap_allgather, fp8_communication=fp8_communication)
        self.verbose = verbose
        self.cast_inputs = cast_inputs
        self.use_fp8 = use_fp8
        self.lora_enabled = False
        self.logger = get_dist_logger()

    def support_no_sync(self) -> bool:
        return self.stage == 1

    def support_lora(self) -> bool:
        return True

    def control_precision(self) -> bool:
        return True

    def supported_precisions(self) -> List[str]:
        return SUPPORTED_PRECISION

    def control_device(self) -> bool:
        return True

    def supported_devices(self) -> List[str]:
        return ["cuda", "cpu"]

    def configure(self, model: nn.Module, optimizer: Optional[Optimizer] = None, criterion: Optional[Callable] = None,
                  dataloader: Optional[DataLoader] = None, lr_scheduler: Optional[LRScheduler] = None):
        if not isinstance(model, ModelWrapper):
            model = LowLevelZeroModel(model, self.precision, overlap_allgather=self.zero_optim_kwargs["overlap_allgather"],
                                      cast_inputs=self.cast_inputs, use_fp8=self.use_fp8)
        if optimizer is not None and not isinstance(optimizer, OptimizerWrapper):
            # the model was cast/moved: re-point the optimizer at the live parameters
            live = [p for p in model.parameters() if p.requires_grad]
            if len(optimizer.param_groups) == 1:
                optimizer.param_groups[0]["params"] = live
            optimizer.state.clear()
            optimizer = LowLevelZeroOptimizer(optimizer, **self.zero_optim_kwargs, verbose=self.verbose,
                                              dp_process_group=self.dp_group, extra_dp_group=self.extra_dp_group)
            optimizer.model = model
            import weakref

            model._zero_optimizer = weakref.ref(optimizer)
        return model, optimizer, criterion, dataloader, lr_scheduler

    def control_checkpoint_io(self) -> bool:
        return True

    def get_checkpoint_io(self) -> CheckpointIO:
        return LowLevelZeroCheckpointIO()

    def no_sync(self, model: nn.Module, optimizer: OptimizerWrapper) -> Iterator[None]:
        assert isinstance(optimizer, LowLevelZeroOptimizer)
        return optimizer.no_sync()

    def enable_lora(self, model: nn.Module, pretrained_dir: Optional[str] = None, lora_config: Optional[Dict] = None,
                    bnb_quantization_config=None) -> nn.Module:
        from ..lora import apply_lora

        self.lora_enabled = True
        if bnb_quantization_config is not None:
            from ...quantization import quantize_model

            model = quantize_model(model, bnb_quantization_config)
        return apply_lora(model, lora_config, pretrained_dir)
