"""ShardConfig: the one dataclass that carries parallel groups and feature flags to policies and layers.

Parity: reference `colossalai/shardformer/shard/shard_config.py:13-130`.  Additions: `comm_backend`
("nccl" | "fused") selects the fused compute+collective kernels, `seq_dim` is the token dim of activations
(token-major models use 0).
"""
from __future__ import annotations

from dataclasses import dataclass, field
from typing import Any, Dict, Optional

import torch.distributed as dist
from torch.distributed import ProcessGroup

from .grad_ckpt_config import GradientCheckpointConfig

__all__ = ["ShardConfig", "SUPPORT_SP_MODE"]

SUPPORT_SP_MODE = ["split_gather", "ring", "all_to_all", "ring_attn"]


@dataclass
class ShardConfig:
    tensor_parallel_process_group: Optional[ProcessGroup] = None
    sequence_parallel_process_group: Optional[ProcessGroup] = None
    pipeline_stage_manager: Optional[Any] = None
    enable_tensor_parallelism: bool = True
    enable_all_optimization: bool = False
    enable_fused_normalization: bool = False
    enable_flash_attention: bool = False
    enable_jit_fused: bool = False
    enable_sequence_parallelism: bool = False
    sequence_parallelism_mode: Optional[str] = None
    parallel_output: bool = True
    make_vocab_size_divisible_by: int = 64
    gradient_checkpoint_config: Optional[GradientCheckpointConfig] = None
    extra_kwargs: Dict[str, Any] = field(default_factory=dict)
    fp8_communication: bool = False
    # expert / mesh info
    ep_group: Optional[ProcessGroup] = None
    moe_dp_group: Optional[ProcessGroup] = None
    sp_axis: Optional[int] = None
    pg_mesh: Optional[Any] = None
    inner_ring_size: Optional[int] = None
    # H100-native knobs
    comm_backend: str = "nccl"
    seq_dim: int = 0
    use_zbv: bool = False

    @property
    def tensor_parallel_size(self) -> int:
        return self._tensor_parallel_size

    @property
    def sequence_parallel_size(self) -> int:
        return self._sequence_parallel_size

    @property
    def expert_parallel_size(self) -> int:
        return self._expert_parallel_size

    def __post_init__(self) -> None:
        if self.enable_all_optimization:
            self._turn_on_all_optimization()
        if self.enable_sequence_parallelism:
            self.sequence_parallelism_mode = self.sequence_parallelism_mode or "split_gather"
            assert self.sequence_parallelism_mode in SUPPORT_SP_MODE, (
                f"sequence parallelism mode {self.sequence_parallelism_mode} not in {SUPPORT_SP_MODE}")
            if self.sequence_parallelism_mode in ("split_gather", "ring"):
                assert self.enable_tensor_parallelism, (
                    f"sequence parallelism mode {self.sequence_parallelism_mode} requires tensor parallelism")
                # these modes share the TP group
                self.sequence_parallel_process_group = self.tensor_parallel_process_group
        elif self.sequence_parallelism_mode:
            self.sequence_parallelism_mode = None
        init = dist.is_initialized()
        self._tensor_parallel_size = (dist.get_world_size(self.tensor_parallel_process_group)
                                      if (init and self.enable_tensor_parallelism) else 1)
        self._sequence_parallel_size = (dist.get_world_size(self.sequence_parallel_process_group)
                                        if (init and self.enable_sequence_parallelism) else 1)
        self._expert_parallel_size = dist.get_world_size(self.ep_group) if (init and self.ep_group is not None) else 1
        assert self.comm_backend in ("nccl", "fused")

    def _turn_on_all_optimization(self) -> None:
        self.enable_fused_normalization = True
        self.enable_flash_attention = True
        self.enable_jit_fused = True
        if self.enable_tensor_parallelism and dist.is_initialized() and \
                dist.get_world_size(self.tensor_parallel_process_group) > 1:
            self.enable_sequence_parallelism = True
            self.sequence_parallelism_mode = self.sequence_parallelism_mode or "split_gather"

    @property
    def sp_mode(self) -> Optional[str]:
        return self.sequence_parallelism_mode if self.enable_sequence_parallelism else None

    @property
    def tp_group(self):
        return self.tensor_parallel_process_group if self.enable_tensor_parallelism else None

    @property
    def sp_group(self):
        return self.sequence_parallel_process_group if self.enable_sequence_parallelism else None
