"""Logical device mesh with an alpha-beta communication cost model (used by the auto-parallel / layout-conversion code).

Parity: reference `colossalai/device/device_mesh.py:22-525` (`DeviceMesh(physical_mesh_id, mesh_shape, mesh_alpha,
mesh_beta, init_process_group)`, per-axis process groups, `global_rank_to_local_rank`, `flatten`, collective cost
formulas).  The runtime mesh of the training stack is `colossalai_b200.cluster.DeviceMesh` (named axes); this class is
the analysable one: it can exist without any process group and prices collectives.

Default alpha/beta describe an NVSwitch domain: every pair of GPUs sees the same ~1.5 us launch+sync latency and
770 GB/s per direction, so a logical axis costs the same wherever it is placed (no ring-per-link penalty).
"""
from __future__ import annotations

import operator
from functools import reduce
from typing import Dict, List, Optional, Sequence, Union

import torch
import torch.distributed as dist
from torch.distributed import ProcessGroup

__all__ = ["DeviceMesh"]

NVSWITCH_ALPHA = 1.5e-6            # seconds per collective step
NVSWITCH_BETA = 1.0 / 770e9        # seconds per byte per direction


class DeviceMesh:
    def __init__(self, physical_mesh_id: torch.Tensor, mesh_shape: Optional[Sequence[int]] = None,
                 logical_mesh_id: Optional[torch.Tensor] = None, mesh_alpha: Optional[List[float]] = None,
                 mesh_beta: Optional[List[float]] = None, init_process_group: bool = False,
                 device: str = "cuda") -> None:
        self._physical_mesh_id = torch.as_tensor(physical_mesh_id).flatten()
        if logical_mesh_id is None:
            assert mesh_shape is not None, "either mesh_shape or logical_mesh_id is required"
            self._mesh_shape = tuple(mesh_shape)
            self._logical_mesh_id = self._physical_mesh_id.reshape(self._mesh_shape)
        else:
            self._logical_mesh_id = torch.as_tensor(logical_mesh_id)
            self._mesh_shape = tuple(self._logical_mesh_id.shape)
        assert reduce(operator.mul, self._mesh_shape, 1) == self._physical_mesh_id.numel(), \
            "mesh shape does not match the number of devices"
        nd = len(self._mesh_shape)
        self.mesh_alpha = list(mesh_alpha) if mesh_alpha is not None else [NVSWITCH_ALPHA] * nd
        self.mesh_beta = list(mesh_beta) if mesh_beta is not None else [NVSWITCH_BETA] * nd
        assert len(self.mesh_alpha) == nd and len(self.mesh_beta) == nd
        self._device = device
        self._global_to_local: Dict[int, List[int]] = {}
        for coord in torch.cartesian_prod(*[torch.arange(s) for s in self._mesh_shape]).reshape(-1, nd).tolist():
            self._global_to_local[int(self._logical_mesh_id[tuple(coord)])] = coord
        self._process_group_dict: Dict[int, Dict[int, ProcessGroup]] = {}
        self._ranks_in_group: Dict[int, Dict[int, List[int]]] = {}
        self._is_initialized = False
        self._collate_groups()
        if init_process_group:
            self.init_logical_process_group()

    # ---- basic properties
    @property
    def shape(self) -> torch.Size:
        return torch.Size(self._mesh_shape)

    @property
    def num_devices(self) -> int:
        return int(self._physical_mesh_id.numel())

    @property
    def logical_mesh_id(self) -> torch.Tensor:
        return self._logical_mesh_id

    @property
    def is_initialized(self) -> bool:
        return self._is_initialized

    @property
    def device(self) -> str:
        return self._device

    # ---- groups
    def _collate_groups(self) -> None:
        nd = len(self._mesh_shape)
        for rank, coord in self._global_to_local.items():
            self._ranks_in_group[rank] = {}
            for axis in range(nd):
                idx = [slice(None) if a == axis else coord[a] for a in range(nd)]
                self._ranks_in_group[rank][axis] = self._logical_mesh_id[tuple(idx)].flatten().tolist()

    def init_logical_process_group(self) -> None:
        """Collective: every rank creates every axis group (torch.distributed requires it)."""
        assert dist.is_initialized(), "torch.distributed must be initialised first"
        seen: Dict[tuple, ProcessGroup] = {}
        for rank in sorted(self._ranks_in_group):
            for axis, ranks in self._ranks_in_group[rank].items():
                key = (axis, tuple(ranks))
                if key not in seen:
                    seen[key] = dist.new_group(ranks)
                self._process_group_dict.setdefault(rank, {})[axis] = seen[key]
        self._is_initialized = True

    @staticmethod
    def from_process_group(process_group: Union[ProcessGroup, List[ProcessGroup]]) -> "DeviceMesh":
        groups = process_group if isinstance(process_group, (list, tuple)) else [process_group]
        shape = [dist.get_world_size(g) for g in groups]
        world = reduce(operator.mul, shape, 1)
        mesh = DeviceMesh(torch.arange(world), shape)
        me = dist.get_rank()
        for axis, g in enumerate(groups):
            mesh._process_group_dict.setdefault(me, {})[axis] = g
        mesh._is_initialized = True
        return mesh

    def get_process_group(self, axis: int, global_rank: Optional[int] = None) -> ProcessGroup:
        rank = dist.get_rank() if global_rank is None else global_rank
        return self._process_group_dict[rank][axis]

    def get_process_group_for_all_axes(self, global_rank: Optional[int] = None) -> Dict[int, ProcessGroup]:
        rank = dist.get_rank() if global_rank is None else global_rank
        return self._process_group_dict[rank]

    def get_ranks_in_process_group(self, axis: int, global_rank: Optional[int] = None) -> List[int]:
        rank = (dist.get_rank() if dist.is_initialized() else 0) if global_rank is None else global_rank
        return self._ranks_in_group[rank][axis]

    def global_rank_to_local_rank(self, rank: int, axis: Optional[int] = None) -> Union[List[int], int]:
        coord = self._global_to_local[rank]
        return coord if axis is None else coord[axis]

    def flatten(self) -> "DeviceMesh":
        """1-D view of the same devices (cost = the slowest axis)."""
        return DeviceMesh(self._physical_mesh_id, (self.num_devices,), mesh_alpha=[max(self.mesh_alpha)],
                          mesh_beta=[max(self.mesh_beta)], device=self._device)

    def __deepcopy__(self, memo) -> "DeviceMesh":
        new = DeviceMesh(self._physical_mesh_id.clone(), self._mesh_shape, mesh_alpha=list(self.mesh_alpha),
                         mesh_beta=list(self.mesh_beta), device=self._device)
        new._process_group_dict = self._process_group_dict      # process groups cannot be copied
        new._is_initialized = self._is_initialized
        return new

    # ---- alpha-beta costs (seconds); num_bytes = size of the FULL tensor taking part in the collective
    def all_gather_cost(self, num_bytes: float, mesh_dim: int) -> float:
        n = self._mesh_shape[mesh_dim]
        return self.mesh_alpha[mesh_dim] + self.mesh_beta[mesh_dim] * (n - 1) / n * num_bytes

    def all_reduce_cost(self, num_bytes: float, mesh_dim: int) -> float:
        n = self._mesh_shape[mesh_dim]
        return self.mesh_alpha[mesh_dim] + self.mesh_beta[mesh_dim] * 2 * (n - 1) / n * num_bytes

    def reduce_scatter_cost(self, num_bytes: float, mesh_dim: int) -> float:
        n = self._mesh_shape[mesh_dim]
        return self.mesh_alpha[mesh_dim] + self.mesh_beta[mesh_dim] * (n - 1) / n * num_bytes

    def all_to_all_cost(self, num_bytes: float, mesh_dim: int) -> float:
        n = self._mesh_shape[mesh_dim]
        penalty = n / 2.0
        return self.mesh_alpha[mesh_dim] + self.mesh_beta[mesh_dim] * (n - 1) / n / n * num_bytes * penalty

    def __repr__(self) -> str:
        return f"DeviceMesh(shape={tuple(self._mesh_shape)}, devices={self._physical_mesh_id.tolist()})"
