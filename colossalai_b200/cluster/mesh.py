"""N-D cartesian rank mesh with lazily-created, cached process groups.

Parity: reference `colossalai/cluster/process_group_mesh.py:25-276` (`ProcessGroupMesh`: ravel/unravel,
`get_group_along_axis`, `create_group_along_axis`, wrap-around neighbours for PP).  The H100-first addition
is `DeviceMesh`: the same object with *named* axes (dp, pp, ep, sp, tp) so higher layers ask for
`mesh.group("tp")` and fused kernels can cache symmetric-memory handles per axis group.
"""
from __future__ import annotations

import gc
import itertools
from functools import reduce
from operator import mul
from typing import Dict, List, Optional, Sequence, Tuple, Union

import numpy as np
import torch.distributed as dist
from torch.distributed import ProcessGroup

__all__ = ["ProcessGroupMesh", "DeviceMesh", "prod"]


def prod(nums: Sequence[int]) -> int:
    return reduce(mul, nums, 1)


class ProcessGroupMesh:
    """Cartesian mesh over the world ranks.  Rank r has coordinate `unravel(r, shape)` (row-major: the last
    axis varies fastest, so make the most bandwidth-hungry axis — tp — last)."""

    def __init__(self, *size: int) -> None:
        assert dist.is_initialized(), "initialise torch.distributed before building a mesh"
        world = dist.get_world_size()
        assert prod(size) == world, f"mesh {size} does not cover world size {world}"
        self._shape = tuple(int(s) for s in size)
        self._rank = dist.get_rank()
        self._coord = self.unravel(self._rank, self._shape)
        self._ranks_to_group: Dict[Tuple[int, ...], ProcessGroup] = {}
        self._group_to_ranks: Dict[ProcessGroup, Tuple[int, ...]] = {}
        self._axis_group_cache: Dict[tuple, ProcessGroup] = {}

    # ------------------------------------------------------------------ geometry
    @property
    def shape(self) -> Tuple[int, ...]:
        return self._shape

    @property
    def rank(self) -> int:
        return self._rank

    def size(self, dim: Optional[int] = None) -> Union[int, Tuple[int, ...]]:
        return self._shape if dim is None else self._shape[dim]

    def coordinate(self, dim: Optional[int] = None) -> Union[int, Tuple[int, ...]]:
        return self._coord if dim is None else self._coord[dim]

    @staticmethod
    def unravel(rank: int, shape: Tuple[int, ...]) -> Tuple[int, ...]:
        return tuple(int(x) for x in np.unravel_index(rank, shape))

    @staticmethod
    def ravel(coord: Tuple[int, ...], shape: Tuple[int, ...], mode: str = "raise") -> int:
        assert mode in ("raise", "wrap", "clip")
        return int(np.ravel_multi_index(coord, shape, mode))

    # ------------------------------------------------------------------ groups
    def _get_group(self, ranks: Sequence[int], backend: Optional[str] = None) -> ProcessGroup:
        ranks = tuple(sorted(ranks))
        if ranks not in self._ranks_to_group:
            group = dist.new_group(list(ranks), backend=backend)
            self._ranks_to_group[ranks] = group
            if group is not None and group != dist.GroupMember.NON_GROUP_MEMBER:
                self._group_to_ranks[group] = ranks
        return self._ranks_to_group[ranks]

    def get_ranks_in_group(self, group: ProcessGroup) -> List[int]:
        if group in self._group_to_ranks:
            return list(self._group_to_ranks[group])
        return dist.get_process_group_ranks(group)

    @staticmethod
    def get_coords_along_axis(
        base_coord: Tuple[int, ...], axis: Union[int, Sequence[int]], indices_at_axis: Union[List[int], List[List[int]]]
    ) -> List[Tuple[int, ...]]:
        if isinstance(axis, int):
            axis = [axis]
            indices_at_axis = [indices_at_axis]  # type: ignore[list-item]
        coords = []
        for combo in itertools.product(*indices_at_axis):
            c = list(base_coord)
            for a, i in zip(axis, combo):
                c[a] = i
            coords.append(tuple(c))
        return coords

    def create_group_along_axis(
        self,
        axis: Union[int, Sequence[int]],
        indices_at_axis: Optional[Union[List[int], List[List[int]]]] = None,
        backend: Optional[str] = None,
    ) -> ProcessGroup:
        """Collectively create *every* group along `axis` (all ranks must call this in the same order) and
        return the one that contains the calling rank."""
        axes = [axis] if isinstance(axis, int) else list(axis)
        if indices_at_axis is None:
            idx = [list(range(self._shape[a])) for a in axes]
        else:
            idx = [indices_at_axis] if isinstance(axis, int) else list(indices_at_axis)  # type: ignore[list-item]
        other_axes = [a for a in range(len(self._shape)) if a not in axes]
        target = None
        for base in itertools.product(*[range(self._shape[a]) for a in other_axes]):
            base_coord = [0] * len(self._shape)
            for a, v in zip(other_axes, base):
                base_coord[a] = v
            coords = self.get_coords_along_axis(tuple(base_coord), axes, idx)
            ranks = tuple(self.ravel(c, self._shape) for c in coords)
            group = self._get_group(ranks, backend)
            if self._rank in ranks:
                target = group
        assert target is not None
        return target

    def get_group_along_axis(
        self,
        axis: Union[int, Sequence[int]],
        indices_at_axis: Optional[Union[List[int], List[List[int]]]] = None,
        backend: Optional[str] = None,
    ) -> ProcessGroup:
        axes = (axis,) if isinstance(axis, int) else tuple(axis)
        key = (axes, repr(indices_at_axis), backend)
        if key not in self._axis_group_cache:
            self._axis_group_cache[key] = self.create_group_along_axis(axis, indices_at_axis, backend)
        return self._axis_group_cache[key]

    def destroy_mesh_process_groups(self) -> None:
        for group in list(self._group_to_ranks.keys()):
            try:
                dist.destroy_process_group(group)
            except Exception:
                pass
        self._ranks_to_group.clear()
        self._group_to_ranks.clear()
        self._axis_group_cache.clear()
        gc.collect()


class DeviceMesh(ProcessGroupMesh):
    """Named-axis mesh.  `DeviceMesh(dp=2, pp=1, tp=4)`; axis order = keyword order (last is fastest)."""

    CANONICAL = ("dp", "pp", "ep", "sp", "tp")

    def __init__(self, **axes: int) -> None:
        if not axes:
            axes = {"dp": dist.get_world_size()}
        self.axis_names: Tuple[str, ...] = tuple(axes.keys())
        super().__init__(*axes.values())

    @classmethod
    def from_sizes(cls, order: Sequence[str], **sizes: int) -> "DeviceMesh":
        return cls(**{n: sizes.get(n, 1) for n in order})

    def axis(self, name: str) -> int:
        return self.axis_names.index(name)

    def has_axis(self, name: str) -> bool:
        return name in self.axis_names

    def axis_size(self, name: str) -> int:
        return self._shape[self.axis(name)] if name in self.axis_names else 1

    def axis_rank(self, name: str) -> int:
        return self._coord[self.axis(name)] if name in self.axis_names else 0

    def group(self, *names: str, backend: Optional[str] = None) -> ProcessGroup:
        """Group spanning one or several named axes (e.g. `group("dp", "sp")` = the mixed dp×sp group)."""
        axes = [self.axis(n) for n in names]
        return self.get_group_along_axis(axes[0] if len(axes) == 1 else axes, backend=backend)

    def neighbor(self, name: str, offset: int) -> int:
        """World rank of the neighbour at `offset` along `name` (wraps around — used for PP prev/next)."""
        c = list(self._coord)
        a = self.axis(name)
        c[a] = (c[a] + offset) % self._shape[a]
        return self.ravel(tuple(c), self._shape)

    def __repr__(self) -> str:
        dims = ", ".join(f"{n}={s}" for n, s in zip(self.axis_names, self._shape))
        return f"DeviceMesh({dims}; rank={self._rank} coord={self._coord})"
