"""`MoeParallelInfo`: the ep x dp layout an expert parameter lives on (reference `tensor/moe_tensor/moe_info.py`)."""
from __future__ import annotations

from typing import List, Optional

import torch.distributed as dist

__all__ = ["MoeParallelInfo"]


class MoeParallelInfo:
    """Ranks are laid out `[pp, dp, ep]` (`ep_inside=True`, expert-parallel ranks adjacent — one NVSwitch hop
    either way) or `[pp, ep, dp]`.  Holds the EP / DP group of the calling rank and their rank lists."""

    def __init__(self, ep_inside: bool, ep_size: int, dp_size: int, pp_size: int = 1) -> None:
        self.ep_inside, self.ep_size, self.dp_size, self.pp_size = ep_inside, ep_size, dp_size, pp_size
        self.ep_group = self.dp_group = None
        self.ep_group_ranks: Optional[List[int]] = None
        self.dp_group_ranks: Optional[List[int]] = None
        self.ep_rank = self.dp_rank = 0
        if not dist.is_initialized():
            return
        world, me = dist.get_world_size(), dist.get_rank()
        assert ep_size * dp_size * pp_size == world, f"ep {ep_size} x dp {dp_size} x pp {pp_size} != world {world}"
        per_stage = ep_size * dp_size
        for stage in range(pp_size):
            base = stage * per_stage
            for d in range(dp_size):
                ranks = [base + (d * ep_size + e if ep_inside else e * dp_size + d) for e in range(ep_size)]
                g = dist.new_group(ranks)
                if me in ranks:
                    self.ep_group, self.ep_group_ranks, self.ep_rank = g, ranks, ranks.index(me)
            for e in range(ep_size):
                ranks = [base + (d * ep_size + e if ep_inside else e * dp_size + d) for d in range(dp_size)]
                g = dist.new_group(ranks)
                if me in ranks:
                    self.dp_group, self.dp_group_ranks, self.dp_rank = g, ranks, ranks.index(me)

    def __repr__(self) -> str:
        return (f"MoeParallelInfo(ep={self.ep_size}, dp={self.dp_size}, pp={self.pp_size}, ep_inside={self.ep_inside}, "
                f"ep_ranks={self.ep_group_ranks}, dp_ranks={self.dp_group_ranks})")
