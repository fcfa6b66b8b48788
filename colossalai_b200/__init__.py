"""colossalai_b200 — a H100-native (sm_90a) hybrid-parallel training & inference framework.

Capability parity target: hpcaitech/ColossalAI 0.5.0 (see SURVEY.md).  The public surface mirrors the
reference's (`launch*`, `Booster` + plugins, `ShardFormer`, pipeline schedules, ZeRO / Gemini, inference
engine) while the compute path is hand-written CUDA for sm_90a (wgmma/TMA) plus fused
compute+collective kernels over NVLink peer memory; NCCL is the control plane and the multi-node fallback.
"""
from .initialize import (
    launch,
    launch_from_openmpi,
    launch_from_slurm,
    launch_from_torch,
)
from .accelerator import get_accelerator
from .logging import get_dist_logger, disable_existing_loggers

__version__ = "0.1.0"

__all__ = [
    "launch",
    "launch_from_torch",
    "launch_from_slurm",
    "launch_from_openmpi",
    "get_accelerator",
    "get_dist_logger",
    "disable_existing_loggers",
    "__version__",
]
