"""Distributed bring-up.

Parity: reference `colossalai/initialize.py:33-197` (launch / launch_from_torch / launch_from_slurm /
launch_from_openmpi).  Design differences (H100-first):
  * one process per GPU, NCCL on CUDA boxes, gloo on CPU boxes (the plumbing tier of the test-suite);
  * we do NOT force CUDA_DEVICE_MAX_CONNECTIONS=1 — overlap is obtained with explicit streams and fused
    compute+collective kernels rather than launch-order tricks;
  * rendezvous defaults to 127.0.0.1 because container hostnames may not resolve.
"""
from __future__ import annotations

import os
import warnings
from typing import Optional

import torch
import torch.distributed as dist

from .accelerator import get_accelerator
from .logging import get_dist_logger
from .utils.common import set_seed


def launch(
    rank: int,
    world_size: int,
    host: str,
    port: int,
    backend: Optional[str] = None,
    local_rank: Optional[int] = None,
    seed: int = 1024,
    verbose: bool = True,
    timeout_s: int = 1800,
) -> None:
    """Initialise torch.distributed and bind this process to its device."""
    acc = get_accelerator()
    if backend is None:
        backend = acc.communication_backend
    if not dist.is_initialized():
        import datetime

        init_method = f"tcp://[{host}]:{port}" if ":" in host else f"tcp://{host}:{port}"
        kwargs = {}
        if backend == "nccl" and torch.cuda.is_available():
            lr = local_rank if local_rank is not None else rank % max(torch.cuda.device_count(), 1)
            torch.cuda.set_device(lr)
            kwargs["device_id"] = torch.device("cuda", lr)
        dist.init_process_group(
            backend=backend,
            init_method=init_method,
            rank=rank,
            world_size=world_size,
            timeout=datetime.timedelta(seconds=timeout_s),
            **kwargs,
        )
    if local_rank is None:
        n = acc.device_count()
        local_rank = rank % n if n > 0 else 0
    acc.set_device(local_rank)
    set_seed(seed)
    if verbose:
        get_dist_logger().info(
            f"distributed environment initialised: world={world_size} backend={backend} device={acc.name}",
            ranks=[0],
        )


def launch_from_torch(backend: Optional[str] = None, seed: int = 1024, verbose: bool = True) -> None:
    """Read RANK / LOCAL_RANK / WORLD_SIZE / MASTER_* exported by torchrun."""
    try:
        rank = int(os.environ["RANK"])
        local_rank = int(os.environ.get("LOCAL_RANK", rank))
        world_size = int(os.environ["WORLD_SIZE"])
        host = os.environ.get("MASTER_ADDR", "127.0.0.1")
        port = int(os.environ.get("MASTER_PORT", 29500))
    except KeyError as e:  # pragma: no cover - message path
        raise RuntimeError(f"launch_from_torch: environment variable {e} missing (run under torchrun)") from e
    launch(rank, world_size, host, port, backend, local_rank, seed, verbose)


def launch_from_slurm(host: str, port: int, backend: Optional[str] = None, seed: int = 1024, verbose: bool = True):
    try:
        rank = int(os.environ["SLURM_PROCID"])
        world_size = int(os.environ["SLURM_NPROCS"])
    except KeyError as e:  # pragma: no cover
        raise RuntimeError(f"launch_from_slurm: {e} missing (run under srun)") from e
    local_rank = int(os.environ.get("SLURM_LOCALID", rank))
    launch(rank, world_size, host, port, backend, local_rank, seed, verbose)


def launch_from_openmpi(host: str, port: int, backend: Optional[str] = None, seed: int = 1024, verbose: bool = True):
    try:
        rank = int(os.environ["OMPI_COMM_WORLD_RANK"])
        local_rank = int(os.environ["OMPI_COMM_WORLD_LOCAL_RANK"])
        world_size = int(os.environ["OMPI_COMM_WORLD_SIZE"])
    except KeyError as e:  # pragma: no cover
        raise RuntimeError(f"launch_from_openmpi: {e} missing (run under mpirun)") from e
    launch(rank, world_size, host, port, backend, local_rank, seed, verbose)


def shutdown() -> None:
    if dist.is_initialized():
        try:
            dist.destroy_process_group()
        except Exception as e:  # pragma: no cover
            warnings.warn(f"destroy_process_group failed: {e}")
