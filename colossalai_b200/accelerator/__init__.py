"""Device abstraction.  Parity: reference `colossalai/accelerator/{api,base_accelerator,cuda_accelerator,
cpu_accelerator}.py`.  Only two targets exist here by design: the H100 (`cuda`, NCCL) and the CPU plumbing tier
(`cpu`, gloo) — no multi-vendor dispatch."""
from __future__ import annotations

import contextlib
import random
from typing import Any, Optional

import numpy as np
import torch

__all__ = ["BaseAccelerator", "CudaAccelerator", "CpuAccelerator", "get_accelerator", "set_accelerator", "auto_set_accelerator"]


class _NullEvent:
    """Event of a device without asynchronous streams (the CPU tier): everything has already happened."""

    def record(self, stream=None) -> None:
        pass

    def wait(self, stream=None) -> None:
        pass

    def synchronize(self) -> None:
        pass

    def query(self) -> bool:
        return True

    def elapsed_time(self, other) -> float:
        return 0.0


class _NullStream:
    """Stream stand-in of the CPU tier: work is synchronous, so every ordering primitive is a no-op."""

    def wait_event(self, event) -> None:
        pass

    def wait_stream(self, stream) -> None:
        pass

    def record_event(self, event=None):
        return event if event is not None else _NullEvent()

    def synchronize(self) -> None:
        pass

    def query(self) -> bool:
        return True


class BaseAccelerator:
    name = "base"
    communication_backend = "gloo"
    support_set_device = False

    # ---- device
    def get_current_device(self) -> torch.device:
        raise NotImplementedError

    def current_device(self) -> int:
        return 0

    def set_device(self, device: Optional[int] = None) -> None:
        pass

    def device_count(self) -> int:
        return 0

    def synchronize(self, device=None) -> None:
        pass

    def get_device_name(self, device=None) -> str:
        return self.name

    # ---- RNG
    def manual_seed(self, seed: int) -> None:
        torch.manual_seed(seed)

    def manual_seed_all(self, seed: int) -> None:
        torch.manual_seed(seed)

    def seed(self) -> None:
        torch.seed()

    def get_rng_state(self, device="cpu"):
        return torch.get_rng_state()

    def set_rng_state(self, state, device="cpu") -> None:
        torch.set_rng_state(state)

    # ---- memory
    def empty_cache(self) -> None:
        pass

    def memory_allocated(self, device=None) -> int:
        return 0

    def max_memory_allocated(self, device=None) -> int:
        return 0

    def memory_reserved(self, device=None) -> int:
        return 0

    def max_memory_reserved(self, device=None) -> int:
        return 0

    def reset_peak_memory_stats(self, device=None) -> None:
        pass

    def mem_get_info(self, device=None):
        import psutil

        vm = psutil.virtual_memory()
        return vm.available, vm.total

    def get_device_capability(self, device=None):
        return (0, 0)

    def set_per_process_memory_fraction(self, fraction: float, device=None) -> None:
        pass

    # ---- streams / events
    def Stream(self, *a, **k):
        return _NullStream()

    def Event(self, *a, **k):
        return _NullEvent()

    def current_stream(self, device=None):
        return _NullStream()

    def stream(self, stream_):
        return contextlib.nullcontext()

    # ---- amp
    def autocast(self, enabled: bool = True, dtype: torch.dtype = torch.bfloat16, cache_enabled: bool = True):
        return torch.autocast(self.name, dtype=dtype, enabled=enabled, cache_enabled=cache_enabled)


class CudaAccelerator(BaseAccelerator):
    name = "cuda"
    communication_backend = "nccl"
    support_set_device = True

    def get_current_device(self) -> torch.device:
        return torch.device("cuda", torch.cuda.current_device())

    def current_device(self) -> int:
        return torch.cuda.current_device()

    def set_device(self, device: Optional[int] = None) -> None:
        if device is None:
            import torch.distributed as dist

            device = (dist.get_rank() if dist.is_initialized() else 0) % self.device_count()
        torch.cuda.set_device(device)

    def device_count(self) -> int:
        return torch.cuda.device_count()

    def synchronize(self, device=None) -> None:
        torch.cuda.synchronize(device)

    def get_device_name(self, device=None) -> str:
        return torch.cuda.get_device_name(device)

    def manual_seed(self, seed: int) -> None:
        torch.cuda.manual_seed(seed)

    def manual_seed_all(self, seed: int) -> None:
        torch.cuda.manual_seed_all(seed)

    def get_rng_state(self, device="cuda"):
        return torch.cuda.get_rng_state(device)

    def set_rng_state(self, state, device="cuda") -> None:
        torch.cuda.set_rng_state(state, device)

    def empty_cache(self) -> None:
        torch.cuda.empty_cache()

    def memory_allocated(self, device=None) -> int:
        return torch.cuda.memory_allocated(device)

    def max_memory_allocated(self, device=None) -> int:
        return torch.cuda.max_memory_allocated(device)

    def memory_reserved(self, device=None) -> int:
        return torch.cuda.memory_reserved(device)

    def max_memory_reserved(self, device=None) -> int:
        return torch.cuda.max_memory_reserved(device)

    def reset_peak_memory_stats(self, device=None) -> None:
        torch.cuda.reset_peak_memory_stats(device)

    def mem_get_info(self, device=None):
        return torch.cuda.mem_get_info(device)

    def get_device_capability(self, device=None):
        return torch.cuda.get_device_capability(device)

    def set_per_process_memory_fraction(self, fraction: float, device=None) -> None:
        torch.cuda.set_per_process_memory_fraction(fraction, device)

    def Stream(self, *a, **k):
        return torch.cuda.Stream(*a, **k)

    def Event(self, *a, **k):
        return torch.cuda.Event(*a, **k)

    def current_stream(self, device=None):
        return torch.cuda.current_stream(device)

    def stream(self, stream_):
        return torch.cuda.stream(stream_)


class CpuAccelerator(BaseAccelerator):
    name = "cpu"
    communication_backend = "gloo"

    def get_current_device(self) -> torch.device:
        return torch.device("cpu")

    def device_count(self) -> int:
        return 1


_ACCELERATOR: Optional[BaseAccelerator] = None
_MAPPING = {"cuda": CudaAccelerator, "cpu": CpuAccelerator}


def set_accelerator(name: str) -> None:
    global _ACCELERATOR
    if name not in _MAPPING:
        raise ValueError(f"accelerator {name!r} unsupported; choose from {list(_MAPPING)}")
    _ACCELERATOR = _MAPPING[name]()


def auto_set_accelerator() -> None:
    set_accelerator("cuda" if torch.cuda.is_available() else "cpu")


def get_accelerator() -> BaseAccelerator:
    if _ACCELERATOR is None:
        auto_set_accelerator()
    return _ACCELERATOR  # type: ignore[return-value]
