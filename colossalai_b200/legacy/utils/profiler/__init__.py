"""Legacy profilers.  Parity: reference `colossalai/legacy/utils/profiler/{profiler.py:1-200 (ProfilerContext wrapper
over torch.profiler), legacy/comm_profiler.py:56-300, legacy/pcie_profiler.py:1-150, legacy/mem_profiler.py}`."""
from __future__ import annotations

from pathlib import Path
from typing import Dict, List, Optional

import torch

from ....utils.profiler import CommProfiler

__all__ = ["ProfilerContext", "CommProfiler", "PcieProfiler", "MemProfiler", "BaseProfiler"]


class BaseProfiler:
    def __init__(self, profiler_name: str, priority: int = 0) -> None:
        self.name, self.priority = profiler_name, priority

    def enable(self) -> None: ...
    def disable(self) -> None: ...
    def to_tensorboard(self, writer) -> None: ...
    def to_file(self, filename: Path) -> None:
        Path(filename).write_text(self.result_str())

    def show(self) -> None:
        print(self.result_str())

    def result_str(self, sep: str = "\n") -> str:
        return ""


class PcieProfiler(BaseProfiler):
    """Host<->device copy profiler: records every `Memcpy HtoD / DtoH` of a `torch.profiler` trace with bytes, time
    and achieved bandwidth (the PCIe link the offload paths ride on)."""

    def __init__(self, dtype: str = "fp32", depth: int = 1) -> None:
        super().__init__("Pcie", 10)
        self.depth = depth
        self.data_size = {"fp16": 2, "bf16": 2, "fp32": 4}.get(dtype, 4)
        self.h2d_count = self.d2h_count = 0
        self.h2d_time = self.d2h_time = 0.0
        self.events: List[Dict] = []
        self._prof: Optional[torch.profiler.profile] = None

    def enable(self) -> None:
        acts = [torch.profiler.ProfilerActivity.CPU]
        if torch.cuda.is_available():
            acts.append(torch.profiler.ProfilerActivity.CUDA)
        self._prof = torch.profiler.profile(activities=acts, record_shapes=True)
        self._prof.__enter__()

    def disable(self) -> None:
        if self._prof is None:
            return
        self._prof.__exit__(None, None, None)
        for ev in self._prof.events():
            name = ev.name
            if "Memcpy HtoD" in name or "Memcpy DtoH" in name:
                t = getattr(ev, "device_time_total", 0.0) or getattr(ev, "cuda_time_total", 0.0)
                rec = {"name": name, "time_us": float(t)}
                self.events.append(rec)
                if "HtoD" in name:
                    self.h2d_count += 1
                    self.h2d_time += float(t)
                else:
                    self.d2h_count += 1
                    self.d2h_time += float(t)
        self._prof = None

    def result_str(self, sep: str = "\n") -> str:
        return sep.join([
            "Pcie profiling result:",
            f"time of data transmission (CPU -> GPU): {self.h2d_time / 1e6:.6f} s",
            f"number of transmission (CPU -> GPU): {self.h2d_count}",
            f"time of data transmission (GPU -> CPU): {self.d2h_time / 1e6:.6f} s",
            f"number of transmission (GPU -> CPU): {self.d2h_count}"])


class MemProfiler(BaseProfiler):
    """Samples allocated / reserved device memory at `step()` boundaries."""

    def __init__(self, log_dir: Optional[str] = None) -> None:
        super().__init__("Mem", 0)
        self.samples: List[Dict[str, float]] = []
        self.log_dir = log_dir
        self._on = False

    def enable(self) -> None:
        self._on = True
        if torch.cuda.is_available():
            torch.cuda.reset_peak_memory_stats()

    def disable(self) -> None:
        self._on = False

    def step(self, tag: str = "") -> None:
        if not self._on:
            return
        if torch.cuda.is_available():
            self.samples.append({"tag": tag, "allocated": float(torch.cuda.memory_allocated()),
                                 "peak": float(torch.cuda.max_memory_allocated()),
                                 "reserved": float(torch.cuda.memory_reserved())})
        else:
            self.samples.append({"tag": tag, "allocated": 0.0, "peak": 0.0, "reserved": 0.0})

    def result_str(self, sep: str = "\n") -> str:
        return sep.join(f"{s['tag']}: allocated {s['allocated'] / 2**20:.1f} MB peak {s['peak'] / 2**20:.1f} MB"
                        for s in self.samples)


class ProfilerContext:
    """`with ProfilerContext([CommProfiler(), PcieProfiler()]) as prof: ...; prof.show()`."""

    def __init__(self, profilers: Optional[List[BaseProfiler]] = None, enable: bool = True) -> None:
        self.enable = enable
        self.profilers = sorted(profilers or [], key=lambda p: getattr(p, "priority", 0))

    def __enter__(self):
        if self.enable:
            for p in self.profilers:
                p.enable()
        return self

    def __exit__(self, *exc):
        if self.enable:
            for p in reversed(self.profilers):
                p.disable()
        return False

    def to_file(self, log_dir) -> None:
        Path(log_dir).mkdir(parents=True, exist_ok=True)
        for p in self.profilers:
            if hasattr(p, "result_str"):
                (Path(log_dir) / f"{getattr(p, 'name', type(p).__name__).lower()}.log").write_text(p.result_str())

    def show(self) -> None:
        for p in self.profilers:
            if hasattr(p, "show"):
                p.show()
