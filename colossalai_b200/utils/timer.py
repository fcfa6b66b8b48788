"""Device-synchronising timers.  Parity: reference `colossalai/utils/timer.py:9,91`.  `CudaEventTimer` is the
Addition: device-side timing with CUDA events (what every reported number must use)."""
from __future__ import annotations

import time
from typing import Dict, List, Optional

import torch


def _sync() -> None:
    if torch.cuda.is_available():
        torch.cuda.synchronize()


class Timer:
    def __init__(self) -> None:
        self._started = False
        self._start_time = 0.0
        self._elapsed = 0.0
        self._history: List[float] = []

    @property
    def has_history(self) -> bool:
        return len(self._history) != 0

    @property
    def current_time(self) -> float:
        _sync()
        return time.time()

    def start(self) -> None:
        self._elapsed = 0.0
        self._start_time = self.current_time
        self._started = True

    def lap(self) -> float:
        return self.current_time - self._start_time

    def stop(self, keep_in_history: bool = False) -> float:
        end = self.current_time
        if self._started:
            self._elapsed = end - self._start_time
        else:
            raise RuntimeError("Timer.stop() called before start()")
        if keep_in_history:
            self._history.append(self._elapsed)
        self._started = False
        return self._elapsed

    def get_history_mean(self) -> float:
        return sum(self._history) / len(self._history)

    def get_history_sum(self) -> float:
        return sum(self._history)

    def get_elapsed_time(self) -> float:
        assert not self._started, "timer still running"
        return self._elapsed

    def reset(self) -> None:
        self._history.clear()
        self._started = False
        self._elapsed = 0.0


class MultiTimer:
    def __init__(self, on: bool = True) -> None:
        self._on = on
        self._timers: Dict[str, Timer] = {}

    def start(self, name: str) -> None:
        if self._on:
            self._timers.setdefault(name, Timer()).start()

    def stop(self, name: str, keep_in_history: bool) -> None:
        if self._on:
            self._timers[name].stop(keep_in_history)

    def get_timer(self, name: str) -> Timer:
        return self._timers[name]

    def reset(self, name: Optional[str] = None) -> None:
        if self._on:
            if name is not None:
                self._timers[name].reset()
            else:
                for t in self._timers.values():
                    t.reset()

    def is_on(self) -> bool:
        return self._on

    def set_status(self, mode: bool) -> None:
        self._on = mode

    def __iter__(self):
        return iter(self._timers.items())


class CudaEventTimer:
    """Device-timed regions on the current stream.  `with t.region("fwd"): ...`; `t.summary()` -> ms."""

    def __init__(self) -> None:
        self._pairs: Dict[str, List] = {}

    class _Region:
        def __init__(self, owner: "CudaEventTimer", name: str):
            self.owner, self.name = owner, name

        def __enter__(self):
            self.s = torch.cuda.Event(enable_timing=True)
            self.e = torch.cuda.Event(enable_timing=True)
            self.s.record()
            return self

        def __exit__(self, *exc):
            self.e.record()
            self.owner._pairs.setdefault(self.name, []).append((self.s, self.e))

    def region(self, name: str) -> "CudaEventTimer._Region":
        return CudaEventTimer._Region(self, name)

    def summary(self) -> Dict[str, float]:
        torch.cuda.synchronize()
        return {k: sum(s.elapsed_time(e) for s, e in v) for k, v in self._pairs.items()}

    def reset(self) -> None:
        self._pairs.clear()
