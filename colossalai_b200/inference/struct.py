"""Request / sequence bookkeeping.  Parity: reference `colossalai/inference/struct.py`."""
from __future__ import annotations

import enum
from dataclasses import dataclass, field
from typing import Any, List, Optional

__all__ = ["RequestStatus", "Sequence"]


class RequestStatus(enum.Enum):
    WAITING = enum.auto()
    RUNNING = enum.auto()
    ABORTED = enum.auto()
    OVERLENGTH = enum.auto()
    COMPLETED = enum.auto()
    LENGTH_CAPPED = enum.auto()
    RECYCLED = enum.auto()

    @staticmethod
    def is_finished(status: "RequestStatus") -> bool:
        return status in (RequestStatus.OVERLENGTH, RequestStatus.COMPLETED, RequestStatus.LENGTH_CAPPED)

    @staticmethod
    def is_running(status: "RequestStatus") -> bool:
        return status == RequestStatus.RUNNING

    @staticmethod
    def is_waiting(status: "RequestStatus") -> bool:
        return status == RequestStatus.WAITING


@dataclass
class Sequence:
    request_id: int
    prompt: str
    input_token_id: List[int]
    block_size: int
    sample_params: Any
    eos_token_id: int
    pad_token_id: int
    max_output_len: int = 256
    ignore_eos: bool = False
    output: str = None

    def __post_init__(self) -> None:
        self.output_token_id: List[int] = []
        self.status = RequestStatus.WAITING
        # prompt tokens whose K/V the cache holds while the prompt is prefilled: the prefix-cache hit at admission (a
        # whole number of blocks), advanced by each chunk under chunked prefill.  The prefill computes and writes only
        # the positions from here on
        self.num_cached_tokens = 0

    @property
    def sentence_len(self) -> int:
        return len(self.input_token_id) + len(self.output_token_id)

    @property
    def input_len(self) -> int:
        return len(self.input_token_id)

    @property
    def output_len(self) -> int:
        return len(self.output_token_id)

    def check_finish(self) -> bool:
        if RequestStatus.is_finished(self.status):
            return True
        if self.output_token_id:
            if (self.output_token_id[-1] == self.eos_token_id and not self.ignore_eos) \
                    or len(self.output_token_id) >= self.max_output_len:
                self.status = RequestStatus.COMPLETED
                return True
        return False

    def revoke_finished_status(self) -> None:
        if len(self.output_token_id) < self.max_output_len:
            self.status = RequestStatus.RUNNING

    def mark_running(self) -> None:
        assert self.status in (RequestStatus.WAITING, RequestStatus.RECYCLED)
        self.status = RequestStatus.RUNNING

    def mark_finished(self) -> None:
        self.status = RequestStatus.COMPLETED

    def mark_aborted(self) -> None:
        self.status = RequestStatus.ABORTED

    def recycle(self) -> None:
        assert not self.check_finish() and self.status != RequestStatus.ABORTED
        self.status = RequestStatus.RECYCLED
        self.num_cached_tokens = 0

    def __hash__(self) -> int:
        return hash(self.request_id)

    def __repr__(self) -> str:
        return (f"Sequence(request_id={self.request_id}, status={self.status.name}, in={self.input_len}, "
                f"out={self.output_len})")
