"""Fused compute+collective backend ("fused" comm backend) over NVLink peer memory.

Python side of `kernel/csrc/fused_comm_gemm.cu`: symmetric-memory workspaces (allocation + rendezvous through
`torch.distributed._symmetric_memory`, i.e. cuMem handles exchanged over the bootstrap process group, peer mappings and
the NVLS multicast mapping), epoch bookkeeping for the flag protocol, and the three entry points used by the TP/SP
linear layers:

    all_gather_gemm(x_local, w, group)        ->  (gather(x) @ w^T  or  gather(x) @ w,  gathered x)
    gemm_reduce_scatter(a, w, group)          ->  reduce_scatter_rows(a @ w^T  or  a @ w)
    all_gather(x_local, group)                ->  gathered rows (P2P pull kernel)

SURVEY §5.8 items 2-4.  Every function falls back to the NCCL composition when a shape does not meet the kernel's
alignment rules, so callers never need to special-case.
"""
from __future__ import annotations

import ctypes
import os
from typing import Dict, List, Optional, Tuple

import torch
import torch.distributed as dist
from torch.distributed import ProcessGroup

from ..kernel import loader
from ..ops import matmul_nn
from ..ops._dtypes import code
from . import comm

__all__ = ["available", "build_available", "all_gather_gemm", "gemm_reduce_scatter", "gemm_all_reduce", "all_gather",
           "reduce_scatter", "ulysses_all_to_all",
           "FusedWorkspace", "stats"]

_lib = None
_workspaces: Dict[tuple, "FusedWorkspace"] = {}
_disabled = os.environ.get("CB200_DISABLE_FUSED_COMM", "0") == "1"
stats = {"ag_gemm": 0, "gemm_rs": 0, "all_gather": 0, "fallback": 0}


def _get_lib():
    global _lib
    if _lib is None:
        lib = loader.load("cb200_comm")
        lib.cb_fused_flag_words.restype = ctypes.c_int
        _lib = lib
    return _lib


def build_available() -> bool:
    if _disabled or not torch.cuda.is_available():
        return False
    try:
        _get_lib()
        import importlib

        importlib.import_module("torch.distributed._symmetric_memory")

        return True
    except Exception:
        return False


def available(group: Optional[ProcessGroup]) -> bool:
    if not build_available() or not dist.is_initialized():
        return False
    ws = comm.group_size(group)
    if ws < 2 or ws > 16:
        return False
    try:
        return workspace(group) is not None
    except Exception as e:  # pragma: no cover - depends on the box
        from ..logging import get_dist_logger

        get_dist_logger().warning(f"fused comm backend unavailable ({e}); using NCCL", ranks=[0])
        _workspaces[comm.group_key(group)] = None  # type: ignore[assignment]
        return False


class _SymmBuffer:
    """A symmetric allocation: local tensor + every peer's mapping of its copy (+ multicast mapping)."""

    def __init__(self, nbytes: int, group: ProcessGroup, zero: bool = False) -> None:
        import torch.distributed._symmetric_memory as symm_mem

        self.nbytes = nbytes
        dev = torch.device("cuda", torch.cuda.current_device())
        self.tensor = symm_mem.empty(nbytes, dtype=torch.uint8, device=dev)
        if zero:
            self.tensor.zero_()
        elif os.environ.get("CB200_POISON_SYMM", "0") == "1":
            # debug: data buffers start as 0xFF (bf16 NaN) so a read-before-write in a flag protocol shows up as NaNs
            self.tensor.fill_(0xFF)
        self.handle = symm_mem.rendezvous(self.tensor, group)
        self.peer_ptrs: List[int] = [int(p) for p in self.handle.buffer_ptrs]
        mc = 0
        try:
            if self.handle.has_multicast_support:
                mc = int(self.handle.multicast_ptr)
        except Exception:
            mc = 0
        self.mc_ptr = mc
        self.last_epoch = 0

    def ptr_array(self, world: int):
        return (ctypes.c_void_p * world)(*self.peer_ptrs[:world])


class FusedWorkspace:
    """Per-process-group state of the fused backend."""

    def __init__(self, group: Optional[ProcessGroup]) -> None:
        self.group = group if group is not None else dist.group.WORLD
        self.world = comm.group_size(group)
        self.rank = comm.group_rank(group)
        lib = _get_lib()
        self.flags = _SymmBuffer(4 * lib.cb_fused_flag_words(), self.group, zero=True)
        torch.cuda.synchronize()
        dist.barrier(group=self.group)      # flag pages are zero everywhere before first use
        self.epoch = 0
        self._in: Dict[int, List[_SymmBuffer]] = {}
        self._part: Dict[int, List[_SymmBuffer]] = {}
        self._toggle: Dict[Tuple[str, int], int] = {}
        self._counters: Dict[int, torch.Tensor] = {}
        dev = torch.device("cuda", torch.cuda.current_device())
        self.chunk_counter = torch.zeros(64, dtype=torch.int32, device=dev)

    def next_epoch(self) -> int:
        self.epoch += 1
        return self.epoch

    def _pool(self, pools: Dict[int, List[_SymmBuffer]], kind: str, nbytes: int) -> _SymmBuffer:
        size = 1 << max(20, (nbytes - 1).bit_length())        # power-of-two size classes, >= 1 MiB
        if size not in pools:
            pools[size] = [_SymmBuffer(size, self.group), _SymmBuffer(size, self.group)]
        t = self._toggle.get((kind, size), 0)
        self._toggle[(kind, size)] = t ^ 1
        buf = pools[size][t]
        if buf.last_epoch:
            # buffer reuse guard: every peer must have finished reading what we published at `last_epoch`
            lib = _get_lib()
            loader.check(lib.cb_wait_pull_done(ctypes.c_void_p(self.flags.peer_ptrs[self.rank]), self.world,
                                               ctypes.c_uint32(buf.last_epoch), loader.stream_ptr()), "wait_pull_done")
        return buf

    def in_buffer(self, nbytes: int) -> _SymmBuffer:
        return self._pool(self._in, "in", nbytes)

    def part_buffer(self, nbytes: int) -> _SymmBuffer:
        return self._pool(self._part, "part", nbytes)

    def counters(self, n_blocks: int) -> Tuple[torch.Tensor, torch.Tensor]:
        """(ready flags, block counters): uint32[n_blocks] each, zero-initialised once (epochs make them reusable)."""
        key = 1 << max(6, (n_blocks - 1).bit_length())
        if key not in self._counters:
            dev = torch.device("cuda", torch.cuda.current_device())
            self._counters[key] = torch.zeros(2, key, dtype=torch.int32, device=dev)
        c = self._counters[key]
        return c[0], c[1]


def workspace(group: Optional[ProcessGroup]) -> Optional[FusedWorkspace]:
    key = comm.group_key(group)
    if key not in _workspaces:
        _workspaces[key] = FusedWorkspace(group)
    return _workspaces[key]


def _aligned(T: int, world: int, *dims: int) -> bool:
    return T % (world * 128) == 0 and all(d % 8 == 0 for d in dims)


def _ok_dtype(*ts: torch.Tensor) -> bool:
    return all(t.dtype in (torch.bfloat16, torch.float16) and t.dtype == ts[0].dtype for t in ts)


# ------------------------------------------------------------------------------------------------ all-gather
def all_gather(x_local: torch.Tensor, group: Optional[ProcessGroup]) -> torch.Tensor:
    """Gather rows of every rank's [t, K] tensor -> [t * world, K] by pulling over NVLink."""
    ws = workspace(group)
    t, K = x_local.shape
    if ws is None or not _ok_dtype(x_local) or K % 8 != 0:
        stats["fallback"] += 1
        return comm.all_gather(x_local, 0, group)
    lib = _get_lib()
    nbytes = x_local.numel() * x_local.element_size()
    buf = ws.in_buffer(nbytes)
    buf.tensor[:nbytes].view(x_local.dtype).view(t, K).copy_(x_local)
    epoch = ws.next_epoch()
    out = torch.empty(t * ws.world, K, dtype=x_local.dtype, device=x_local.device)
    n_ctas = 2 * torch.cuda.get_device_properties(x_local.device).multi_processor_count
    loader.check(lib.cb_all_gather_pull(buf.ptr_array(ws.world), ws.flags.ptr_array(ws.world), loader.ptr(out), t, K,
                                        ws.rank, ws.world, ctypes.c_uint32(epoch), n_ctas, loader.stream_ptr()),
                 "all_gather_pull")
    buf.last_epoch = epoch
    loader.launch_counter.add("fused_all_gather")
    stats["all_gather"] += 1
    return out


def reduce_scatter(x: torch.Tensor, group: Optional[ProcessGroup]) -> torch.Tensor:
    """Sum `x` ([world * t, ...], bf16 or fp32) over the group and return this rank's chunk [t, ...]: every rank
    publishes its tensor in symmetric memory and reduces its own chunk straight out of the NVSwitch."""
    ws = workspace(group)
    world = comm.group_size(group)
    nbytes = x.numel() * x.element_size()
    if (ws is None or x.dtype not in (torch.bfloat16, torch.float32) or x.shape[0] % world != 0
            or (nbytes // world) % 16 != 0 or not x.is_cuda):
        stats["fallback"] += 1
        return comm.reduce_scatter(x.contiguous(), 0, group)
    part = ws.part_buffer(nbytes)
    part.tensor[:nbytes].view(x.dtype).view(x.shape).copy_(x)
    epoch = ws.next_epoch()
    out = torch.empty((x.shape[0] // world,) + tuple(x.shape[1:]), dtype=x.dtype, device=x.device)
    use_mc = part.mc_ptr and os.environ.get("CB200_NO_MULTIMEM", "0") != "1"
    n_ctas = 2 * torch.cuda.get_device_properties(x.device).multi_processor_count
    loader.check(_get_lib().cb_reduce_scatter(part.ptr_array(world), ctypes.c_void_p(part.mc_ptr if use_mc else 0),
                                              ws.flags.ptr_array(world), loader.ptr(out),
                                              ctypes.c_int64(nbytes // world), 0 if x.dtype == torch.bfloat16 else 1,
                                              ws.rank, world, ctypes.c_uint32(epoch), n_ctas, loader.stream_ptr()),
                 "reduce_scatter")
    part.last_epoch = epoch
    loader.launch_counter.add("fused_reduce_scatter")
    stats["reduce_scatter"] = stats.get("reduce_scatter", 0) + 1
    return out


# ------------------------------------------------------------------------------------------------ AG + GEMM
def all_gather_gemm(x_local: torch.Tensor, w: torch.Tensor, group: Optional[ProcessGroup], transpose_b: bool = True,
                    block_n: int = 0) -> Tuple[torch.Tensor, torch.Tensor]:
    """y = gather_rows(x_local) @ (w^T if transpose_b else w).  Returns (y, gathered x)."""
    ws = workspace(group)
    t, K = x_local.shape
    N = w.shape[0] if transpose_b else w.shape[1]
    kdim_ok = (w.shape[1] == K) if transpose_b else (w.shape[0] == K)
    assert kdim_ok, f"all_gather_gemm: inner dims mismatch {tuple(x_local.shape)} x {tuple(w.shape)}"
    world = comm.group_size(group)
    T = t * world
    if (ws is None or not _ok_dtype(x_local, w) or not _aligned(T, world, K, N) or not w.is_contiguous()
            or w.data_ptr() % 16 != 0):
        stats["fallback"] += 1
        xf = comm.all_gather(x_local.contiguous(), 0, group)
        return (torch.nn.functional.linear(xf, w) if transpose_b else matmul_nn(xf, w)), xf
    lib = _get_lib()
    nbytes = x_local.numel() * x_local.element_size()
    buf = ws.in_buffer(nbytes)
    buf.tensor[:nbytes].view(x_local.dtype).view(t, K).copy_(x_local)
    epoch = ws.next_epoch()
    gathered = torch.empty(T, K, dtype=x_local.dtype, device=x_local.device)
    y = torch.empty(T, N, dtype=x_local.dtype, device=x_local.device)
    ready, blk_cnt = ws.counters(T // 128)
    loader.check(lib.cb_ag_gemm(buf.ptr_array(world), ws.flags.ptr_array(world), loader.ptr(gathered),
                                loader.ptr(ready), loader.ptr(blk_cnt), loader.ptr(w), loader.ptr(y), T, N, K,
                                w.stride(0), y.stride(0), 0 if transpose_b else 1, code(x_local.dtype), ws.rank, world,
                                ctypes.c_uint32(epoch), 0, block_n, loader.stream_ptr()), "ag_gemm")
    buf.last_epoch = epoch
    loader.launch_counter.add("fused_ag_gemm")
    stats["ag_gemm"] += 1
    return y, gathered


# ------------------------------------------------------------------------------------------------ GEMM + RS
_rs_choice: Dict[Tuple, str] = {}            # autotuned variant per (world, T, N, K, layout, dtype)
rs_tuning_log: List[dict] = []               # what the autotuner measured (bench.py / profiles print it)


def _rs_fusable(ws, a, w, T, K, N, world) -> bool:
    return (ws is not None and _ok_dtype(a, w) and _aligned(T, world, K, N) and w.is_contiguous()
            and a.is_contiguous() and a.data_ptr() % 16 == 0 and w.data_ptr() % 16 == 0)


def _gemm_rs_lib(a, w, group, transpose_b):
    full = torch.nn.functional.linear(a, w) if transpose_b else matmul_nn(a, w)
    return comm.reduce_scatter(full, 0, group)


def _gemm_rs_launch(ws, a, w, transpose_b, block_n):
    lib = _get_lib()
    T, K = a.shape
    N = w.shape[0] if transpose_b else w.shape[1]
    world = ws.world
    part = ws.part_buffer(T * N * a.element_size())
    epoch = ws.next_epoch()
    out = torch.empty(T // world, N, dtype=a.dtype, device=a.device)
    mc = ctypes.c_void_p(part.mc_ptr) if (part.mc_ptr and a.dtype == torch.bfloat16
                                          and os.environ.get("CB200_NO_MULTIMEM", "0") != "1") else ctypes.c_void_p(0)
    loader.check(lib.cb_gemm_rs(loader.ptr(a), loader.ptr(w), ctypes.c_void_p(part.peer_ptrs[ws.rank]),
                                part.ptr_array(world), mc, ws.flags.ptr_array(world), loader.ptr(ws.chunk_counter),
                                loader.ptr(out), T, N, K, a.stride(0),
                                w.stride(0), N, 0,
                                0 if transpose_b else 1, code(a.dtype), ws.rank, world, ctypes.c_uint32(epoch), block_n,
                                loader.stream_ptr()), "gemm_rs")
    part.last_epoch = epoch
    return out


def _time_rs(fn, group, iters: int = 3) -> float:
    """Device time of `fn` (ms per call), max over the ranks of `group`; every rank calls this in lock-step."""
    fn()
    torch.cuda.synchronize()
    dist.barrier(group=group)
    s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    s.record()
    for _ in range(iters):
        fn()
    e.record()
    torch.cuda.synchronize()
    t = torch.tensor([s.elapsed_time(e) / iters], device="cuda")
    dist.all_reduce(t, op=dist.ReduceOp.MAX, group=group)
    return float(t.item())


def rs_variant(a: torch.Tensor, w: torch.Tensor, group: Optional[ProcessGroup], transpose_b: bool = True) -> str:
    """Which implementation `gemm_reduce_scatter` uses for this shape: 'fused' (one kernel: the wgmma GEMM writes
    partial tiles to symmetric memory, then every rank reduces its own chunk - in the switch with `multimem.ld_reduce`
    when a multicast mapping exists, else with P2P loads - once all peers have finished that chunk; the reduction
    does not overlap the GEMM), or 'lib' (cuBLAS/own GEMM followed by the NCCL reduce-scatter).  Chosen ONCE per shape by measuring all candidates on the
    live tensors (device-timed, max over ranks, identical decision on every rank); `CB200_FUSED_RS` forces one."""
    ws = workspace(group)
    T, K = a.shape
    N = w.shape[0] if transpose_b else w.shape[1]
    world = comm.group_size(group)
    if not _rs_fusable(ws, a, w, T, K, N, world):
        return "lib"
    forced = os.environ.get("CB200_FUSED_RS", "auto")
    if forced in ("fused", "lib"):
        return forced
    key = (world, T, N, K, transpose_b, a.dtype)
    got = _rs_choice.get(key)
    if got is not None:
        return got
    cands = ["fused", "lib"]
    times = {}
    for c in cands:
        if c == "lib":
            times[c] = _time_rs(lambda: _gemm_rs_lib(a, w, group, transpose_b), ws.group)
        else:
            times[c] = _time_rs(lambda: _gemm_rs_launch(ws, a, w, transpose_b, 0), ws.group)
    # prefer our own kernels on a tie (2 %): the library path is the fallback, not the product
    best = min(cands, key=lambda c: times[c] * (1.02 if c == "lib" else 1.0))
    _rs_choice[key] = best
    rs_tuning_log.append({"world": world, "T": T, "N": N, "K": K, "transpose_b": transpose_b, "ms": times,
                          "choice": best})
    return best


def gemm_reduce_scatter(a: torch.Tensor, w: torch.Tensor, group: Optional[ProcessGroup], transpose_b: bool = True,
                        block_n: int = 0, variant: str = "auto") -> torch.Tensor:
    """out[T/world, N] = reduce_scatter_rows(a @ (w^T if transpose_b else w)).

    variant: 'auto' = the autotuned choice of `rs_variant`; 'fused' forces the fused kernel; 'lib' = GEMM + NCCL
    reduce-scatter."""
    if variant not in ("auto", "fused", "lib"):
        raise ValueError(f"unknown GEMM->reduce-scatter variant {variant!r} (auto / fused / lib)")
    ws = workspace(group)
    T, K = a.shape
    N = w.shape[0] if transpose_b else w.shape[1]
    world = comm.group_size(group)
    if not _rs_fusable(ws, a, w, T, K, N, world):
        stats["fallback"] += 1
        return _gemm_rs_lib(a, w, group, transpose_b)
    if variant == "auto" and block_n == 0:
        variant = rs_variant(a, w, group, transpose_b)
    elif variant == "auto":
        variant = "fused"
    if variant == "lib":
        stats["rs_lib"] = stats.get("rs_lib", 0) + 1
        return _gemm_rs_lib(a, w, group, transpose_b)
    out = _gemm_rs_launch(ws, a, w, transpose_b, block_n)
    loader.launch_counter.add("fused_gemm_rs")
    stats["gemm_rs"] += 1
    stats["rs_" + variant] = stats.get("rs_" + variant, 0) + 1
    return out


# ------------------------------------------------------------------------------------------------ GEMM + AR
def gemm_all_reduce(a: torch.Tensor, w: torch.Tensor, group: Optional[ProcessGroup]) -> torch.Tensor:
    """all_reduce(a @ w^T) as the fused GEMM->reduce-scatter followed by the NVLink pull all-gather - the row-linear
    forward of tensor parallelism without sequence parallelism (reference: `F.linear` + `dist.all_reduce`,
    `layer/linear.py:586-587`)."""
    ws = workspace(group)
    world = comm.group_size(group)
    T, K = a.shape
    N = w.shape[0]
    if not _rs_fusable(ws, a, w, T, K, N, world):
        stats["fallback"] += 1
        y = torch.nn.functional.linear(a, w)
        comm.all_reduce(y, group)
        return y
    return all_gather(gemm_reduce_scatter(a, w, group, transpose_b=True), group)


# ------------------------------------------------------------------------------------------------ Ulysses all-to-all
def _ulysses_launch(x: torch.Tensor, group, mode: int, B: int, Sl: int, segs, out_cols: int) -> torch.Tensor:
    """One pull kernel for a sequence <-> head layout switch.  `segs`: [(in_base, out_base, ncols)] in elements."""
    ws = workspace(group)
    lib = _get_lib()
    world = ws.world
    nbytes = x.numel() * x.element_size()
    buf = ws.in_buffer(nbytes)
    buf.tensor[:nbytes].view(x.dtype).view(x.shape).copy_(x)
    epoch = ws.next_epoch()
    rows_out = B * Sl * world if mode == 0 else B * Sl
    out = torch.empty(rows_out, out_cols, dtype=x.dtype, device=x.device)
    n = len(segs)
    arr = lambda i: (ctypes.c_int * n)(*[int(sg[i]) for sg in segs])
    n_ctas = 2 * torch.cuda.get_device_properties(x.device).multi_processor_count
    loader.check(lib.cb_ulysses_a2a(buf.ptr_array(world), ws.flags.ptr_array(world), loader.ptr(out), mode, B, Sl, n,
                                    arr(0), arr(1), arr(2), x.shape[1], out_cols, x.element_size(), ws.rank, world,
                                    ctypes.c_uint32(epoch), n_ctas, loader.stream_ptr()), "ulysses_a2a")
    buf.last_epoch = epoch
    loader.launch_counter.add("fused_ulysses_a2a")
    stats["ulysses_a2a"] = stats.get("ulysses_a2a", 0) + 1
    return out


class _UlyssesA2A(torch.autograd.Function):
    """mode 0: [B*Sl, sum_s sp*w_s] -> [B*sp*Sl, sum_s w_s] (gather sequence, scatter the heads of every segment);
    mode 1: the inverse.  The backward of one mode is the other mode on the gradient."""

    @staticmethod
    def forward(ctx, x, group, mode, B, Sl, widths):
        world = comm.group_size(group)
        ctx.group, ctx.mode, ctx.B, ctx.Sl, ctx.widths = group, mode, B, Sl, widths
        return _UlyssesA2A._run(x.contiguous(), group, mode, B, Sl, widths, world)

    @staticmethod
    def _run(x, group, mode, B, Sl, widths, world):
        segs, full, local = [], 0, 0
        for w in widths:                      # w = columns of ONE rank's head slice of this segment
            segs.append((full, local, w) if mode == 0 else (local, full, w))
            full += w * world
            local += w
        return _ulysses_launch(x, group, mode, B, Sl, segs, local if mode == 0 else full)

    @staticmethod
    def backward(ctx, dy):
        world = comm.group_size(ctx.group)
        dx = _UlyssesA2A._run(dy.contiguous(), ctx.group, 1 - ctx.mode, ctx.B, ctx.Sl, ctx.widths, world)
        return dx, None, None, None, None, None


def ulysses_all_to_all(x: torch.Tensor, group: Optional[ProcessGroup], gather_sequence: bool, batch: int,
                       local_seqlen: int, widths) -> Optional[torch.Tensor]:
    """Fused Ulysses layout switch of a token-major 2-D tensor made of column segments (e.g. q | k | v).
    gather_sequence=True : x [B*Sl, sum(sp * w)] -> [B*sp*Sl, sum(w)]   (before attention: all tokens, my heads)
    gather_sequence=False: x [B*sp*Sl, sum(w)]   -> [B*Sl, sum(sp * w)] (after attention: my tokens, all heads)
    `widths`: per segment, the column count of one rank's head slice.  Returns None when the shape cannot take the
    kernel (caller falls back to the NCCL all_to_all)."""
    ws = workspace(group)
    per = 16 // x.element_size()
    if ws is None or x.dim() != 2 or not x.is_cuda or x.dtype not in (torch.bfloat16, torch.float16, torch.float32) \
            or any(w % per for w in widths) or len(widths) > 3:
        return None
    return _UlyssesA2A.apply(x, group, 0 if gather_sequence else 1, batch, local_seqlen, tuple(int(w) for w in widths))
