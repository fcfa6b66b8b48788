"""Python face of the multi-tensor optimizer kernels (kernel/csrc/multi_tensor_optim.cu).

A `TensorTable` is a cached device-resident descriptor of a list of (param, grad, exp_avg, exp_avg_sq, lp_copy)
tuples; one kernel launch then covers the whole list.  Parity: reference `multi_tensor_applier` +
`fused_optim.multi_tensor_{adam,sgd,lamb,l2norm,scale}` (`colossalai/utils/multi_tensor_apply`, N3-N7).
"""
from __future__ import annotations

import ctypes
from typing import List, Optional, Sequence, Tuple

import torch

from ..kernel import loader
from ._dtypes import code

_lib = None
_CHUNK = 2048 * 16
_COLS = 8


def _get_lib():
    global _lib, _CHUNK, _COLS
    if _lib is None:
        lib = loader.load("cb200_optim")
        lib.cb_opt_chunk_size.restype = ctypes.c_int
        lib.cb_opt_table_cols.restype = ctypes.c_int
        _CHUNK, _COLS = lib.cb_opt_chunk_size(), lib.cb_opt_table_cols()
        _lib = lib
    return _lib


class TensorTable:
    """Descriptor table for one group of tensors.  Slots: p (required), g, m, v, lp (optional)."""

    def __init__(self, p: Sequence[torch.Tensor], g: Optional[Sequence[torch.Tensor]] = None,
                 m: Optional[Sequence[torch.Tensor]] = None, v: Optional[Sequence[torch.Tensor]] = None,
                 lp: Optional[Sequence[Optional[torch.Tensor]]] = None, keepalive: bool = False) -> None:
        _get_lib()
        n = len(p)
        rows = []
        chunk = 0
        for i in range(n):
            pi = p[i]
            assert pi.is_contiguous(), "multi-tensor ops need contiguous tensors"
            gi = g[i] if g is not None else None
            mi = m[i] if m is not None else None
            vi = v[i] if v is not None else None
            li = lp[i] if lp is not None else None
            for t in (gi, mi, vi, li):
                assert t is None or (t.is_contiguous() and t.numel() == pi.numel())
            dt = code(pi.dtype) | ((code(gi.dtype) if gi is not None else 0) << 8) | \
                ((code(li.dtype) if li is not None else 0) << 16)
            rows.append([pi.data_ptr(), gi.data_ptr() if gi is not None else 0,
                         mi.data_ptr() if mi is not None else 0, vi.data_ptr() if vi is not None else 0,
                         li.data_ptr() if li is not None else 0, pi.numel(), dt, chunk])
            chunk += (pi.numel() + _CHUNK - 1) // _CHUNK
        self.num_tensors = n
        self.total_chunks = chunk
        self.device = p[0].device if n else torch.device("cuda")
        self.table = torch.tensor(rows, dtype=torch.int64).to(self.device) if n else None
        self._partial = None
        # NOTE: the table stores raw pointers.  Callers own the tensors' lifetime (kernels are stream-ordered, so a
        # tensor may be released right after the launch).  `keepalive=True` pins the persistent slots (p, m, v, lp)
        # for cached tables.  The grad slot is never pinned: gradients are usually new tensors every step, and
        # pinning them would keep each step's gradients resident and push the next ones to new addresses, so the
        # cache key (which includes the grad pointers) would never hit.  A key hit means the live gradients sit at
        # exactly the pointers stored in the table.
        self._keepalive = (list(p), m, v, lp) if keepalive else None

    @staticmethod
    def key_of(*lists) -> tuple:
        return tuple((t.data_ptr() if t is not None else 0) for lst in lists if lst is not None for t in lst)

    def partial(self) -> torch.Tensor:
        if self._partial is None:
            self._partial = torch.empty(max(self.total_chunks, 1), dtype=torch.float32, device=self.device)
        return self._partial


def adam(tbl: TensorTable, lr: float, beta1: float, beta2: float, eps: float, weight_decay: float, step: int,
         adamw: bool = True, bias_correction: bool = True, inv_scale: float = 1.0,
         noop_flag: Optional[torch.Tensor] = None, inv_scale_dev: Optional[torch.Tensor] = None) -> None:
    if tbl.num_tensors == 0:
        return
    lib = _get_lib()
    bc1 = 1.0 - beta1 ** step if bias_correction else 1.0
    bc2 = 1.0 - beta2 ** step if bias_correction else 1.0
    f = ctypes.c_float
    loader.check(lib.cb_multi_tensor_adam(loader.ptr(tbl.table), tbl.num_tensors, ctypes.c_int64(tbl.total_chunks),
                                          f(lr), f(beta1), f(beta2), f(eps), f(weight_decay), f(bc1), f(bc2),
                                          f(inv_scale), int(adamw), loader.ptr(noop_flag), loader.ptr(inv_scale_dev),
                                          loader.stream_ptr()), "multi_tensor_adam")
    loader.launch_counter.add("multi_tensor_adam")


def sgd(tbl: TensorTable, lr: float, momentum: float, dampening: float, weight_decay: float, nesterov: bool,
        first_run: bool, wd_after_momentum: bool = False, inv_scale: float = 1.0,
        noop_flag: Optional[torch.Tensor] = None) -> None:
    if tbl.num_tensors == 0:
        return
    lib = _get_lib()
    f = ctypes.c_float
    loader.check(lib.cb_multi_tensor_sgd(loader.ptr(tbl.table), tbl.num_tensors, ctypes.c_int64(tbl.total_chunks),
                                         f(lr), f(momentum), f(dampening), f(weight_decay), f(inv_scale),
                                         int(nesterov), int(first_run), int(wd_after_momentum),
                                         loader.ptr(noop_flag), loader.stream_ptr()), "multi_tensor_sgd")
    loader.launch_counter.add("multi_tensor_sgd")


def norm_sq(tbl: TensorTable, which: str = "grad", per_tensor: bool = False, use_max: bool = False
            ) -> Tuple[torch.Tensor, Optional[torch.Tensor]]:
    """Returns (sum of squares [1] fp32 (or max-abs), per-tensor values or None).  No host sync."""
    lib = _get_lib()
    out = torch.zeros(1, dtype=torch.float32, device=tbl.device)
    pt = torch.zeros(tbl.num_tensors, dtype=torch.float32, device=tbl.device) if per_tensor else None
    if tbl.num_tensors == 0:
        return out, pt
    w = {"param": 0, "grad": 1, "m": 2}[which]
    loader.check(lib.cb_multi_tensor_norm(loader.ptr(tbl.table), tbl.num_tensors, ctypes.c_int64(tbl.total_chunks),
                                          w, int(use_max), loader.ptr(tbl.partial()), loader.ptr(out), loader.ptr(pt),
                                          loader.stream_ptr()), "multi_tensor_norm")
    loader.launch_counter.add("multi_tensor_norm", 2)
    return out, pt


def scale(tbl: TensorTable, factor: float, flag: Optional[torch.Tensor] = None) -> None:
    """grad-slot[i] = param-slot[i] * factor; flag (int32[1]) set on inf/nan."""
    if tbl.num_tensors == 0:
        return
    lib = _get_lib()
    loader.check(lib.cb_multi_tensor_scale(loader.ptr(tbl.table), tbl.num_tensors, ctypes.c_int64(tbl.total_chunks),
                                           ctypes.c_float(factor), loader.ptr(flag), loader.stream_ptr()),
                 "multi_tensor_scale")
    loader.launch_counter.add("multi_tensor_scale")


def lamb(tbl: TensorTable, lr: float, beta1: float, beta2: float, eps: float, weight_decay: float, step: int,
         adamw: bool = True, bias_correction: bool = True, grad_averaging: bool = True, inv_scale: float = 1.0,
         noop_flag: Optional[torch.Tensor] = None, trust_ratio: bool = True) -> None:
    """Two-stage LAMB.  Stage 1 writes the update u into the grad slot, rounded to the grad dtype; stage 2 steps
    p -= lr * ratio * u with ratio = ||p|| / ||u|| per tensor (1 if either norm is 0).  `trust_ratio=False` skips
    both norm launches and steps with ratio 1 (the reference does so unless `use_nvlamb` or weight_decay != 0)."""
    if tbl.num_tensors == 0:
        return
    lib = _get_lib()
    f = ctypes.c_float
    bc1 = 1.0 - beta1 ** step if bias_correction else 1.0
    bc2 = 1.0 - beta2 ** step if bias_correction else 1.0
    beta3 = 1.0 - beta1 if grad_averaging else 1.0
    p_norms = u_norms = None
    if trust_ratio:
        _, p_norms = norm_sq(tbl, "param", per_tensor=True)
    loader.check(lib.cb_multi_tensor_lamb_stage1(loader.ptr(tbl.table), tbl.num_tensors,
                                                 ctypes.c_int64(tbl.total_chunks), f(beta1), f(beta2), f(beta3),
                                                 f(eps), f(weight_decay), f(bc1), f(bc2), f(inv_scale), int(adamw),
                                                 loader.ptr(noop_flag), loader.stream_ptr()), "lamb_stage1")
    if trust_ratio:
        _, u_norms = norm_sq(tbl, "grad", per_tensor=True)
    loader.check(lib.cb_multi_tensor_lamb_stage2(loader.ptr(tbl.table), tbl.num_tensors,
                                                 ctypes.c_int64(tbl.total_chunks), f(lr), loader.ptr(p_norms),
                                                 loader.ptr(u_norms), loader.ptr(noop_flag), loader.stream_ptr()),
                 "lamb_stage2")
    loader.launch_counter.add("multi_tensor_lamb", 2)
