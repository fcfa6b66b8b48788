"""Node-list pipeline executor: zero-bubble V schedule (ZB-V) and, via a different node list, interleaved 1F1B.

Parity: reference `colossalai/pipeline/schedule/zero_bubble_pp.py:40-971` (`ZeroBubbleVPipeScheduler`: iterate a
precomputed list of `ScheduledNode{F,B,W,SEND_*,RECV_*}`; B computes dX only, W pops the `WeightGradStore`).
Communication design differs (NCCL-first): every adjacent stage pair gets TWO dedicated 2-rank process groups, one
per direction, so opposite-direction traffic never shares a NCCL stream (no send/recv cross dead-lock, no need to
coalesce ops); all sends are asynchronous; receives on a channel are posted in the SENDER's order (known from the global
schedule), a bounded number of messages ahead of their consumer.
"""
from __future__ import annotations

import pickle
from collections import defaultdict, deque
from typing import Any, Callable, Dict, Iterable, List, Optional, Tuple, Union

import torch
import torch.distributed as dist
from torch import Tensor
from torch.nn import Module, ModuleList
from torch.utils._pytree import tree_flatten, tree_map, tree_unflatten

from ...accelerator import get_accelerator
from ...interface import OptimizerWrapper
from ..p2p import P2PMetadata, create_send_metadata
from ..stage_manager import PipelineStageManager
from ..weight_grad_store import WeightGradStore
from ._utils import (default_criterion, detach, get_batch_size, get_micro_batch, merge_batch, model_forward,
                     retain_grad)
from .base import PipelineSchedule
from .v_schedule import PipelineGraph, ScheduledNode, _locate, _stage_of

__all__ = ["ZeroBubbleVPipeScheduler", "NodeListScheduler"]

_CHANNEL_CACHE: Dict[Tuple, Dict] = {}


class _Channels:
    """Directed 2-rank process groups between adjacent pipeline stages (including the wrap-around pair):
    `fwd[i]` carries stage i -> i+1 traffic, `bwd[i]` carries stage i+1 -> i traffic."""

    def __init__(self, sm: PipelineStageManager) -> None:
        pg_ranks = tuple(dist.get_process_group_ranks(sm.pp_group))
        if pg_ranks not in _CHANNEL_CACHE:
            # every rank of the WORLD must take part in every new_group call, in the same order
            world = dist.get_world_size()
            all_groups: List = [None] * world
            dist.all_gather_object(all_groups, pg_ranks)
            for ranks in sorted(set(tuple(g) for g in all_groups)):
                n = len(ranks)
                fwd, bwd = [], []
                for i in range(n):
                    pair = sorted({ranks[i], ranks[(i + 1) % n]})
                    fwd.append(dist.new_group(pair) if len(pair) == 2 else None)
                    bwd.append(dist.new_group(pair) if len(pair) == 2 else None)
                _CHANNEL_CACHE[ranks] = {"fwd": fwd, "bwd": bwd}
        self.ranks = pg_ranks
        self.n = len(pg_ranks)
        self.fwd = _CHANNEL_CACHE[pg_ranks]["fwd"]
        self.bwd = _CHANNEL_CACHE[pg_ranks]["bwd"]

    def group(self, src_stage: int, dst_stage: int):
        """Process group carrying src -> dst messages."""
        if (src_stage + 1) % self.n == dst_stage:
            return self.fwd[src_stage]
        if (dst_stage + 1) % self.n == src_stage:
            return self.bwd[dst_stage]
        raise ValueError(f"stages {src_stage}->{dst_stage} are not adjacent")


def _dev(group) -> torch.device:
    return torch.device("cuda", torch.cuda.current_device()) if dist.get_backend(group) == "nccl" else torch.device("cpu")


class NodeListScheduler(PipelineSchedule):
    """Executes per-stage `ScheduledNode` lists.  `schedule` is the list itself or a function `n_micro -> list` (the
    list is then built as soon as the number of micro-batches is known, and rebuilt when it changes)."""

    def __init__(self, stage_manager: PipelineStageManager,
                 schedule: Union[List[List[ScheduledNode]], Callable[[int], List[List[ScheduledNode]]]],
                 num_model_chunks: int,
                 num_microbatch: Optional[int] = None, microbatch_size: Optional[int] = None, v_shape: bool = True,
                 split_w: bool = True, enable_metadata_cache: bool = True, overlap_p2p: bool = True,
                 recv_lookahead: int = 1) -> None:
        super().__init__(stage_manager)
        self.num_microbatch, self.microbatch_size = num_microbatch, microbatch_size
        self.num_model_chunks = num_model_chunks
        self.v_shape, self.split_w = v_shape, split_w
        self.batch = None
        self.batch_size = None
        self.last_batch_size = None
        self.enable_metadata_cache = enable_metadata_cache
        self.recv_lookahead = recv_lookahead
        self._schedule_fn = schedule if callable(schedule) else None
        self._built_for: Optional[int] = None
        if self._schedule_fn is not None:
            self._built_for = num_microbatch
            schedule = self._schedule_fn(num_microbatch) if num_microbatch is not None \
                else [[] for _ in range(stage_manager.num_stages)]
        self.full_schedule = schedule
        self.channels = _Channels(stage_manager) if stage_manager.num_stages > 1 else None
        self._meta_cache: Dict[Tuple, P2PMetadata] = {}
        self._sent_meta: set = set()
        self._prepare(schedule)

    # ------------------------------------------------------------------ schedule analysis
    def _prepare(self, schedule: List[List[ScheduledNode]]) -> None:
        sm = self.stage_manager
        n = sm.num_stages
        self.my_nodes = schedule[sm.stage]
        self.n_pos = n * self.num_model_chunks
        # per incoming channel (src stage): the sender's message order
        self.incoming: Dict[int, deque] = defaultdict(deque)
        for s, nodes in enumerate(schedule):
            for nd in nodes:
                if nd.type not in ("SEND_FORWARD", "SEND_BACKWARD"):
                    continue
                pos = _stage_of(nd.chunk, s, n, self.v_shape)
                if nd.type == "SEND_FORWARD":
                    dc, ds = _locate(pos + 1, n, self.v_shape)
                    key = ("F", dc, nd.minibatch)
                else:
                    dc, ds = _locate(pos - 1, n, self.v_shape)
                    key = ("B", dc, nd.minibatch)
                if ds == sm.stage:
                    self.incoming[s].append(key)
        self._incoming_template = {k: list(v) for k, v in self.incoming.items()}

    def load_batch(self, data_iter, device=None) -> None:
        super().load_batch(data_iter, device)
        if self._schedule_fn is not None and self._built_for != self.num_microbatch:
            self.full_schedule = self._schedule_fn(self.num_microbatch)
            self._prepare(self.full_schedule)
            self._built_for = self.num_microbatch

    def reset_metadata_cache(self) -> None:
        self._meta_cache.clear()
        self._sent_meta.clear()

    # ------------------------------------------------------------------ p2p
    def _isend_obj(self, obj: Any, dst_stage: int, kind: Tuple) -> None:
        sm = self.stage_manager
        group = self.channels.group(sm.stage, dst_stage)
        dst_rank = self.channels.ranks[dst_stage]
        dev = _dev(group)
        md, tensors = create_send_metadata(obj, return_tensor=True)
        mkey = (dst_stage, kind[0], kind[1])
        if not (self.enable_metadata_cache and mkey in self._sent_meta):
            buf = pickle.dumps(md)
            size = torch.tensor([len(buf)], dtype=torch.int64, device=dev)
            data = torch.frombuffer(bytearray(buf), dtype=torch.uint8).to(dev)
            self._send_keep.append((dist.isend(size, dst_rank, group=group), size))
            self._send_keep.append((dist.isend(data, dst_rank, group=group), data))
            self._sent_meta.add(mkey)
        for t in tensors:
            t = t.detach().contiguous()
            if t.device != dev:
                t = t.to(dev)
            self._send_keep.append((dist.isend(t, dst_rank, group=group), t))

    def _post_recv(self, src_stage: int, kind: Tuple) -> None:
        sm = self.stage_manager
        group = self.channels.group(src_stage, sm.stage)
        src_rank = self.channels.ranks[src_stage]
        dev = _dev(group)
        mkey = (src_stage, kind[0], kind[1])
        md = self._meta_cache.get(mkey) if self.enable_metadata_cache else None
        if md is None:
            size = torch.empty(1, dtype=torch.int64, device=dev)
            dist.recv(size, src_rank, group=group)
            data = torch.empty(int(size.item()), dtype=torch.uint8, device=dev)
            dist.recv(data, src_rank, group=group)
            md = pickle.loads(data.cpu().numpy().tobytes())
            self._meta_cache[mkey] = md
        bufs, works = [], []
        for shape, dtype, _ in md.tensor_metadata:
            b = torch.empty(shape, dtype=dtype, device=dev)
            works.append(dist.irecv(b, src_rank, group=group))
            bufs.append(b)
        self._recv_posted[(src_stage,) + kind] = (md, bufs, works)

    def _recv_obj(self, src_stage: int, kind: Tuple) -> Any:
        """Post receives on the channel in the sender's order up to `kind` (+ lookahead), then wait for `kind`."""
        q = self._incoming_runtime[src_stage]
        need = (src_stage,) + kind
        while need not in self._recv_posted:
            nxt = q.popleft()
            self._post_recv(src_stage, nxt)
        for _ in range(self.recv_lookahead):
            if q:
                mkey = (src_stage, q[0][0], q[0][1])
                if mkey in self._meta_cache or not self.enable_metadata_cache:
                    if mkey in self._meta_cache:
                        self._post_recv(src_stage, q.popleft())
        md, bufs, works = self._recv_posted.pop(need)
        for w in works:
            w.wait()
        leaves: List[Any] = [None] * (len(bufs) + len(md.non_tensor_obj_idx))
        for i, o in zip(md.non_tensor_obj_idx, md.non_tensor_objs):
            leaves[i] = o
        it = iter(zip(bufs, md.tensor_metadata))
        for i in range(len(leaves)):
            if i not in md.non_tensor_obj_idx:
                t, (_, _, rg) = next(it)
                leaves[i] = t.requires_grad_(rg) if t.is_floating_point() else t
        return tree_unflatten(leaves, md.tree_spec)

    # ------------------------------------------------------------------ compute
    def _chunk_module(self, model: Union[Module, ModuleList], chunk: int) -> Module:
        inner = model.module if hasattr(model, "module") and isinstance(getattr(model, "module"), ModuleList) else model
        return inner[chunk] if isinstance(inner, ModuleList) else model

    def _forward(self, model, chunk: int, mb: int, criterion, accum_loss, outputs) -> None:
        sm = self.stage_manager
        n = sm.num_stages
        pos = _stage_of(chunk, sm.stage, n, self.v_shape)
        micro_batch = get_micro_batch(self.batch, mb * self.microbatch_size, self.microbatch_size)
        input_obj = None
        if pos > 0:
            pc, ps = _locate(pos - 1, n, self.v_shape)
            if ps == sm.stage:
                prev_out = self._local_fwd.pop((pc, mb))
                input_obj = tree_map(lambda t: t.detach().requires_grad_(t.requires_grad) if isinstance(t, Tensor)
                                     and t.is_floating_point() else t, prev_out)
            else:
                input_obj = self._recv_obj(ps, ("F", chunk, mb))
        with sm.switch_model_chunk_id(chunk):
            out = model_forward(self._chunk_module(model, chunk), micro_batch, input_obj)
            if pos == self.n_pos - 1:
                loss = criterion(out, micro_batch) / self.num_microbatch
                if accum_loss is not None:
                    accum_loss.add_(loss.detach())
                if outputs is not None:
                    outputs.append(tree_map(detach, out))
                out = loss
        self._saved[(chunk, mb)] = (input_obj, out)
        if pos < self.n_pos - 1:
            nc, ns = _locate(pos + 1, n, self.v_shape)
            if ns == sm.stage:
                self._local_fwd[(chunk, mb)] = out

    def _backward(self, optimizer, chunk: int, mb: int) -> None:
        sm = self.stage_manager
        n = sm.num_stages
        pos = _stage_of(chunk, sm.stage, n, self.v_shape)
        input_obj, out = self._saved.pop((chunk, mb))
        grad_obj = None
        if pos < self.n_pos - 1:
            nc, ns = _locate(pos + 1, n, self.v_shape)
            grad_obj = self._local_bwd.pop((nc, mb)) if ns == sm.stage else self._recv_obj(ns, ("B", chunk, mb))
        tree_map(retain_grad, input_obj)
        WeightGradStore.enabled = self.split_w
        try:
            if grad_obj is None:
                optimizer.backward(out)
            else:
                tensors, grads = [], []
                for k, g in grad_obj.items():
                    if isinstance(g, Tensor) and isinstance(out[k], Tensor) and out[k].requires_grad:
                        tensors.append(out[k])
                        grads.append(g)
                optimizer.backward_by_grad(tensors, grads)
        finally:
            WeightGradStore.enabled = False
        if self.split_w:
            WeightGradStore.flush(chunk)
        in_grad = None
        if input_obj is not None:
            in_grad = {k: v.grad for k, v in input_obj.items() if isinstance(v, Tensor) and v.grad is not None}
        if pos > 0:
            pc, ps = _locate(pos - 1, n, self.v_shape)
            if ps == sm.stage:
                self._local_bwd[(chunk, mb)] = in_grad
            else:
                self._grad_out[(chunk, mb)] = in_grad

    # ------------------------------------------------------------------ run
    def run(self, model, data_iter, criterion, optimizer, return_loss: bool, return_outputs: bool,
            forward_only: bool) -> Dict:
        self.load_batch(data_iter)
        sm = self.stage_manager
        n = sm.num_stages
        self._saved: Dict = {}
        self._local_fwd: Dict = {}
        self._local_bwd: Dict = {}
        self._grad_out: Dict = {}
        self._fwd_out: Dict = {}
        self._send_keep: List = []
        self._recv_posted: Dict = {}
        self._incoming_runtime = {k: deque(v) for k, v in self._incoming_template.items()}
        WeightGradStore.clear()
        last_holder = any(_stage_of(c, sm.stage, n, self.v_shape) == self.n_pos - 1
                          for c in range(self.num_model_chunks))
        accum_loss = torch.scalar_tensor(0, device=get_accelerator().get_current_device()) \
            if (return_loss and last_holder) else None
        outputs = [] if (return_outputs and last_holder) else None
        for nd in self.my_nodes:
            if nd.type == "F":
                self._forward(model, nd.chunk, nd.minibatch, criterion, accum_loss, outputs)
            elif nd.type == "B":
                if not forward_only:
                    self._backward(optimizer, nd.chunk, nd.minibatch)
            elif nd.type == "W":
                if not forward_only and self.split_w:
                    WeightGradStore.pop(nd.chunk)
            elif nd.type == "SEND_FORWARD":
                pos = _stage_of(nd.chunk, sm.stage, n, self.v_shape)
                dc, ds = _locate(pos + 1, n, self.v_shape)
                _, out = self._saved[(nd.chunk, nd.minibatch)] if (nd.chunk, nd.minibatch) in self._saved else (None, None)
                self._isend_obj(out, ds, ("F", dc, nd.minibatch))
                if forward_only:
                    self._saved.pop((nd.chunk, nd.minibatch), None)
            elif nd.type == "SEND_BACKWARD":
                if forward_only:
                    continue
                pos = _stage_of(nd.chunk, sm.stage, n, self.v_shape)
                dc, ds = _locate(pos - 1, n, self.v_shape)
                self._isend_obj(self._grad_out.pop((nd.chunk, nd.minibatch)), ds, ("B", dc, nd.minibatch))
            # RECV_* nodes are satisfied lazily by _recv_obj (posting order == sender order)
        for w, _ in self._send_keep:
            w.wait()
        self._send_keep.clear()
        if forward_only:
            self._saved.clear()
        assert not self._saved and not self._local_fwd and not self._local_bwd, "pipeline buffers not drained"
        if outputs is not None:
            outputs = merge_batch(outputs)
        return {"loss": accum_loss, "outputs": outputs}

    def forward_backward_step(self, model: Module, data_iter: Iterable, criterion: Optional[Callable] = None,
                              optimizer: Optional[OptimizerWrapper] = None, return_loss: bool = False,
                              return_outputs: bool = False) -> dict:
        criterion = criterion or default_criterion
        forward_only = not torch.is_grad_enabled()
        if optimizer is None:
            assert forward_only, "Optimizer should be passed when doing backward."
        return self.run(model, data_iter, criterion, optimizer, return_loss, return_outputs, forward_only)


class ZeroBubbleVPipeScheduler(NodeListScheduler):
    """ZB-V: 2 chunks per stage in a V, B = dX only, W deferred.  `schedule` defaults to `PipelineGraph` output."""

    def __init__(self, stage_manager: PipelineStageManager, schedule: Optional[List[List[ScheduledNode]]] = None,
                 num_model_chunks: int = 2, num_microbatch: Optional[int] = None,
                 microbatch_size: Optional[int] = None, enable_metadata_cache: bool = True,
                 overlap_p2p: bool = True) -> None:
        assert num_model_chunks == 2, "ZB-V uses exactly 2 model chunks per stage"
        if schedule is None:
            assert num_microbatch is not None, "num_microbatch is needed to build the default ZB-V schedule"
            schedule = PipelineGraph(stage_manager.num_stages, num_microbatch, f_cost=2, b_cost=2, w_cost=2, c_cost=0,
                                     f_mem=1.0, b_mem=-0.5, w_mem=-0.5).get_v_schedule()
        super().__init__(stage_manager, schedule, num_model_chunks, num_microbatch, microbatch_size, v_shape=True,
                         split_w=True, enable_metadata_cache=enable_metadata_cache, overlap_p2p=overlap_p2p)

    def assert_buffer_empty(self) -> None:
        assert not getattr(self, "_saved", None) and not getattr(self, "_local_fwd", None)
