"""Vocab-parallel cross entropy and log-prob.

Parity: reference `colossalai/shardformer/layer/loss.py:25-356` (`DistCrossEntropy`, `DistLogProb`,
`dist_cross_entropy` with label shift + SP/ring-attn label split + loss reduction over SP).
H100-first: the three all-reduces of the reference (max, target-logit, exp-sum) are packed into two
(one MAX, one SUM over a stacked [2, T] buffer) and the softmax statistics / gradient come from a fused kernel
(`ops.cross_entropy`), so the [T, V/tp] logits are read once in forward and written once in backward.
"""
from __future__ import annotations

from typing import Optional, Tuple

import torch
import torch.distributed as dist
import torch.nn.functional as F
from torch.distributed import ProcessGroup

from ...ops import cross_entropy as ce_ops
from ...parallel import comm
from ._operation import reduce_forward, split_batch_zigzag

__all__ = ["DistCrossEntropy", "DistLogProb", "cross_entropy_1d", "dist_log_prob_1d", "dist_cross_entropy", "dist_log_prob"]

_IGNORE_INDEX = -100
_LOCAL = "local"   # sentinel process group: no vocab parallelism (None means WORLD, torch semantics)


def _ws_rank(process_group):
    if isinstance(process_group, str) and process_group == _LOCAL:
        return 1, 0
    return comm.group_size(process_group), comm.group_rank(process_group)


class DistCrossEntropy(torch.autograd.Function):
    """loss = mean_{valid}( log(sum_j exp(x_j)) - x_target ) over vocab-parallel logits [T, V_local]."""

    @staticmethod
    def forward(ctx, vocab_logits: torch.Tensor, target: torch.Tensor, ignore_index: int, process_group,
                vocab_size: Optional[int], dtype=torch.float32, mode: str = "mean"):
        T, V_local = vocab_logits.shape
        ws, rank = _ws_rank(process_group)
        # vocab range owned by this rank (padded vocab is sharded evenly)
        global_vocab = V_local * ws if vocab_size is None else vocab_size
        start = rank * V_local
        # columns beyond the true vocab (padding added so the vocab divides tp * 64) must not enter the softmax
        vcols = V_local if vocab_size is None else max(min(V_local, vocab_size - start), 0)
        # local statistics: max, sumexp (relative to the GLOBAL max after all-reduce), target logit
        local_max = ce_ops.row_max(vocab_logits, vcols) if vcols > 0 else \
            torch.full((T,), float("-inf"), device=vocab_logits.device)           # [T] fp32
        if ws > 1:
            dist.all_reduce(local_max, op=dist.ReduceOp.MAX, group=process_group)
        stats = ce_ops.sumexp_and_target(vocab_logits, target, local_max, start, ignore_index, vcols)  # [2, T] fp32
        if ws > 1:
            dist.all_reduce(stats, group=process_group)
        sumexp, tgt_logit = stats[0], stats[1]
        valid = target != ignore_index
        n_valid = valid.sum()
        loss_tok = torch.where(valid, torch.log(sumexp) + local_max - tgt_logit, torch.zeros_like(sumexp))
        if mode == "mean":
            loss = loss_tok.sum() / n_valid.clamp(min=1)
        elif mode == "sum":
            loss = loss_tok.sum()
        else:
            raise ValueError(mode)
        ctx.save_for_backward(vocab_logits, target, local_max, sumexp, n_valid)
        ctx.start, ctx.ignore_index, ctx.mode, ctx.valid = start, ignore_index, mode, vcols
        return loss.to(dtype)

    @staticmethod
    def backward(ctx, grad_output):
        logits, target, gmax, sumexp, n_valid = ctx.saved_tensors
        scale = grad_output.float()
        if ctx.mode == "mean":
            scale = scale / n_valid.clamp(min=1)
        grad = ce_ops.softmax_grad(logits, target, gmax, sumexp, scale, ctx.start, ctx.ignore_index,
                                   valid_cols=ctx.valid)
        return grad, None, None, None, None, None, None


class DistLogProb(torch.autograd.Function):
    """log p(target) per token from vocab-parallel logits (RLHF / GRPO)."""

    @staticmethod
    def forward(ctx, vocab_logits: torch.Tensor, target: torch.Tensor, process_group, vocab_size, dtype=torch.float32):
        shape = target.shape
        logits = vocab_logits.reshape(-1, vocab_logits.shape[-1])
        tgt = target.reshape(-1)
        ws, rank = _ws_rank(process_group)
        V_local = logits.shape[-1]
        start = rank * V_local
        valid = V_local if vocab_size is None else max(min(V_local, vocab_size - start), 0)
        gmax = ce_ops.row_max(logits, valid)
        if ws > 1:
            dist.all_reduce(gmax, op=dist.ReduceOp.MAX, group=process_group)
        stats = ce_ops.sumexp_and_target(logits, tgt, gmax, start, -(10**9), valid)
        if ws > 1:
            dist.all_reduce(stats, group=process_group)
        logp = stats[1] - gmax - torch.log(stats[0])
        ctx.save_for_backward(logits, tgt, gmax, stats[0])
        ctx.start, ctx.shape, ctx.valid = start, shape, valid
        return logp.view(shape).to(dtype)

    @staticmethod
    def backward(ctx, grad_output):
        logits, tgt, gmax, sumexp = ctx.saved_tensors
        # d logp / d x_j = 1[j == t] - softmax_j  == -(softmax - onehot)
        g = ce_ops.softmax_grad(logits, tgt, gmax, sumexp, None, ctx.start, -(10**9),
                                row_scale=-grad_output.reshape(-1).float(), valid_cols=ctx.valid)
        return g.view(logits.shape), None, None, None, None


def cross_entropy_1d(vocab_logits: torch.Tensor, labels: torch.Tensor, ignore_index: int = _IGNORE_INDEX,
                     process_group: ProcessGroup = None, vocab_size: int = None, dtype: torch.dtype = None,
                     mode: str = "mean") -> torch.Tensor:
    return DistCrossEntropy.apply(vocab_logits, labels, ignore_index, process_group, vocab_size,
                                  dtype or torch.float32, mode)


def dist_log_prob_1d(vocab_logits, labels, process_group=None, vocab_size=None, dtype=None) -> torch.Tensor:
    return DistLogProb.apply(vocab_logits, labels, process_group, vocab_size, dtype or torch.float32)


def dist_cross_entropy(labels: torch.Tensor, logits: torch.Tensor, shard_config, vocab_size: int,
                       dtype: torch.dtype = torch.float32, seq_dim: int = 1, shift: bool = True) -> torch.Tensor:
    """Causal-LM loss on token-major or [B, S, V] logits, aware of TP (vocab-parallel logits), SP modes and
    ring attention's zigzag layout.  `labels` are the FULL un-shifted labels [B, S]."""
    sp_group = getattr(shard_config, "sequence_parallel_process_group", None)
    sp_mode = getattr(shard_config, "sequence_parallelism_mode", None)
    sp_size = comm.group_size(sp_group) if getattr(shard_config, "enable_sequence_parallelism", False) else 1
    parallel_output = getattr(shard_config, "parallel_output", True)
    is_sp = sp_size > 1 and not (sp_mode in ("split_gather", "ring"))  # logits still sequence-sharded
    B = labels.shape[0]
    if shift:
        # predict token t+1: pad the shifted labels with ignore_index so the split stays even
        labels = torch.cat([labels[:, 1:], labels.new_full((B, 1), _IGNORE_INDEX)], dim=1)
    if is_sp:
        if sp_mode == "ring_attn":
            labels = split_batch_zigzag(labels, sp_group, seq_dim=1)
        else:
            labels = labels.chunk(sp_size, dim=1)[comm.group_rank(sp_group)]
    labels = labels.reshape(-1).contiguous()
    logits = logits.reshape(-1, logits.shape[-1])
    assert logits.shape[0] == labels.shape[0], f"logits rows {logits.shape[0]} vs labels {labels.shape[0]}"
    tp_group = getattr(shard_config, "tensor_parallel_process_group", None)
    use_dist = getattr(shard_config, "enable_tensor_parallelism", False) and parallel_output \
        and comm.group_size(tp_group) > 1
    if is_sp:
        n_local = (labels != _IGNORE_INDEX).sum()
        loss_sum = cross_entropy_1d(logits, labels, process_group=tp_group if use_dist else _LOCAL,
                                    vocab_size=vocab_size, dtype=dtype, mode="sum")
        # reduce (sum, count) over SP.  Parameter grads are later AVERAGED over the dp x sp group, so every rank's
        # partial gradient is scaled up by sp here (reference: loss.py:350-355, grad_scale=sp)
        loss_sum = reduce_forward(loss_sum, sp_group, grad_scale=float(sp_size))
        n_total = n_local.clone()
        dist.all_reduce(n_total, group=sp_group)
        return loss_sum / n_total.clamp(min=1)
    return cross_entropy_1d(logits, labels, process_group=tp_group if use_dist else _LOCAL, vocab_size=vocab_size,
                            dtype=dtype)


def dist_log_prob(labels: torch.Tensor, logits: torch.Tensor, shard_config, vocab_size: int,
                  dtype: torch.dtype = torch.float32, seq_dim: int = 1) -> torch.Tensor:
    tp_group = getattr(shard_config, "tensor_parallel_process_group", None)
    use_dist = getattr(shard_config, "enable_tensor_parallelism", False) and \
        getattr(shard_config, "parallel_output", True) and comm.group_size(tp_group) > 1
    return dist_log_prob_1d(logits, labels, tp_group if use_dist else _LOCAL, vocab_size, dtype)
