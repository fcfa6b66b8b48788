"""Continuous-batching scheduler.

Parity: reference `colossalai/inference/core/request_handler.py:19-452` (`RunningList`, `RequestHandler.schedule`:
waiting lists bucketed by prompt length, prefill bucket vs decoding bucket, prefill-ratio trigger, recycle on KV OOM,
abort over-long prompts, streamingLLM update, finished-sequence collection).
"""
from __future__ import annotations

from typing import Dict, List, Optional

import torch

from ...logging import get_dist_logger
from ..batch_bucket import BatchBucket
from ..config import InferenceConfig
from ..kv_cache import KVCacheManager
from ..sampler import search_tokens
from ..struct import RequestStatus, Sequence

__all__ = ["RunningList", "RequestHandler", "NaiveRequestHandler"]

logger = get_dist_logger(__name__)


class RunningList:
    """Sequences currently on the device: `prefill` (not yet run) and `decoding`."""

    def __init__(self, prefill_ratio: float, prefill: List[Sequence] = None) -> None:
        self.prefill_ratio = prefill_ratio
        self._decoding: Dict[int, Sequence] = {}
        self._prefill: Dict[int, Sequence] = {s.request_id: s for s in prefill} if prefill else {}

    @property
    def decoding(self) -> List[Sequence]:
        return list(self._decoding.values())

    @property
    def prefill(self) -> List[Sequence]:
        return list(self._prefill.values())

    @property
    def prefill_seq_num(self) -> int:
        return len(self._prefill)

    @property
    def decoding_seq_num(self) -> int:
        return len(self._decoding)

    @property
    def total_seq_num(self) -> int:
        return self.prefill_seq_num + self.decoding_seq_num

    def append(self, seq: Sequence) -> None:
        assert seq.request_id not in self._prefill and seq.request_id not in self._decoding
        self._prefill[seq.request_id] = seq

    def extend(self, seqs: List[Sequence]) -> None:
        for s in seqs:
            self._prefill[s.request_id] = s

    def find_seq(self, request_id: int) -> Optional[Sequence]:
        return self._decoding.get(request_id) or self._prefill.get(request_id)

    def remove(self, seq: Sequence) -> None:
        if seq.request_id in self._decoding:
            self._decoding.pop(seq.request_id)
        elif seq.request_id in self._prefill:
            self._prefill.pop(seq.request_id)
        else:
            raise ValueError(f"Sequence {seq.request_id} is not in the running list")

    def ready_for_prefill(self) -> bool:
        if not self._decoding:
            return len(self._prefill) > 0
        return len(self._prefill) / len(self._decoding) >= self.prefill_ratio

    def is_empty(self) -> bool:
        return not self._decoding and not self._prefill

    def mark_prefill_running(self) -> None:
        for s in self._prefill.values():
            s.mark_running()

    def move_prefill_to_decoding(self, seq_ids: List[int]) -> None:
        for sid in seq_ids:
            assert sid in self._prefill, f"Sequence {sid} is not in the prefill list"
            self._decoding[sid] = self._prefill.pop(sid)


class NaiveRequestHandler:
    """Minimal FIFO handler used by non-LLM engines (diffusion)."""

    def __init__(self) -> None:
        self.running_list: List = []
        self.waiting_list: List = []

    def _has_waiting(self) -> bool:
        return len(self.waiting_list) > 0

    def _has_running(self) -> bool:
        return len(self.running_list) > 0

    def check_unfinished_reqs(self) -> bool:
        return self._has_waiting() or self._has_running()

    def add_sequence(self, seq) -> None:
        self.waiting_list.append(seq)

    def _find_sequence(self, request_id: int):
        for lst in (self.waiting_list, self.running_list):
            for s in lst:
                if getattr(s, "request_id", None) == request_id:
                    return s
        return None

    def schedule(self):
        if self._has_waiting():
            s = self.waiting_list.pop(0)
            self.running_list.append(s)
            return s
        return None


class RequestHandler(NaiveRequestHandler):
    def __init__(self, inference_config: InferenceConfig, model_config) -> None:
        super().__init__()
        self.inference_config = inference_config
        self.running_list: RunningList = RunningList(inference_config.prefill_ratio)
        self.waiting_list: List[List[Sequence]] = [[], [], []]
        self.done_list: List[Sequence] = []
        self.dtype = inference_config.dtype
        self.max_batch_size = inference_config.max_batch_size
        self._init_cache(model_config)
        head_dim = model_config.head_dim
        kw = dict(num_heads=model_config.num_attention_heads // inference_config.tp_size, head_dim=head_dim,
                  max_batch_size=self.max_batch_size, max_length=inference_config.max_input_len + inference_config.max_output_len,
                  block_size=inference_config.block_size, kv_max_split_num=1, dtype=self.dtype,
                  enable_streamingllm=inference_config.enable_streamingllm,
                  start_token_size=inference_config.start_token_size,
                  generated_token_size=inference_config.generated_token_size)
        self.running_bb = BatchBucket(**kw)
        self.prefill_bb = BatchBucket(**kw)
        # chunked prefill: the step `_schedule_chunks` planned
        self.prefill_chunks: List[int] = []
        self.decode_in_step = False

    def _init_cache(self, model_config) -> None:
        self.cache_manager = KVCacheManager(self.inference_config, model_config)

    def _has_waiting(self) -> bool:
        return any(lst for lst in self.waiting_list)

    def _has_running(self) -> bool:
        return not self.running_bb.is_empty

    def get_kvcache(self):
        return self.cache_manager.get_kv_cache()

    def set_spec_dec_mode(self, n_spec_tokens: int) -> None:
        self.prefill_bb.set_use_spec_dec(n_spec_tokens)
        self.running_bb.set_use_spec_dec(n_spec_tokens)

    def unset_spec_dec_mode(self) -> None:
        self.prefill_bb.reset_use_spec_dec()
        self.running_bb.reset_use_spec_dec()

    def schedule(self) -> BatchBucket:
        """Returns the bucket to run this step: a prefill bucket when enough prompts are waiting, else decoding.  With
        `max_num_batched_tokens` set, see `_schedule_chunks`."""
        if self._has_waiting():
            for lst in reversed(self.waiting_list):
                if not lst:
                    continue
                # abort over-long prompts
                if lst[0].input_len > self.inference_config.max_input_len:
                    seq = lst.pop(0)
                    logger.warning(f"prompt of request {seq.request_id} is longer than max_input_len; aborted")
                    seq.mark_aborted()
                    self.done_list.append(seq)
                    continue
                remain = self.max_batch_size - self.running_list.total_seq_num
                while lst and remain > 0 and self.cache_manager.check_allocation(lst[0]):
                    seq = lst.pop(0)
                    self.running_list.append(seq)
                    remain -= 1
        if self.inference_config.max_num_batched_tokens is not None:
            return self._schedule_chunks()
        if self.running_list.ready_for_prefill() and self.prefill_bb.is_empty:
            n = min(self.running_list.prefill_seq_num, self.running_bb.available_batch_size)
            seqs = self.running_list.prefill[:n]
            if seqs:
                self._start_prefill(seqs)
                return self.prefill_bb
        self._reserve_decode_tokens()
        return self.running_bb

    def _start_prefill(self, seqs: List[Sequence]) -> None:
        """Move admitted prompts into the prefill bucket with blocks for their whole prompt (sharing prefix-cache
        hits)."""
        self.running_list.mark_prefill_running()
        alloc = self.cache_manager.allocate_context_from_block_tables
        if self.inference_config.enable_prefix_caching:
            def alloc(tables, lens, seqs=list(seqs)):
                for i, s in enumerate(seqs):
                    s.num_cached_tokens = self.cache_manager.allocate_context_with_prefix(tables[i],
                                                                                          s.input_token_id)
        self.prefill_bb.add_seqs(list(seqs), alloc_block_tables_fn=alloc)
        self.running_list.move_prefill_to_decoding([s.request_id for s in seqs])

    def _schedule_chunks(self) -> BatchBucket:
        """Chunked prefill.  Admitted prompts join the prefill bucket at once and stay there until their last chunk
        has run.  A step holds one token of every decoding sequence, then prompt chunks up to `max_num_batched_tokens`
        in total, first come first served: a prompt gets tokens only once every earlier prompt is fully scheduled.
        Every chunk but a prompt's last is a whole number of blocks, and chunks start where the cached tokens end, on a
        block boundary.  Speculative decoding verifies in a pass of its own, so while prompts are pending its steps
        hold chunks only.

        Returns the prefill bucket when the step feeds chunks - `prefill_chunks[i]` tokens of its i-th sequence,
        followed by the decoding bucket's rows when `decode_in_step` - else the decoding bucket (a plain decode
        step)."""
        seqs = self.running_list.prefill
        if seqs:
            self._start_prefill(seqs)
        budget = self.inference_config.max_num_batched_tokens
        self.decode_in_step = self.prefill_bb.is_empty or not self.running_bb.use_spec_dec
        if self.decode_in_step:
            self._reserve_decode_tokens()
            budget -= self.running_bb.current_batch_size
        bs = self.inference_config.block_size
        self.prefill_chunks = []
        for s in self.prefill_bb.seqs_li:
            left = s.input_len - s.num_cached_tokens
            n = min(left, budget)
            if n < left:
                n -= n % bs
            if n == 0:
                break
            self.prefill_chunks.append(n)
            budget -= n
            if n < left:
                break
        return self.prefill_bb if self.prefill_chunks else self.running_bb

    def _reserve_decode_tokens(self) -> None:
        # room for this step's token(s) of every running sequence.  The cache is sized for the worst case, so this
        # only fails under over-subscription (speculative look-ahead); then the youngest sequence goes back to the
        # waiting list and the allocation is RETRIED - the failed pass stopped at the first sequence without a block,
        # the ones behind it have none yet either (allocation of an already assigned slot is a no-op)
        while not self.running_bb.is_empty:
            try:
                n_new = self.running_bb.num_tokens_to_verify + 1 if self.running_bb.use_spec_dec else 1
                if n_new == 1:
                    self.cache_manager.allocate_tokens_from_block_tables(self.running_bb.block_tables,
                                                                         self.running_bb.seq_lengths + 1,
                                                                         self.running_bb.current_batch_size)
                else:
                    self.cache_manager.allocate_n_tokens_from_block_tables(
                        self.running_bb.block_tables, self.running_bb.seq_lengths,
                        self.running_bb.current_batch_size, n_new)
                break
            except RuntimeError:
                self._recycle_last()

    def _recycle_last(self) -> None:
        """KV cache exhausted: push the most recent sequence back to the waiting list and free its blocks.  Prompts
        still being prefilled (chunked prefill) are younger than every decoding sequence, so they go first."""
        bucket = self.running_bb if self.prefill_bb.is_empty else self.prefill_bb
        self._index_prefix(bucket, bucket.seqs_li[-1:])
        seqs, _ = bucket.pop_n_seqs(1, self.cache_manager.free_block_table)
        for s in seqs:
            self.running_list.remove(s)
            s.recycle()
            s.input_token_id = s.input_token_id + s.output_token_id
            s.output_token_id = []
            self.waiting_list[-1].insert(0, s)

    def allocate_batch_spec_dec(self, batch: BatchBucket, n: int) -> None:
        if batch.current_batch_size:
            self.cache_manager.allocate_n_tokens_from_block_tables(batch.block_tables, batch.seq_lengths,
                                                                   batch.current_batch_size, n)

    def add_sequence(self, req: Sequence) -> None:
        assert not self._find_sequence(req.request_id), f"Sequence {req.request_id} already exists."
        assert req.input_len <= self.inference_config.max_input_len, (
            f"Sequence {req.request_id} exceeds input length limit")
        idx = min((req.input_len * 3 - 1) // max(self.inference_config.max_input_len, 1), 2)
        self.waiting_list[idx].append(req)

    def abort_sequence(self, request_id: int) -> None:
        seq, where = self._find_sequence_with_list(request_id)
        if seq is None:
            return
        if where == "waiting":
            for lst in self.waiting_list:
                if seq in lst:
                    lst.remove(seq)
        else:
            for bucket in (self.running_bb, self.prefill_bb):      # a prompt mid-prefill sits in the prefill bucket
                if request_id in bucket.seqs_ids:
                    self._index_prefix(bucket, [seq])
                    bucket.pop_seq_update_batch(request_id, self.cache_manager.free_block_table)
            self.running_list.remove(seq)
        seq.mark_aborted()

    def _find_sequence_with_list(self, request_id: int):
        for lst in self.waiting_list:
            for s in lst:
                if s.request_id == request_id:
                    return s, "waiting"
        s = self.running_list.find_seq(request_id)
        return (s, "running") if s is not None else (None, None)

    def _find_sequence(self, request_id: int) -> Optional[Sequence]:
        return self._find_sequence_with_list(request_id)[0]

    def update_seq_finished(self, sequence: Sequence, generation_config) -> bool:
        return sequence.check_finish()

    def update_batch_finished(self, batch: BatchBucket, generation_config) -> None:
        for s in batch.seqs_li:
            s.check_finish()

    def check_unfinished_reqs(self) -> bool:
        return self._has_waiting() or not self.running_list.is_empty()

    def total_requests_in_batch_bucket(self) -> int:
        return self.prefill_bb.current_batch_size + self.running_bb.current_batch_size

    def append_next_tokens(self, sample_tokens: torch.Tensor) -> None:
        if not self.prefill_bb.is_empty:
            self.prefill_bb.append_batch_tokens(sample_tokens)
        else:
            self.running_bb.append_batch_tokens(sample_tokens)

    def append_chunked_tokens(self, sample_tokens: List[int]) -> None:
        """After a chunked-prefill step: every fed prompt advances by its chunk; the prompts completed by it take their
        first token (the leading entries of `sample_tokens`), the decoding sequences the rest."""
        i = 0
        for s, n in zip(self.prefill_bb.seqs_li, self.prefill_chunks):
            s.num_cached_tokens += n
            if s.num_cached_tokens == s.input_len:
                s.output_token_id.append(sample_tokens[i])
                i += 1
        if self.decode_in_step and not self.running_bb.is_empty:
            self.running_bb.append_batch_tokens(torch.tensor(sample_tokens[i:]))

    def update(self) -> List[Sequence]:
        """Move freshly prefetched sequences into the decoding bucket, collect finished ones."""
        if self.inference_config.max_num_batched_tokens is not None:
            done = [s for s in self.prefill_bb.seqs_li if s.output_len]         # prompts completed in this step
            self._index_prefix(self.prefill_bb, done)
            self.running_bb.merge(self.prefill_bb, [s.request_id for s in done])
        elif not self.prefill_bb.is_empty:
            self._index_prefix(self.prefill_bb, self.prefill_bb.seqs_li)
            self.running_bb.merge(self.prefill_bb)
        self._index_prefix(self.running_bb, [s for s in self.running_bb.seqs_li if s.check_finish()])
        finished = self.running_bb.pop_finished(self.cache_manager.free_block_table)
        for s in finished:
            self.running_list.remove(s)
        self.done_list.extend(finished)
        if self.inference_config.enable_streamingllm and not self.running_bb.is_empty:
            freed = self.running_bb.streamingllm_update_batch(self.inference_config.start_token_size,
                                                              self.inference_config.generated_token_size)
            self.cache_manager.streamingllm_free_block_tables(freed)
        return finished

    def _index_prefix(self, bucket: BatchBucket, seqs: List[Sequence]) -> None:
        """Prefix caching: index the full blocks of `seqs` whose K/V are written - every position but the last
        sampled token's (which has none yet, as have rejected speculative tokens), or, for a prompt still being
        prefilled, its first `num_cached_tokens` positions."""
        if not self.inference_config.enable_prefix_caching:
            return
        for s in seqs:
            written = s.sentence_len - 1 if s.output_len else s.num_cached_tokens
            self.cache_manager.register_prefix_blocks(bucket.block_table_of(s.request_id),
                                                      s.input_token_id + s.output_token_id, written)

    def streamingllm_free_block_tables(self, updated_block_ids: List[int]) -> None:
        self.cache_manager.streamingllm_free_block_tables(updated_block_ids)


class RPCRequestHandler(RequestHandler):
    """Scheduler-side handler for the RPC engine: logical block tables only, the physical KV cache lives in the worker
    processes.  Parity: reference `inference/core/request_handler.py:352-398`."""

    def _init_cache(self, model_config) -> None:
        from ..kv_cache import RPCKVCacheManager

        self.cache_manager = RPCKVCacheManager(self.inference_config, model_config)

    def get_kvcache(self):
        raise RuntimeError("the RPC scheduler holds no physical KV cache")
