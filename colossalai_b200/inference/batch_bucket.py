"""Tensor-backed batch state.  Parity: reference `colossalai/inference/batch_bucket.py:9-560` (block tables + sequence
lengths per running batch, add / pop / merge / compaction, speculative-token revoke, StreamingLLM window update)."""
from __future__ import annotations

from typing import Callable, Dict, List, Optional, Tuple, Union

import torch

from .struct import Sequence

__all__ = ["BatchBucket"]


class BatchBucket:
    def __init__(self, num_heads: int, head_dim: int, max_batch_size: int, max_length: int, block_size: int,
                 kv_max_split_num: int, fd_interm_tensor=None, device=None, dtype=torch.float16,
                 enable_streamingllm: bool = False, start_token_size: int = 4, generated_token_size: int = 512) -> None:
        self.num_heads, self.head_dim = num_heads, head_dim
        self.max_batch_size, self.max_length = max_batch_size, max_length
        self.block_size, self.kv_max_split_num = block_size, kv_max_split_num
        self.fd_interm_tensor = fd_interm_tensor
        self.device = device or torch.device("cpu")
        self.dtype = dtype
        self.enable_streamingllm = enable_streamingllm
        self.start_token_size, self.generated_token_size = start_token_size, generated_token_size
        self._use_spec_dec = False
        self._num_tokens_to_verify = None
        self._current_batch_size = 0
        self._sequences_dict: Dict[int, Sequence] = {}
        self._sequences_indexes: Dict[int, int] = {}
        self._sequence_lengths = torch.zeros(max_batch_size, dtype=torch.int32)
        self._sequence_lengths_helper = torch.zeros_like(self._sequence_lengths)
        max_blocks = (max_length + block_size - 1) // block_size
        self._block_tables = torch.full((max_batch_size, max_blocks), -1, dtype=torch.int32)
        self._block_tables_helper = torch.full_like(self._block_tables, -1)

    # ------------------------------------------------------------------ properties
    @property
    def is_empty(self) -> bool:
        return self._current_batch_size == 0

    @property
    def current_batch_size(self) -> int:
        return self._current_batch_size

    def __len__(self) -> int:
        return self._current_batch_size

    @property
    def available_batch_size(self) -> int:
        return self.max_batch_size - self._current_batch_size

    @property
    def block_tables(self) -> torch.Tensor:
        return self._block_tables

    @property
    def seq_lengths(self) -> torch.Tensor:
        return self._sequence_lengths

    @property
    def seqs_ids(self) -> List[int]:
        return list(self._sequences_dict.keys())

    @property
    def seqs_li(self) -> List[Sequence]:
        return list(self._sequences_dict.values())

    @property
    def is_compact(self) -> bool:
        assert len(self._sequences_dict) == len(self._sequences_indexes)
        n = len(self._sequences_dict)
        return bool((self._sequence_lengths[:n] > 0).all()) and not bool(self._sequence_lengths[n:].any())

    @property
    def use_spec_dec(self) -> bool:
        return self._use_spec_dec

    @property
    def num_tokens_to_verify(self) -> int:
        return self._num_tokens_to_verify

    @property
    def batch_token_ids(self) -> List[List[int]]:
        return [s.input_token_id + s.output_token_id for s in self.seqs_li]

    def has_reused_seqs(self) -> bool:
        return any(s.output_len > 0 for s in self._sequences_dict.values())

    def set_use_spec_dec(self, num_tokens_to_verify: int = 5) -> None:
        self._use_spec_dec = True
        self._num_tokens_to_verify = num_tokens_to_verify

    def reset_use_spec_dec(self) -> None:
        self._use_spec_dec = False
        self._num_tokens_to_verify = None

    # ------------------------------------------------------------------ mutation
    def _make_compact(self) -> None:
        if self.is_compact:
            return
        valid = self._sequence_lengths.nonzero().view(-1)
        n = valid.numel()
        self._sequence_lengths_helper[:n] = self._sequence_lengths[valid]
        self._sequence_lengths_helper[n:] = 0
        self._sequence_lengths, self._sequence_lengths_helper = self._sequence_lengths_helper, self._sequence_lengths
        self._block_tables_helper[:n] = self._block_tables[valid]
        self._block_tables_helper[n:] = -1
        self._block_tables, self._block_tables_helper = self._block_tables_helper, self._block_tables
        new_idx = {}
        order = {int(v): i for i, v in enumerate(valid.tolist())}
        for sid, old in self._sequences_indexes.items():
            new_idx[sid] = order[old]
        self._sequences_indexes = new_idx

    def add_seq(self, seq: Sequence, alloc_block_table: torch.Tensor = None,
                alloc_block_table_fn: Callable[[torch.Tensor, int], None] = None) -> Union[torch.Tensor, None]:
        if self._current_batch_size >= self.max_batch_size:
            return None
        self._sequences_dict[seq.request_id] = seq
        idx = self._current_batch_size
        self._sequences_indexes[seq.request_id] = idx
        self._sequence_lengths[idx] = seq.sentence_len
        block_table = self._block_tables[idx]
        if alloc_block_table is not None:
            self._block_tables[idx] = alloc_block_table
        elif alloc_block_table_fn:
            alloc_block_table_fn(block_table, int(self._sequence_lengths[idx]))
        self._current_batch_size += 1
        return block_table

    def add_seqs(self, seqs: List[Sequence], alloc_block_tables: torch.Tensor = None,
                 alloc_block_tables_fn: Callable[[torch.Tensor, torch.Tensor], None] = None) -> torch.Tensor:
        assert seqs
        n = min(len(seqs), self.available_batch_size)
        if n == 0:
            return None
        start = self._current_batch_size
        for i, seq in enumerate(seqs[:n]):
            self._sequences_dict[seq.request_id] = seq
            self._sequences_indexes[seq.request_id] = start + i
            self._sequence_lengths[start + i] = seq.sentence_len
        tables = self._block_tables[start:start + n]
        lens = self._sequence_lengths[start:start + n]
        if alloc_block_tables is not None:
            self._block_tables[start:start + n] = alloc_block_tables
        elif alloc_block_tables_fn:
            alloc_block_tables_fn(tables, lens)
        self._current_batch_size += n
        seqs[:] = seqs[n:]
        return tables

    def pop_seq_update_batch(self, request_id: int, free_block_table_fn: Callable = None
                             ) -> Tuple[Optional[Sequence], Optional[torch.Tensor]]:
        if request_id not in self._sequences_dict:
            return None, None
        seq = self._sequences_dict.pop(request_id)
        idx = self._sequences_indexes.pop(request_id)
        table = self._block_tables[idx].clone()
        if free_block_table_fn:
            free_block_table_fn(self._block_tables[idx])
        else:
            self._block_tables[idx].fill_(-1)
        self._sequence_lengths[idx] = 0
        self._current_batch_size -= 1
        self._make_compact()
        return seq, table

    def pop_seqs(self, request_ids: List[int], free_block_table_fn: Callable = None):
        seqs, tables = [], []
        for rid in request_ids:
            s, t = self.pop_seq_update_batch(rid, free_block_table_fn)
            if s is not None:
                seqs.append(s)
                tables.append(t)
        return seqs, tables

    def pop_n_seqs(self, n: int, free_block_table_fn: Callable = None):
        ids = list(self._sequences_dict.keys())[-n:]
        return self.pop_seqs(ids, free_block_table_fn)

    def pop_finished(self, free_block_table_fn: Callable = None) -> List[Sequence]:
        done = [s.request_id for s in self._sequences_dict.values() if s.check_finish()]
        return self.pop_seqs(done, free_block_table_fn)[0]

    def append_batch_tokens(self, tokens: torch.Tensor) -> None:
        """tokens: [bsz] or [bsz, n]"""
        bsz = self._current_batch_size
        assert bsz == tokens.size(0)
        toks = tokens.tolist()
        for sid, idx in self._sequences_indexes.items():
            t = toks[idx]
            self._sequences_dict[sid].output_token_id += t if isinstance(t, list) else [t]
        self._sequence_lengths[:bsz] += 1 if tokens.dim() == 1 else tokens.size(1)

    def revoke_batch_tokens(self, n_tokens: int, n_seqs: int = 1) -> None:
        if n_tokens >= 1:
            for seq in list(self._sequences_dict.values())[:n_seqs]:
                seq.output_token_id = seq.output_token_id[:-n_tokens]
                seq.revoke_finished_status()
            self._sequence_lengths[:n_seqs] -= n_tokens

    def clear(self, free_block_tables_fn: Optional[Callable[[torch.Tensor], None]] = None) -> List[int]:
        ids = list(self._sequences_dict.keys())
        if free_block_tables_fn:
            free_block_tables_fn(self._block_tables, self._current_batch_size)
        self._block_tables.fill_(-1)
        self._sequence_lengths.fill_(0)
        self._sequences_dict.clear()
        self._sequences_indexes.clear()
        self._current_batch_size = 0
        return ids

    def merge(self, other: "BatchBucket", request_ids: Optional[List[int]] = None) -> List[int]:
        """Move as many sequences of `other` (only those in `request_ids` when given) as fit into this bucket (block
        tables travel with them)."""
        unmerged = []
        ids = other.seqs_ids if request_ids is None else list(request_ids)
        n = min(self.available_batch_size, len(ids))
        for rid in ids[:n]:
            seq, table = other.pop_seq_update_batch(rid)
            self.add_seq(seq, alloc_block_table=table)
        for rid in ids[n:]:
            unmerged.append(rid)
        return unmerged

    # ------------------------------------------------------------------ model inputs
    def get_1D_inputs(self) -> torch.Tensor:
        """Prefill: all prompt tokens, un-padded and concatenated.  Decode: last token of every sequence."""
        first = next(iter(self._sequences_dict.values()))
        if first.output_len == 0 and all(s.output_len == 0 for s in self._sequences_dict.values()):
            out = []
            for s in self._sequences_dict.values():
                out.extend(s.input_token_id[s.num_cached_tokens:])       # prefix-cache hits are not recomputed
            return torch.tensor(out, dtype=torch.long, device=self.device)
        if self._use_spec_dec and self._num_tokens_to_verify:
            out = []
            for s in self._sequences_dict.values():
                out.extend((s.input_token_id + s.output_token_id)[-(self._num_tokens_to_verify + 1):])
            return torch.tensor(out, dtype=torch.long, device=self.device)
        return torch.tensor([(s.output_token_id or s.input_token_id)[-1] for s in self._sequences_dict.values()],
                            dtype=torch.long, device=self.device)

    get_1D_inputs_spec_dec = get_1D_inputs

    def block_table_of(self, request_id: int) -> torch.Tensor:
        """The block-table row of a sequence in this bucket (a view)."""
        return self._block_tables[self._sequences_indexes[request_id]]

    def get_num_cached_tokens(self) -> List[int]:
        """Prompt tokens of every sequence (in batch order) whose K/V the prefix cache already holds."""
        return [s.num_cached_tokens for s in self._sequences_dict.values()]

    def get_block_table_tensor(self) -> torch.Tensor:
        return self._block_tables[: self._current_batch_size].to(self.device)

    def get_sequence_lengths(self) -> torch.Tensor:
        return self._sequence_lengths[: self._current_batch_size].to(self.device)

    def streamingllm_update_batch(self, start_token_size: int, generated_token_size: int) -> List[int]:
        """Drop the oldest non-sink block of sequences whose generated window is full; returns freed block ids."""
        freed = []
        window = start_token_size + generated_token_size
        for sid, idx in self._sequences_indexes.items():
            if int(self._sequence_lengths[idx]) >= window + self.block_size:
                n_blocks = int((self._block_tables[idx] >= 0).sum())
                bid = int(self._block_tables[idx][1])
                freed.append(bid)
                self._block_tables[idx][1:n_blocks - 1] = self._block_tables[idx][2:n_blocks].clone()
                self._block_tables[idx][n_blocks - 1] = -1
                self._sequence_lengths[idx] -= self.block_size
        return freed

    def __repr__(self) -> str:
        return f"BatchBucket(size={self._current_batch_size}, seqs={self.seqs_ids})"
