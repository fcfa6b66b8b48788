"""Paged KV cache manager.

Parity: reference `colossalai/inference/kv_cache/kvcache_manager.py:18-604`: per-layer K / V tensors of fixed-size
blocks, free-list allocation for a whole prompt / one decode token / n speculative tokens, block-table maintenance,
StreamingLLM window eviction, a logical-only RPC variant.
Layout (H100-first, see kernel/csrc/inference.cu): K and V are both `[num_blocks, block_size, kv_heads, head_dim]`.

Prefix caching (`InferenceConfig.enable_prefix_caching`, no reference equivalent): full blocks whose K/V are written
are indexed under (serial id of the parent entry, the block's token ids); serial ids are never reused, so an entry
whose parent was evicted can never match again, even when the parent's block now holds other tokens.  A prompt takes
references to the longest indexed chain that matches it (at most (L - 1) // block_size blocks: its last token is always
computed).  Indexed blocks nobody references are *cached-free*: they count as available and are evicted least recently
freed first, only when no never-indexed free block is left.
"""
from __future__ import annotations

from collections import OrderedDict
from typing import Dict, List, Optional, Sequence, Tuple

import torch

from ...accelerator import get_accelerator
from ...logging import get_dist_logger
from .block_cache import CacheBlock

__all__ = ["KVCacheManager", "RPCKVCacheManager"]

GIGABYTE = 1024**3


class KVCacheManager:
    def __init__(self, config, model_config, verbose: bool = False) -> None:
        """`config`: InferenceConfig; `model_config`: our ModelConfig (or anything exposing the same fields)."""
        self.logger = get_dist_logger(__name__)
        self.device = get_accelerator().get_current_device()
        self.tp_size = config.tp_size
        self.num_layers = model_config.num_hidden_layers
        self.head_num = model_config.num_attention_heads // self.tp_size
        self.head_size = model_config.head_dim
        kv = getattr(model_config, "num_key_value_heads", model_config.num_attention_heads)
        assert kv % self.tp_size == 0 or self.tp_size % kv == 0
        self.kv_head_num = max(kv // self.tp_size, 1)
        self.dtype = config.dtype
        self.kv_cache_dtype = torch.uint8 if config.kv_cache_dtype == "fp8" else config.dtype
        self.elem_size_in_bytes = torch.tensor([], dtype=self.kv_cache_dtype).element_size()
        self.max_batch_size = config.max_batch_size
        self.max_input_length, self.max_output_length = config.max_input_len, config.max_output_len
        self.beam_width = config.beam_width
        self.block_size = config.block_size
        self.enable_streamingllm = config.enable_streamingllm
        self.start_token_size, self.generated_token_size = config.start_token_size, config.generated_token_size
        self.max_blocks_per_sequence = (self.max_input_length + self.max_output_length + self.block_size - 1) \
            // self.block_size
        self.num_blocks = self.max_blocks_per_sequence * self.max_batch_size * self.beam_width
        self._kv_caches = self._init_device_caches()
        self._cache_blocks: Tuple[CacheBlock, ...] = self._init_logical_caches()
        self._available_blocks = self.num_blocks
        self._block_states = torch.ones(self.num_blocks, dtype=torch.bool)
        self._block_states_cum = torch.zeros(self.num_blocks + 1, dtype=torch.int64)
        self._block_finder = torch.zeros(self.num_blocks, dtype=torch.int64)
        self.enable_prefix_caching = getattr(config, "enable_prefix_caching", False)
        self._prefix_index: Dict[Tuple[int, Tuple[int, ...]], Tuple[int, int]] = {}   # key -> (block id, serial)
        self._block_entry: Dict[int, Tuple[Tuple[int, Tuple[int, ...]], int]] = {}    # block id -> (key, serial)
        self._cached_free: "OrderedDict[int, None]" = OrderedDict()                    # LRU order, oldest first
        self._next_serial = 1                                                          # 0 = the root
        self._queried_tokens = 0
        self._hit_tokens = 0
        if verbose:
            tot = self.total_physical_cache_size_in_bytes / GIGABYTE
            self.logger.info(f"KV cache: {self.num_blocks} blocks x {self.block_size} tokens, {tot:.2f} GB", ranks=[0])

    @property
    def total_num_blocks(self) -> int:
        return self.num_blocks

    @property
    def num_available_blocks(self) -> int:
        return self._available_blocks

    @property
    def prefix_cache_stats(self) -> Dict[str, int]:
        """Prompt tokens looked up in the prefix index and tokens served from it since construction."""
        return {"queried_tokens": self._queried_tokens, "hit_tokens": self._hit_tokens}

    @property
    def total_physical_cache_size_in_bytes(self) -> int:
        return (2 * self.num_layers * self.num_blocks * self.block_size * self.kv_head_num * self.head_size
                * self.elem_size_in_bytes)

    def get_head_size(self) -> int:
        return self.head_size

    def get_kv_cache(self):
        return self._kv_caches

    def get_max_blocks_per_sequence(self) -> int:
        return self.max_blocks_per_sequence

    def check_allocation(self, seq) -> bool:
        need = (seq.input_len + self.max_output_length + self.block_size - 1) // self.block_size
        return need <= self.num_available_blocks

    def get_block_kv_ptrs(self, block_id: int, layer_id: int) -> Tuple[int, int]:
        k, v = self._kv_caches[0][layer_id], self._kv_caches[1][layer_id]
        off = block_id * k.stride(0) * k.element_size()
        return k.data_ptr() + off, v.data_ptr() + off

    # ------------------------------------------------------------------ allocation
    def _take_free_blocks(self, n: int) -> List[int]:
        """`n` blocks for new content: never-indexed free blocks first (lowest ids), then cached-free blocks evicted
        least recently freed first.  The caller checked that `n` blocks are available."""
        free = torch.nonzero(self._block_states, as_tuple=False).flatten()[:n].tolist()
        for bid in free:
            self._block_states[bid] = False
        while len(free) < n:
            bid, _ = self._cached_free.popitem(last=False)
            key, _ = self._block_entry.pop(bid)
            del self._prefix_index[key]
            free.append(bid)
        self._available_blocks -= n
        return free

    def allocate_context_from_block_table(self, block_table: torch.Tensor, context_len: int) -> None:
        """Allocate the blocks of one prompt; `block_table` is the sequence's 1-D int32 row (-1 = unassigned)."""
        assert block_table.dim() == 1
        if not torch.all(block_table < 0):
            self.logger.error("Some slots on provided block table have been allocated.")
        need = (context_len + self.block_size - 1) // self.block_size
        if need > self._available_blocks:
            raise RuntimeError(f"No enough blocks to allocate. Available {self._available_blocks}; need {need}.")
        free = self._take_free_blocks(need)
        block_table[:need] = torch.tensor(free, dtype=block_table.dtype).to(block_table.device)
        for i, bid in enumerate(free):
            blk = self._cache_blocks[bid]
            blk.add_ref()
            blk.allocate(self.block_size if i < need - 1 else context_len - (need - 1) * self.block_size)

    def match_prefix(self, token_ids: Sequence[int]) -> List[int]:
        """Block ids of the longest indexed chain equal to the prompt's leading full blocks, capped at
        (len - 1) // block_size blocks so that at least one prompt token is computed."""
        bs = self.block_size
        parent, hits = 0, []
        for i in range((len(token_ids) - 1) // bs):
            entry = self._prefix_index.get((parent, tuple(token_ids[i * bs:(i + 1) * bs])))
            if entry is None:
                break
            hits.append(entry[0])
            parent = entry[1]
        return hits

    def allocate_context_with_prefix(self, block_table: torch.Tensor, token_ids: Sequence[int]) -> int:
        """Allocate one prompt's blocks, sharing the matched prefix chain (`match_prefix`): references are added to
        the matched blocks (a cached-free block goes from 0 to 1 reference), the rest are fresh.  Returns the number of
        prompt tokens whose K/V are cached (a whole number of blocks)."""
        assert block_table.dim() == 1
        bs, L = self.block_size, len(token_ids)
        hits = self.match_prefix(token_ids)
        need = (L + bs - 1) // bs
        revived = sum(1 for bid in hits if not self._cache_blocks[bid].has_ref())
        if need - len(hits) > self._available_blocks - revived:
            raise RuntimeError(f"No enough blocks to allocate. Available {self._available_blocks}; need {need}.")
        for bid in hits:
            blk = self._cache_blocks[bid]
            if not blk.has_ref():
                del self._cached_free[bid]
                self._available_blocks -= 1
                blk.allocate()
            blk.add_ref()
        fresh = self._take_free_blocks(need - len(hits))
        for i, bid in enumerate(fresh):
            blk = self._cache_blocks[bid]
            blk.add_ref()
            pos = (len(hits) + i) * bs
            blk.allocate(min(bs, L - pos))
        block_table[:need] = torch.tensor(hits + fresh, dtype=block_table.dtype).to(block_table.device)
        self._queried_tokens += L
        self._hit_tokens += len(hits) * bs
        return len(hits) * bs

    def register_prefix_blocks(self, block_table: torch.Tensor, token_ids: Sequence[int], num_written: int) -> None:
        """Index the sequence's full blocks whose positions are all `< num_written` (K/V written).  A block whose key
        is already indexed (the same prefix computed by another sequence) stays out of the index; the chain goes on
        from the indexed entry."""
        if not self.enable_prefix_caching:
            return
        bs = self.block_size
        n_full = min(num_written, len(token_ids)) // bs
        table = block_table[:n_full].tolist()
        parent = 0
        for i in range(n_full):
            bid = table[i]
            if bid < 0:
                break
            key = (parent, tuple(token_ids[i * bs:(i + 1) * bs]))
            entry = self._prefix_index.get(key)
            if entry is None:
                if bid in self._block_entry:          # indexed under another chain: the two chains diverge here
                    break
                entry = (bid, self._next_serial)
                self._next_serial += 1
                self._prefix_index[key] = entry
                self._block_entry[bid] = (key, entry[1])
            parent = entry[1]

    def allocate_context_from_block_tables(self, block_tables: torch.Tensor, context_lengths: torch.Tensor) -> None:
        assert block_tables.dim() == 2 and block_tables.size(0) == context_lengths.size(0)
        for i in range(block_tables.size(0)):
            self.allocate_context_from_block_table(block_tables[i], int(context_lengths[i]))

    def allocate_token_from_block_table(self, block_table: torch.Tensor, context_len: int) -> None:
        """Make room for the token at position `context_len - 1` (allocates a new block when crossing a boundary)."""
        assert block_table.dim() == 1
        local = (context_len - 1) // self.block_size
        if local >= block_table.numel():
            raise RuntimeError("sequence exceeds max_blocks_per_sequence")
        bid = int(block_table[local])
        if bid < 0:
            if self._available_blocks < 1:
                raise RuntimeError("No available blocks to allocate.")
            bid = self._take_free_blocks(1)[0]
            self._cache_blocks[bid].add_ref()
            block_table[local] = bid
        self._cache_blocks[bid].allocate(1) if self._cache_blocks[bid].available_space > 0 else None

    def allocate_tokens_from_block_tables(self, block_tables: torch.Tensor, context_lens: torch.Tensor,
                                          bsz: Optional[int] = None) -> List[int]:
        bsz = block_tables.size(0) if bsz is None else bsz
        for i in range(bsz):
            self.allocate_token_from_block_table(block_tables[i], int(context_lens[i]))
        return []

    def allocate_n_tokens_from_block_tables(self, block_tables: torch.Tensor, context_lens: torch.Tensor,
                                            bsz: int, n: int) -> None:
        """Speculative decoding: reserve room for `n` more tokens per sequence."""
        for i in range(bsz):
            for j in range(n):
                self.allocate_token_from_block_table(block_tables[i], int(context_lens[i]) + j + 1)

    def allocate_single_block(self, block_table: torch.Tensor, block_local_idx: int) -> int:
        bid = int(block_table[block_local_idx])
        if bid < 0:
            if self._available_blocks < 1:
                raise RuntimeError("No available blocks to allocate.")
            bid = self._take_free_blocks(1)[0]
            self._cache_blocks[bid].add_ref()
            block_table[block_local_idx] = bid
        return bid

    # ------------------------------------------------------------------ free
    def free_block_table(self, block_table: torch.Tensor) -> None:
        assert block_table.dim() == 1
        for i in range(block_table.numel()):
            bid = int(block_table[i])
            if bid < 0:
                continue
            blk = self._cache_blocks[bid]
            blk.remove_ref()
            if not blk.has_ref():
                blk.clear()
                self._available_blocks += 1
                if bid in self._block_entry:
                    self._cached_free[bid] = None         # keeps its K/V and index entry until evicted
                else:
                    self._block_states[bid] = True
            block_table[i] = -1

    def free_block_tables(self, block_tables: torch.Tensor, first_n: Optional[int] = None) -> None:
        n = block_tables.size(0) if first_n is None else first_n
        for i in range(n):
            self.free_block_table(block_tables[i])

    def clear_all(self) -> None:
        for b in self._cache_blocks:
            b.clear()
        self._available_blocks = self.num_blocks
        self._block_states[:] = True
        self._prefix_index.clear()
        self._block_entry.clear()
        self._cached_free.clear()

    def streamingllm_free_block_tables(self, updated_block_ids: List[int]) -> None:
        """Free blocks pushed out of the attention window (StreamingLLM)."""
        for bid in updated_block_ids:
            blk = self._cache_blocks[bid]
            blk.remove_ref()
            if not blk.has_ref():
                blk.clear()
                self._available_blocks += 1
                self._block_states[bid] = True

    # ------------------------------------------------------------------ init
    def _init_logical_caches(self) -> Tuple[CacheBlock, ...]:
        return tuple(CacheBlock(i, self.block_size, self.elem_size_in_bytes) for i in range(self.num_blocks))

    def _init_device_caches(self):
        shape = (self.num_blocks, self.block_size, self.kv_head_num, self.head_size)
        k = [torch.zeros(shape, dtype=self.kv_cache_dtype, device=self.device) for _ in range(self.num_layers)]
        v = [torch.zeros(shape, dtype=self.kv_cache_dtype, device=self.device) for _ in range(self.num_layers)]
        return k, v


class RPCKVCacheManager(KVCacheManager):
    """Driver-side manager of the RPC engine: logical blocks only (workers own the physical cache)."""

    def __init__(self, config, model_config, verbose: bool = False) -> None:
        self._no_physical = True
        super().__init__(config, model_config, verbose)

    def _init_device_caches(self):
        return None, None

    def get_physical_cache_shape(self) -> Tuple[int, ...]:
        return (self.num_blocks, self.block_size, self.kv_head_num, self.head_size)
