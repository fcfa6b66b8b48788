"""Paged KV cache manager.

Parity: reference `colossalai/inference/kv_cache/kvcache_manager.py:18-604`: per-layer K / V tensors of fixed-size
blocks, free-list allocation for a whole prompt / one decode token / n speculative tokens, block-table maintenance,
StreamingLLM window eviction, a logical-only RPC variant.
Layout (H100-first, see kernel/csrc/inference.cu): K and V are both `[num_blocks, block_size, kv_heads, head_dim]`.
"""
from __future__ import annotations

from typing import List, Optional, Tuple

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
    def allocate_context_from_block_table(self, block_table: torch.Tensor, context_len: int) -> None:
        """Allocate the blocks of one prompt; `block_table` is the sequence's 1-D int32 row (-1 = unassigned)."""
        assert block_table.dim() == 1
        if not torch.all(block_table < 0):
            self.logger.error("Some slots on provided block table have been allocated.")
        need = (context_len + self.block_size - 1) // self.block_size
        if need > self._available_blocks:
            raise RuntimeError(f"No enough blocks to allocate. Available {self._available_blocks}; need {need}.")
        free = torch.nonzero(self._block_states, as_tuple=False).flatten()[:need]
        block_table[:need] = free.to(block_table.dtype).to(block_table.device)
        for i, bid in enumerate(free.tolist()):
            blk = self._cache_blocks[bid]
            blk.add_ref()
            blk.allocate(self.block_size if i < need - 1 else context_len - (need - 1) * self.block_size)
            self._block_states[bid] = False
            self._available_blocks -= 1

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
            bid = int(torch.nonzero(self._block_states, as_tuple=False)[0])
            self._block_states[bid] = False
            self._available_blocks -= 1
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
            bid = int(torch.nonzero(self._block_states, as_tuple=False)[0])
            self._block_states[bid] = False
            self._available_blocks -= 1
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
