"""Python face of the paged-KV inference kernels (kernel/csrc/inference.cu) with PyTorch reference paths.
Parity: reference `inference_ops_cuda` bindings used by `inference/modeling/backends/*.py`.

KV-cache format: a floating-point cache holds the K/V values as they are; a `torch.uint8` cache is the fp8 cache and
holds fp8 e5m2 bytes (round to nearest even on write; every e5m2 value decodes exactly to fp16, bf16 and fp32).  This
module is the only one that interprets those bytes: the runtime, engine and drafters write and read the cache through
`kv_cache_write`, `paged_decode_attention` and `gather_paged_kv`."""
from __future__ import annotations

import ctypes
import functools
import math
from typing import Optional, Tuple

import torch

from ..kernel import loader
from ._dispatch import use_native
from ._dtypes import code

_lib = None


def _get_lib():
    global _lib
    if _lib is None:
        _lib = loader.load("cb200_infer")
    return _lib


FP8_CACHE_DTYPE = torch.uint8          # storage dtype of an fp8 (e5m2) KV cache


def _cache_code(cache: torch.Tensor) -> int:
    return code(torch.float8_e5m2 if cache.dtype == FP8_CACHE_DTYPE else cache.dtype)


def _encode(x: torch.Tensor, cache_dtype: torch.dtype) -> torch.Tensor:
    """Values -> what a cache of `cache_dtype` stores."""
    if cache_dtype == FP8_CACHE_DTYPE:
        return x.to(torch.float8_e5m2).view(FP8_CACHE_DTYPE)
    return x.to(cache_dtype)


def _decode(stored: torch.Tensor, dtype: Optional[torch.dtype]) -> torch.Tensor:
    """What a cache stores -> values of `dtype` (None: the stored values' own dtype, torch.float8_e5m2 for fp8)."""
    if stored.dtype == FP8_CACHE_DTYPE:
        stored = stored.view(torch.float8_e5m2)
    return stored if dtype is None else stored.to(dtype)


def kv_cache_write(k: torch.Tensor, v: torch.Tensor, k_cache: torch.Tensor, v_cache: torch.Tensor,
                   block_tables: torch.Tensor, token_seq: torch.Tensor, token_pos: torch.Tensor) -> None:
    """k, v: [tokens, Hkv, D] -> caches [nb, bs, Hkv, D] at (block_tables[seq][pos // bs], pos % bs).  A uint8 cache
    stores the values rounded to fp8 e5m2."""
    tokens, Hkv, D = k.shape
    bs = k_cache.shape[1]
    if (use_native(k) and k.dtype in (torch.float16, torch.bfloat16)
            and k_cache.dtype in (k.dtype, FP8_CACHE_DTYPE)):
        lib = _get_lib()
        loader.check(lib.cb_kv_cache_write(loader.ptr(k), loader.ptr(v), loader.ptr(k_cache), loader.ptr(v_cache),
                                           loader.ptr(block_tables), loader.ptr(token_seq), loader.ptr(token_pos),
                                           tokens, Hkv, D, bs, block_tables.shape[1], ctypes.c_int64(k.stride(0)),
                                           ctypes.c_int64(v.stride(0)), code(k.dtype), _cache_code(k_cache),
                                           loader.stream_ptr()),
                     "kv_cache_write")
        loader.launch_counter.add("kv_cache_write")
        return
    blk = block_tables[token_seq.long(), (token_pos // bs).long()].long()
    slot = (token_pos % bs).long()
    k_cache[blk, slot] = _encode(k, k_cache.dtype)
    v_cache[blk, slot] = _encode(v, v_cache.dtype)


def gather_paged_kv(cache: torch.Tensor, block_table: torch.Tensor, length: int,
                    dtype: Optional[torch.dtype] = None) -> torch.Tensor:
    """One sequence's cached K or V: `cache` [blocks, block_size, Hkv, D] + its block table -> dense [length, Hkv, D]
    values, as `dtype` (None: the cache's value dtype; torch.float8_e5m2 for an fp8 cache)."""
    bs = cache.shape[1]
    nblk = (length + bs - 1) // bs
    return _decode(cache[block_table[:nblk].long()].reshape(-1, cache.shape[2], cache.shape[3])[:length], dtype)


@functools.lru_cache(maxsize=None)
def sm_count(device_index: int) -> int:
    """Streaming multiprocessors of CUDA device `device_index`."""
    return torch.cuda.get_device_properties(device_index).multi_processor_count


def decode_splits(num_seqs: int, kv_heads: int, max_len: int, num_sms: int) -> Tuple[int, int]:
    """Split-KV partition of a paged-attention call over `num_seqs` sequences whose block tables span `max_len`
    positions: (splits, part_len).  A CTA serves up to 8 kv heads of one sequence and split; the splits aim at two
    waves of CTAs on `num_sms` SMs, with partitions of at least 64 tokens rounded up to a multiple of 32.  The kernel's
    partials take [rows, Hq, splits, D] and [rows, Hq, splits, 2] fp32, rows = num_seqs * q_len."""
    ctas_per_split = num_seqs * ((kv_heads + 7) // 8)
    splits = (2 * num_sms + ctas_per_split - 1) // ctas_per_split
    splits = max(1, min(splits, (max_len + 63) // 64))
    part = (max_len + splits - 1) // splits
    part = (part + 31) // 32 * 32
    return max(1, (max_len + part - 1) // part), part


def _split_kv_workspace(q: torch.Tensor, rows: int, heads: int, splits: int, head_dim: int):
    """The split-KV partials (o_part, ml_part) of one call: views of the engine's persistent buffers
    (`inference.flash_decoding_utils.FDIntermTensors`) when they are set up on q's device and large enough, else
    fresh tensors."""
    from ..inference.flash_decoding_utils import FDIntermTensors

    fd = FDIntermTensors()
    if fd.is_initialized and fd.mid_output.device == q.device and fd.mid_output.dtype == torch.float32:
        ws = fd.views(rows, heads, splits, head_dim)
        if ws is not None:
            return ws
    return (torch.empty(rows, heads, splits, head_dim, dtype=torch.float32, device=q.device),
            torch.empty(rows, heads, splits, 2, dtype=torch.float32, device=q.device))


def paged_decode_attention(q: torch.Tensor, k_cache: torch.Tensor, v_cache: torch.Tensor, block_tables: torch.Tensor,
                           seq_lens: torch.Tensor, scale: Optional[float] = None,
                           alibi_slopes: Optional[torch.Tensor] = None, window: Optional[int] = None,
                           q_len: int = 1) -> torch.Tensor:
    """q: [num_seqs * q_len, Hq, D] -> same shape.  `seq_lens` [num_seqs] counts the cached tokens including the
    step's; sequence i's queries are rows i * q_len + j (token-major), and query j sits at position
    seq_lens[i] - q_len + j and sees the positions up to its own.  q_len = 1 is a decode step, q_len > 1 the
    speculative verification of q_len - 1 drafted tokens (one pass over the cache).  `window`: sliding-window attention
    (only the last `window` positions a query sees are visible), handled inside the split-KV kernel (`window_start`).
    An fp8 (uint8) cache is decoded exactly to the query dtype inside the kernel."""
    rows, Hq, D = q.shape
    nb, bs, Hkv, _ = k_cache.shape
    assert q_len >= 1 and rows % q_len == 0, (rows, q_len)
    n = rows // q_len
    scale = scale if scale is not None else 1.0 / math.sqrt(D)
    native = (use_native(q) and q.dtype in (torch.float16, torch.bfloat16)
              and k_cache.dtype in (q.dtype, FP8_CACHE_DTYPE) and D in (64, 128, 256) and Hq // Hkv <= 8)
    if native and q_len <= (1 if D == 256 else 16):
        splits, part = decode_splits(n, Hkv, block_tables.shape[1] * bs, sm_count(q.device.index))
        out = torch.empty_like(q)
        o_part, ml_part = _split_kv_workspace(q, rows, Hq, splits, D)
        qc = q if q.stride(2) == 1 and q.stride(1) == D else q.contiguous()
        loader.check(_get_lib().cb_paged_decode_attention(
            loader.ptr(qc), loader.ptr(k_cache), loader.ptr(v_cache), loader.ptr(block_tables), loader.ptr(seq_lens),
            loader.ptr(out), loader.ptr(o_part), loader.ptr(ml_part), n, q_len, Hq, Hkv, D, bs, block_tables.shape[1],
            splits, part, ctypes.c_float(scale), loader.ptr(alibi_slopes), ctypes.c_int64(qc.stride(0)),
            ctypes.c_int64(out.stride(0)), code(q.dtype), _cache_code(k_cache), int(window or 0), loader.stream_ptr()),
            "paged_decode_attention")
        loader.launch_counter.add("paged_decode_attention", 2)
        return out
    if native:          # q_len > 1 beyond the one-pass kernel (head_dim 256, or q_len > 16): one decode call per query
        qs = q.view(n, q_len, Hq, D)
        outs = [paged_decode_attention(qs[:, j], k_cache, v_cache, block_tables, seq_lens - (q_len - 1 - j), scale,
                                       alibi_slopes, window) for j in range(q_len)]
        return torch.stack(outs, 1).view(rows, Hq, D)
    return paged_decode_attention_ref(q, k_cache, v_cache, block_tables, seq_lens, scale, alibi_slopes, window, q_len)


def paged_decode_attention_ref(q, k_cache, v_cache, block_tables, seq_lens, scale=None, alibi_slopes=None,
                               window=None, q_len=1):
    rows, Hq, D = q.shape
    nb, bs, Hkv, _ = k_cache.shape
    scale = scale if scale is not None else 1.0 / math.sqrt(D)
    G = Hq // Hkv
    out = torch.empty_like(q)
    for i in range(rows):
        s_i = i // q_len                              # sequence of row i; its query sees L positions
        L = int(seq_lens[s_i]) - (q_len - 1 - i % q_len)
        k = gather_paged_kv(k_cache, block_tables[s_i], L, torch.float32)
        v = gather_paged_kv(v_cache, block_tables[s_i], L, torch.float32)
        if window is not None and L > window:
            k, v, L = k[L - window:], v[L - window:], window
        k = k.repeat_interleave(G, dim=1)
        v = v.repeat_interleave(G, dim=1)
        s = torch.einsum("hd,lhd->hl", q[i].float(), k) * scale
        if alibi_slopes is not None:
            s = s + alibi_slopes.float()[:, None] * (torch.arange(L, device=q.device) - (L - 1))[None, :]
        p = s.softmax(-1)
        out[i] = torch.einsum("hl,lhd->hd", p, v).to(q.dtype)
    return out


def paged_prefill_attention(q: torch.Tensor, k_cache: torch.Tensor, v_cache: torch.Tensor, block_tables: torch.Tensor,
                            cu_seqlens_q: torch.Tensor, seq_lens: torch.Tensor, scale: Optional[float] = None,
                            alibi_slopes: Optional[torch.Tensor] = None, window: Optional[int] = None) -> torch.Tensor:
    """Causal prefill whose keys live in the paged cache: q [T, Hq, D] packs n_b = cu_seqlens_q[b+1] - cu_seqlens_q[b]
    new rows per sequence; sequence b holds `seq_lens[b]` tokens (cached + new) and its new rows sit at positions
    seq_lens[b] - n_b .. seq_lens[b] - 1, each attending to every cached position up to its own (the step's K/V must
    already be written).  `window`: only the last `window` positions a query sees are visible.  fp16 / bf16 queries
    over a cache of the same dtype at head_dim 64 / 128 run the paged wgmma flash kernel with no host sync; everything
    else (CPU, fp32, an fp8 cache, other head sizes) takes `paged_prefill_attention_ref`."""
    D = q.shape[-1]
    if (use_native(q) and q.dtype in (torch.float16, torch.bfloat16) and k_cache.dtype == q.dtype
            and v_cache.dtype == q.dtype and D in (64, 128) and q.shape[1] % k_cache.shape[2] == 0):
        from . import flash_attn_native as fan

        return fan.flash_prefill_paged(q.contiguous(), k_cache, v_cache, block_tables, cu_seqlens_q, seq_lens, scale,
                                       window=window or 0, alibi_slopes=alibi_slopes)
    return paged_prefill_attention_ref(q, k_cache, v_cache, block_tables, cu_seqlens_q, seq_lens, scale,
                                       alibi_slopes, window)


def paged_prefill_attention_ref(q, k_cache, v_cache, block_tables, cu_seqlens_q, seq_lens, scale=None,
                                alibi_slopes=None, window=None):
    """One sequence at a time: the sequence's K/V gathered from the cache (`gather_paged_kv`, fp8 decoded exactly),
    then an fp32 masked softmax (float64 for float64 queries)."""
    T, Hq, D = q.shape
    Hkv = k_cache.shape[2]
    scale = scale if scale is not None else 1.0 / math.sqrt(D)
    G = Hq // Hkv
    cdt = torch.float64 if q.dtype == torch.float64 else torch.float32
    out = torch.empty_like(q)
    cu = cu_seqlens_q.tolist()
    lens = seq_lens.tolist()
    for b in range(len(cu) - 1):
        a, e, L = cu[b], cu[b + 1], lens[b]
        if e == a:
            continue
        k = gather_paged_kv(k_cache, block_tables[b], L, cdt).repeat_interleave(G, dim=1)
        v = gather_paged_kv(v_cache, block_tables[b], L, cdt).repeat_interleave(G, dim=1)
        q_pos = torch.arange(L - (e - a), L, device=q.device)
        rel = torch.arange(L, device=q.device)[None, :] - q_pos[:, None]           # key - query
        keep = rel <= 0
        if window is not None and window > 0:
            keep = keep & (rel > -window)
        s = torch.einsum("qhd,khd->hqk", q[a:e].to(cdt), k) * scale
        if alibi_slopes is not None:
            s = s + alibi_slopes.to(device=q.device, dtype=cdt)[:, None, None] * rel.to(cdt)[None]
        s = s.masked_fill(~keep[None], float("-inf"))
        out[a:e] = torch.einsum("hqk,khd->qhd", s.softmax(-1), v).to(q.dtype)
    return out


def convert_fp8(x: torch.Tensor, to_fp8: bool, out_dtype: torch.dtype = torch.bfloat16) -> torch.Tensor:
    """KV-cache fp8 (e5m2) storage conversion."""
    if to_fp8:
        if use_native(x):
            out = torch.empty(x.shape, dtype=torch.uint8, device=x.device)
            loader.check(_get_lib().cb_convert_fp8(loader.ptr(x.contiguous()), loader.ptr(out),
                                                   ctypes.c_int64(x.numel()), code(x.dtype), 0, loader.stream_ptr()),
                         "convert_fp8")
            loader.launch_counter.add("convert_fp8")
            return out
        return _encode(x, FP8_CACHE_DTYPE)
    if use_native(x):
        out = torch.empty(x.shape, dtype=out_dtype, device=x.device)
        loader.check(_get_lib().cb_convert_fp8(loader.ptr(x.contiguous()), loader.ptr(out), ctypes.c_int64(x.numel()),
                                               code(out_dtype), 1, loader.stream_ptr()), "convert_fp8")
        loader.launch_counter.add("convert_fp8")
        return out
    return _decode(x, out_dtype)
