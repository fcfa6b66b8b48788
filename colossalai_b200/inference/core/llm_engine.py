"""LLM inference engine: continuous batching over a paged KV cache, CUDA-graph decode, speculative decoding.

Parity: reference `colossalai/inference/core/llm_engine.py:46-758` (`init_model`, `capture_model`, `generate`,
`add_request`, `step`, `prepare_input`, `enable_spec_dec` / `steps_spec_dec`).
"""
from __future__ import annotations

import time
from itertools import accumulate, count
from typing import Dict, List, Optional, Tuple, Union

import numpy as np
import torch
import torch.distributed as dist
import torch.nn as nn

from ...accelerator import get_accelerator
from ...cluster import DeviceMesh
from ...logging import get_dist_logger
from ...models import build_model
from ...models.config import ModelConfig
from ..batch_bucket import BatchBucket
from ..config import GenerationConfig, InferenceConfig, InputMetaData, ModelShardInferenceConfig
from ..graph_runner import CUDAGraphRunner
from ..modeling import PagedKVRuntime
from ..sampler import search_tokens
from ..spec import Drafter, GlideInput
from ..struct import Sequence
from .base_engine import BaseEngine
from .request_handler import RequestHandler

__all__ = ["LLMEngine"]

PP_AXIS, TP_AXIS = 0, 1
_BATCH_SIZES_TO_CAPTURE = [1, 2, 4] + [8 * i for i in range(1, 33)]


class _SimpleTokenizer:
    """Whitespace-free fallback tokenizer (ids = bytes) so the engine is usable without a HF tokenizer."""

    eos_token_id = 2
    pad_token_id = 0

    def __call__(self, texts, padding=False, **kw):
        if isinstance(texts, str):
            texts = [texts]
        return {"input_ids": [[3 + b for b in t.encode("utf-8")] for t in texts]}

    def batch_decode(self, ids, skip_special_tokens=True):
        return [bytes(max(i - 3, 0) % 256 for i in seq if i >= 3).decode("utf-8", errors="replace") for seq in ids]

    def decode(self, ids, skip_special_tokens=True):
        return self.batch_decode([ids])[0]


def prefix_caching_unsupported(inference_config: InferenceConfig, model_config: ModelConfig) -> Optional[str]:
    """Why a CUDA engine cannot serve prefix-cache hits natively (None when it can).  A hit runs the prefill through
    the paged wgmma flash kernel: fp16 / bf16 model and cache, head_dim 64 / 128, no MLA.  Outside that envelope a hit
    would take the per-sequence reference loop on the GPU."""
    if inference_config.kv_cache_dtype is not None:
        return f"the paged prefill kernel reads 16-bit caches, not kv_cache_dtype={inference_config.kv_cache_dtype!r}"
    if inference_config.dtype not in (torch.float16, torch.bfloat16):
        return f"the paged prefill kernel needs fp16 or bf16, not {inference_config.dtype}"
    if getattr(model_config, "use_mla", False):
        return "MLA models are not supported"
    if model_config.head_dim not in (64, 128):
        return f"the paged prefill kernel needs head_dim 64 or 128, not {model_config.head_dim}"
    return None


class LLMEngine(BaseEngine):
    def __init__(self, model_or_path: Union[nn.Module, str, ModelConfig], tokenizer=None,
                 inference_config: Optional[InferenceConfig] = None, verbose: bool = False, model_policy=None) -> None:
        self.inference_config = inference_config or InferenceConfig()
        self.dtype = self.inference_config.dtype
        self.high_precision = self.inference_config.high_precision
        self.verbose = verbose
        self.logger = get_dist_logger(__name__)
        self.model_shard_infer_config = ModelShardInferenceConfig(dtype=self.dtype,
                                                                  use_cuda_kernel=self.inference_config.use_cuda_kernel)
        self.device = get_accelerator().get_current_device()
        self.init_model(model_or_path, model_policy, self.model_shard_infer_config)
        self.tokenizer = tokenizer or _SimpleTokenizer()
        self.generation_config = self.inference_config.to_generation_config(self.model_config)
        self.generation_config_dict = self.generation_config.to_dict()
        self.request_handler = RequestHandler(self.inference_config, self.model_config)
        k_caches, v_caches = self.request_handler.get_kvcache()
        self.kv_runtime = PagedKVRuntime(k_caches, v_caches, self.inference_config.block_size)
        self._init_decode_workspace(k_caches)
        self.counter = count()
        self.use_cuda_graph = self.inference_config.use_cuda_graph and torch.cuda.is_available()
        if self.use_cuda_graph and (self.model_config.head_dim not in (64, 128, 256)
                                    or self.dtype not in (torch.float16, torch.bfloat16)):
            # the decode step must stay on the native paged kernel to be capturable (the reference path syncs)
            self.logger.warning("CUDA graphs disabled: the native paged-decode kernel needs fp16/bf16 and head_dim in "
                                "{64, 128, 256}", ranks=[0])
            self.use_cuda_graph = False
        self.graph_runners: Dict[int, CUDAGraphRunner] = {}
        self.graph_memory_pool = None
        self.use_spec_dec = False
        self.drafter_model = None
        self.drafter = None
        self.use_glide = False
        self.n_spec_tokens = self.inference_config.max_n_spec_tokens
        self._verify_args()
        if self.use_cuda_graph:
            self.capture_model()

    # ------------------------------------------------------------------ model
    def init_model(self, model_or_path, model_policy=None, model_shard_infer_config=None) -> None:
        hf_dir = None
        if isinstance(model_or_path, str):
            import json
            import os

            from ...models.hf_io import config_from_hf, load_hf_checkpoint

            if self.inference_config.tp_size > 1:
                # build the skeleton, shard it, then stream each rank's slices in (InferCheckpoint_io)
                with open(os.path.join(model_or_path, "config.json")) as f:
                    self.model = build_model(config_from_hf(json.load(f)))
                hf_dir = model_or_path
            else:
                self.model = load_hf_checkpoint(model_or_path, dtype=self.dtype)
        elif isinstance(model_or_path, ModelConfig):
            self.model = build_model(model_or_path)
        else:
            self.model = model_or_path
        self.model_config: ModelConfig = self.model.cfg
        self.model = self.model.to(self.dtype).eval()
        tp = self.inference_config.tp_size
        self.tp_group = None
        if tp > 1:
            assert dist.is_initialized() and dist.get_world_size() % tp == 0
            self.pg_mesh = DeviceMesh(pp=dist.get_world_size() // tp, tp=tp)
            self.tp_group = self.pg_mesh.group("tp")
            self.model = self._shardformer(self.model, model_policy, model_shard_infer_config, None, self.tp_group)
            if hf_dir is not None:
                from .plugin import InferCheckpoint_io

                InferCheckpoint_io().load_model(self.model, hf_dir)
        self.model = self.model.to(self.device)

    def _verify_args(self) -> None:
        assert isinstance(self.inference_config, InferenceConfig), "Invalid type of inference config provided."
        assert isinstance(self.model, nn.Module), f"the model type must be nn.Module, but got {type(self.model)}"
        if self.inference_config.enable_prefix_caching and torch.device(self.device).type == "cuda":
            err = prefix_caching_unsupported(self.inference_config, self.model_config)
            if err:
                raise ValueError(f"enable_prefix_caching: {err}")
        if self.inference_config.max_num_batched_tokens is not None and torch.device(self.device).type == "cuda":
            # every chunk runs the paged prefill, as a prefix-cache hit does
            err = prefix_caching_unsupported(self.inference_config, self.model_config)
            if err:
                raise ValueError(f"max_num_batched_tokens: {err}")

    def _init_decode_workspace(self, k_caches, q_per_seq: int = 1) -> None:
        """Size the persistent split-KV buffers of the paged decode kernel for the largest batch (reference
        `flash_decoding_utils.FDIntermTensors.initialize` called from the request handler); `q_per_seq` query tokens
        per sequence (speculative verification) need that many rows of partials per sequence."""
        if not torch.cuda.is_available() or not k_caches or k_caches[0].device.type != "cuda":
            return
        from ...ops import inference as infer_ops
        from ..flash_decoding_utils import FDIntermTensors

        cfg = self.inference_config
        device = k_caches[0].device
        hkv, d = k_caches[0].shape[2], k_caches[0].shape[3]
        hq = hkv * (self.model_config.num_attention_heads // max(self.model_config.num_key_value_heads, 1))
        max_len = cfg.max_input_len + cfg.max_output_len
        max_len = (max_len + cfg.block_size - 1) // cfg.block_size * cfg.block_size
        sms = infer_ops.sm_count(device.index)
        worst = max(n * q_per_seq * infer_ops.decode_splits(n, hkv, max_len, sms)[0]
                    for n in range(1, cfg.max_batch_size + 1))
        FDIntermTensors().ensure(worst, hq, d, device=device)

    def _model_forward(self, input_ids: torch.Tensor, positions: torch.Tensor) -> torch.Tensor:
        """input_ids: flattened tokens [T]; returns hidden->logits of the LAST token of every sequence."""
        from ...models.transformer import SeqMeta

        meta = SeqMeta(batch=1, seqlen=input_ids.numel(), positions=positions,
                       cu_seqlens=self.kv_runtime.cu_seqlens, max_seqlen=self.kv_runtime.max_seqlen)
        out = self.model(input_ids=input_ids.view(1, -1), kv_cache=self.kv_runtime, meta=meta)
        return out["logits"]

    @torch.inference_mode()
    def capture_model(self) -> None:
        """Capture the decode step for a ladder of batch sizes."""
        t0 = time.perf_counter()
        max_bs = self.inference_config.max_batch_size
        max_blocks = self.request_handler.cache_manager.get_max_blocks_per_sequence()
        for bs in reversed([b for b in _BATCH_SIZES_TO_CAPTURE if b <= max_bs]):
            ids = torch.zeros(bs, dtype=torch.long, device=self.device)
            tables = torch.zeros(bs, max_blocks, dtype=torch.int32, device=self.device)
            lens = torch.ones(bs, dtype=torch.int32, device=self.device)

            def fn(input_ids, block_tables, seq_lens, positions, token_seq, token_pos):
                rt = self.kv_runtime
                rt.block_tables, rt.seq_lens, rt.is_prompt, rt.q_per_seq = block_tables, seq_lens, False, 1
                rt.token_seq, rt.token_pos, rt.cu_seqlens = token_seq, token_pos, None
                return self._model_forward(input_ids, positions)

            runner = CUDAGraphRunner(fn)
            runner.capture(memory_pool=self.graph_memory_pool, input_ids=ids, block_tables=tables, seq_lens=lens,
                           positions=torch.zeros(bs, dtype=torch.long, device=self.device),
                           token_seq=torch.arange(bs, dtype=torch.int32, device=self.device),
                           token_pos=torch.zeros(bs, dtype=torch.int32, device=self.device))
            self.graph_memory_pool = runner.graph.pool()
            self.graph_runners[bs] = runner
        if self.verbose:
            self.logger.info(f"CUDA graph capture took {time.perf_counter() - t0:.2f}s", ranks=[0])

    # ------------------------------------------------------------------ speculative decoding
    def enable_spec_dec(self, drafter_model: nn.Module = None, n_spec_tokens: int = None,
                        use_glide_drafter: bool = False) -> None:
        if drafter_model is None and self.drafter is None:
            raise ValueError("Drafter not initialized. Please provide a Drafter Model")
        if n_spec_tokens is not None:
            assert 1 < n_spec_tokens <= self.inference_config.max_n_spec_tokens
            self.n_spec_tokens = n_spec_tokens
        if drafter_model is not None:
            self.drafter_model = drafter_model.to(self.dtype).to(self.device).eval()
            self.drafter = Drafter(self.drafter_model, self.tokenizer, device=self.device, dtype=self.dtype)
        self.use_glide = use_glide_drafter
        self._init_decode_workspace(self.kv_runtime.k_caches, q_per_seq=self.n_spec_tokens + 1)   # verify pass
        self.request_handler.set_spec_dec_mode(self.n_spec_tokens)
        self.use_spec_dec = True

    def disable_spec_dec(self) -> None:
        self.request_handler.unset_spec_dec_mode()
        self.use_spec_dec = False

    def clear_spec_dec(self) -> None:
        if self.use_spec_dec:
            self.disable_spec_dec()
        self.drafter_model = self.drafter = None
        torch.cuda.empty_cache() if torch.cuda.is_available() else None

    @torch.inference_mode()
    def steps_spec_dec(self) -> List[Sequence]:
        """One speculative round: draft n tokens per sequence, verify them with ONE target-model pass, keep the longest
        matching prefix (+1 corrected token), roll back the rest."""
        batch = self.request_handler.schedule()
        assert batch.current_batch_size > 0
        if batch is self.request_handler.prefill_bb:       # prompts first run through the normal prefill
            return self._step_with_batch(batch)
        n = self.n_spec_tokens
        self.request_handler.allocate_batch_spec_dec(batch, n)
        seqs = batch.seqs_li
        # 1) draft
        drafted = []
        for s in seqs:
            ctx = torch.tensor([s.input_token_id + s.output_token_id], device=self.device)
            glide = None
            if self.use_glide:
                # the drafter glimpses the target model's last-layer KV of the tokens verified so far
                i = len(drafted)
                glide = GlideInput(block_tables=batch.block_tables[i: i + 1].to(self.device),
                                   large_k_cache=self.kv_runtime.k_caches[-1],
                                   large_v_cache=self.kv_runtime.v_caches[-1],
                                   sequence_lengths=batch._sequence_lengths[i: i + 1] - 1, n_spec_tokens=n)
            out = self.drafter.speculate(ctx, n, glide_input=glide)
            drafted.append(out.next_tokens.tolist())
        for s, d in zip(seqs, drafted):
            s.output_token_id += d
        batch._sequence_lengths[: len(seqs)] += n
        # 2) verify: feed last accepted token + n drafted tokens (n+1 queries per sequence)
        batch.set_use_spec_dec(n)
        input_ids = batch.get_1D_inputs().to(self.device)
        lens = batch.get_sequence_lengths()
        positions = self.kv_runtime.set_step(batch.get_block_table_tensor(), lens, False, self.device, q_per_seq=n + 1)
        from ...models.transformer import SeqMeta

        meta = SeqMeta(batch=1, seqlen=input_ids.numel(), positions=positions)
        logits = self.model(input_ids=input_ids.view(1, -1), kv_cache=self.kv_runtime, meta=meta)["logits"]
        target = logits.view(len(seqs), n + 1, -1).argmax(-1).tolist()
        # 3) accept
        for i, (s, d) in enumerate(zip(seqs, drafted)):
            hit = 0
            while hit < n and d[hit] == target[i][hit]:
                hit += 1
            drop = n - hit
            if drop:
                s.output_token_id = s.output_token_id[:-drop]
                batch._sequence_lengths[i] -= drop
            s.output_token_id.append(target[i][hit])
            batch._sequence_lengths[i] += 1
            self.request_handler.cache_manager.allocate_token_from_block_table(batch.block_tables[i],
                                                                               int(batch._sequence_lengths[i]))
        return self.request_handler.update()

    # ------------------------------------------------------------------ public API
    def generate(self, request_ids: Union[List[int], int] = None, prompts: Union[List[str], str] = None,
                 prompts_token_ids: Union[List[int], torch.Tensor, np.ndarray] = None, return_token_ids: bool = False,
                 generation_config: Optional[GenerationConfig] = None):
        gen = generation_config or self.generation_config
        with torch.inference_mode():
            if isinstance(prompts, str) and isinstance(request_ids, int):
                prompts, request_ids = [prompts], [request_ids]
            if prompts is not None or prompts_token_ids is not None:
                self.add_request(request_ids=request_ids, prompts=prompts, prompts_token_ids=prompts_token_ids,
                                 generation_config=gen)
            self.generation_config = gen
            self.generation_config_dict = gen.to_dict()
            finished: List[Sequence] = []
            while self.request_handler.check_unfinished_reqs():
                finished += self.steps_spec_dec() if self.use_spec_dec else self.step()
            finished = sorted(finished, key=lambda s: s.request_id)
            token_ids = [s.input_token_id + s.output_token_id for s in finished]
            out_strs = self.tokenizer.batch_decode([s.output_token_id for s in finished], skip_special_tokens=True)
            return (out_strs, token_ids) if return_token_ids else out_strs

    @property
    def has_prompt_template(self) -> bool:
        return self.inference_config.prompt_template is not None

    def format_prompt(self, prompts: Union[List[str], str]) -> Union[List[str], str]:
        assert self.has_prompt_template
        tpl = self.inference_config.prompt_template
        if isinstance(prompts, (list, tuple)):
            return [tpl.format(input_text=p) for p in prompts]
        return tpl.format(input_text=prompts)

    def add_request(self, request_ids: Union[List[int], int] = None, prompts: Union[List[str], str] = None,
                    prompts_token_ids: Union[List[int], torch.Tensor, np.ndarray] = None, **kwargs) -> None:
        if prompts is not None and self.has_prompt_template:
            prompts = self.format_prompt(prompts)
        block_size = self.inference_config.block_size
        if request_ids is not None and not isinstance(request_ids, list):
            request_ids = [request_ids]
        if prompts is not None and not isinstance(prompts, list):
            prompts = [prompts]
        if prompts_token_ids is None:
            assert prompts, "When prompts_token_ids is None, the input prompt list must be provided."
            prompts_token_ids = self.tokenizer(prompts, padding=False)["input_ids"]
        if isinstance(prompts_token_ids, (torch.Tensor, np.ndarray)):
            prompts_token_ids = prompts_token_ids.tolist()
        if prompts_token_ids and not isinstance(prompts_token_ids[0], (list, tuple)):
            prompts_token_ids = [prompts_token_ids]
        n = len(prompts_token_ids)
        gen = kwargs.get("generation_config") or self.generation_config
        max_new = gen.max_new_tokens or self.inference_config.max_output_len
        for i in range(n):
            rid = request_ids[i] if request_ids else next(self.counter)
            prompt = None if prompts is None else prompts[i]
            eos = getattr(self.tokenizer, "eos_token_id", None)
            if eos is None:
                eos = self.model_config.eos_token_id
            seq = Sequence(rid, prompt, list(prompts_token_ids[i]), block_size, None, eos,
                           getattr(self.tokenizer, "pad_token_id", 0) or 0, max_output_len=max_new,
                           ignore_eos=self.inference_config.ignore_eos)
            self.request_handler.add_sequence(seq)

    def prepare_input(self, batch: BatchBucket) -> Tuple[torch.Tensor, torch.Tensor, InputMetaData]:
        input_ids = batch.get_1D_inputs().to(self.device)
        lens = batch.get_sequence_lengths()
        is_prompt = batch is self.request_handler.prefill_bb
        if is_prompt and self.inference_config.enable_prefix_caching:
            positions = self.kv_runtime.set_step(batch.get_block_table_tensor(), lens, is_prompt, self.device,
                                                 num_cached=batch.get_num_cached_tokens())
        else:
            positions = self.kv_runtime.set_step(batch.get_block_table_tensor(), lens, is_prompt, self.device)
        meta = InputMetaData(block_tables=self.kv_runtime.block_tables, sequence_lengths=self.kv_runtime.seq_lens,
                             batch_size=batch.current_batch_size, is_prompts=is_prompt,
                             use_cuda_kernel=self.inference_config.use_cuda_kernel,
                             kv_seq_len=int(lens.max()) if lens.numel() else 0, head_dim=self.model_config.head_dim,
                             dtype=self.dtype, batch_token_ids=batch.batch_token_ids)
        return input_ids, positions, meta

    def _step_with_batch(self, batch: BatchBucket) -> List[Sequence]:
        if self.inference_config.max_num_batched_tokens is not None and batch is self.request_handler.prefill_bb:
            return self._step_chunked()
        input_ids, positions, meta = self.prepare_input(batch)
        bs = batch.current_batch_size
        if self.use_cuda_graph and not meta.is_prompts and bs in self.graph_runners:
            rt = self.kv_runtime
            logits = self.graph_runners[bs](input_ids=input_ids, block_tables=rt.block_tables, seq_lens=rt.seq_lens,
                                            positions=positions, token_seq=rt.token_seq, token_pos=rt.token_pos)
        else:
            logits = self._model_forward(input_ids, positions)
        if meta.is_prompts:   # keep the logits of the last prompt token of every sequence
            last = (self.kv_runtime.cu_seqlens[1:] - 1).long()
            logits = logits[last]
        next_tokens = self._sample(logits, meta.is_prompts, meta.batch_token_ids)
        self.request_handler.append_next_tokens(next_tokens.cpu())
        return self.request_handler.update()

    def _sample(self, logits: torch.Tensor, is_prompts: bool, batch_token_ids: List[List[int]]) -> torch.Tensor:
        logits = logits[:, : self.model_config.vocab_size]
        if self.tp_group is not None and logits.shape[-1] < self.model_config.vocab_size:
            from ...parallel import comm

            logits = comm.all_gather(logits.contiguous(), -1, self.tp_group)[:, : self.model_config.vocab_size]
        return search_tokens(self.generation_config, logits, is_prompts, batch_token_ids=batch_token_ids)

    def _step_chunked(self) -> List[Sequence]:
        """One chunked-prefill step (`RequestHandler._schedule_chunks`): the planned prompt chunks, then one token of
        every decoding sequence, in one forward.  It samples the last row of every prompt the step completes and every
        decode row, in one call; a prompt with chunks left samples nothing."""
        rh = self.request_handler
        pre, dec = rh.prefill_bb, rh.running_bb
        n_dec = dec.current_batch_size if rh.decode_in_step else 0
        seqs = pre.seqs_li[: len(rh.prefill_chunks)]
        starts = [s.num_cached_tokens for s in seqs]
        ends = [c + n for c, n in zip(starts, rh.prefill_chunks)]
        ids = [t for s, c, e in zip(seqs, starts, ends) for t in s.input_token_id[c:e]]
        if n_dec:
            ids += dec.get_1D_inputs().tolist()
        tables = torch.cat([pre.block_tables[: len(seqs)], dec.block_tables[:n_dec]])
        lens = torch.tensor(ends + dec.seq_lengths[:n_dec].tolist(), dtype=torch.int32)
        positions = self.kv_runtime.set_chunked_step(tables, lens, starts, self.device)
        logits = self._model_forward(torch.tensor(ids, dtype=torch.long, device=self.device), positions)
        cu = list(accumulate(rh.prefill_chunks))
        done = [i for i, (s, e) in enumerate(zip(seqs, ends)) if e == s.input_len]
        pick = [cu[i] - 1 for i in done] + list(range(cu[-1], cu[-1] + n_dec))
        tokens = []
        if pick:
            token_ids = [seqs[i].input_token_id for i in done] + (dec.batch_token_ids if n_dec else [])
            rows = torch.tensor(pick, dtype=torch.long, device=self.device)
            tokens = self._sample(logits[rows], False, token_ids).tolist()
        rh.append_chunked_tokens(tokens)
        return rh.update()

    @torch.inference_mode()
    def step(self) -> List[Sequence]:
        batch = self.request_handler.schedule()
        if batch.is_empty:
            return self.request_handler.update()
        return self._step_with_batch(batch)
