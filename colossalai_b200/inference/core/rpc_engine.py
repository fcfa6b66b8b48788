"""RPC engine: the scheduler lives in this process, one model-executor worker process per GPU.
Parity: reference `colossalai/inference/core/rpc_engine.py:36-297` (`RPCInferenceEngine.{init_workers,
init_worker_env,init_model,init_device_cache,prepare_input,step,kill_workers}`)."""
from __future__ import annotations

import asyncio
import multiprocessing as mp
import time
from itertools import count
from multiprocessing.connection import Client
from typing import Any, List, Optional, Tuple

import torch

from ...logging import get_dist_logger
from ...models import get_config
from ...models.config import ModelConfig
from ..batch_bucket import BatchBucket
from ..config import InferenceConfig
from ..executor.rpc_worker import serve_worker
from ..struct import Sequence
from ..utils import find_available_ports
from .llm_engine import LLMEngine, _SimpleTokenizer
from .request_handler import RPCRequestHandler

__all__ = ["RPCInferenceEngine"]


class RPCInferenceEngine(LLMEngine):
    def __init__(self, model_or_path, tokenizer=None, inference_config: InferenceConfig = None, verbose: bool = False,
                 model_policy=None) -> None:
        assert isinstance(model_or_path, (str, ModelConfig)), "the RPC engine takes a zoo name / config / checkpoint path"
        self.inference_config = inference_config or InferenceConfig()
        self.dtype = self.inference_config.dtype
        self.verbose = verbose
        self.logger = get_dist_logger(__name__)
        self.tokenizer = tokenizer or _SimpleTokenizer()
        self.model_spec = model_or_path
        self.model_config = get_config(model_or_path) if isinstance(model_or_path, str) else model_or_path
        self.tp_size = self.inference_config.tp_size
        self.generation_config = self.inference_config.to_generation_config(self.model_config)
        self.generation_config_dict = self.generation_config.to_dict()
        self.use_spec_dec = False
        self.use_cuda_graph = False
        self.counter = count()
        self.workers: List[Any] = []
        self.procs: List[mp.Process] = []
        self._verify_args()
        self.init_workers()
        asyncio.run(self.init_worker_env())
        asyncio.run(self.init_model(self.model_spec, model_policy))
        self.request_handler = self.init_scheduler(self.inference_config, self.model_config)
        self.init_device_cache(None)

    def _verify_args(self) -> None:
        assert isinstance(self.inference_config, InferenceConfig)
        assert self.inference_config.pp_size == 1, "RPC engine: tensor parallelism only"
        if self.inference_config.enable_prefix_caching:
            raise ValueError("the RPC engine does not support enable_prefix_caching")
        if self.inference_config.max_num_batched_tokens is not None:
            raise ValueError("the RPC engine does not support max_num_batched_tokens")

    # ------------------------------------------------------------------ workers
    def init_workers(self) -> None:
        ctx = mp.get_context("spawn")
        ports = find_available_ports(self.tp_size)
        self.worker_addresses = [("127.0.0.1", p) for p in ports]
        for addr in self.worker_addresses:
            ev = ctx.Event()
            p = ctx.Process(target=serve_worker, args=(addr, b"cb200", ev), daemon=True)
            p.start()
            assert ev.wait(120), "inference worker failed to start"
            self.procs.append(p)
        for addr in self.worker_addresses:
            for _ in range(200):
                try:
                    self.workers.append(Client(addr, authkey=b"cb200"))
                    break
                except ConnectionRefusedError:
                    time.sleep(0.05)
        assert len(self.workers) == self.tp_size

    def _call(self, conn, method: str, *args, **kwargs):
        conn.send((method, args, kwargs))
        status, res = conn.recv()
        if status != "ok":
            raise RuntimeError(f"inference worker failed in {method}: {res}")
        return res

    async def async_parallel_wrapper(self, method: str, per_worker_args: List[tuple]):
        """Issue `method` on every worker concurrently (threads; the sockets block)."""
        loop = asyncio.get_running_loop()
        futs = [loop.run_in_executor(None, self._call, w, method, *a) for w, a in zip(self.workers, per_worker_args)]
        return await asyncio.gather(*futs)

    async def init_worker_env(self) -> None:
        port = find_available_ports(1)[0]
        await self.async_parallel_wrapper("init_dist_env", [(r, self.tp_size, "127.0.0.1", port)
                                                             for r in range(self.tp_size)])

    async def init_model(self, model_or_path, model_policy=None) -> None:
        await self.async_parallel_wrapper("init_model", [(model_or_path, self.inference_config, model_policy)] * self.tp_size)

    def init_scheduler(self, inference_config: InferenceConfig, model_config) -> RPCRequestHandler:
        return RPCRequestHandler(inference_config, model_config)

    def init_device_cache(self, alloc_shape) -> None:
        asyncio.run(self.async_parallel_wrapper("init_cache", [(alloc_shape,)] * self.tp_size))

    # ------------------------------------------------------------------ stepping
    def prepare_input(self, batch: BatchBucket) -> Tuple[List[int], dict]:
        is_prompt = batch is self.request_handler.prefill_bb
        ids = batch.get_1D_inputs().tolist()
        meta = {"block_tables": batch.get_block_table_tensor().tolist(),
                "sequence_lengths": batch.get_sequence_lengths().tolist(), "is_prompts": is_prompt,
                "batch_token_ids": batch.batch_token_ids}
        return ids, meta

    async def step_(self, input_token_ids, meta):
        res = await self.async_parallel_wrapper("execute_model_forward",
                                                [(input_token_ids, meta, self.generation_config_dict)] * self.tp_size)
        return res[0]

    def step(self) -> List[Sequence]:
        batch = self.request_handler.schedule()
        if batch.is_empty:
            return self.request_handler.update()
        ids, meta = self.prepare_input(batch)
        next_tokens = asyncio.run(self.step_(ids, meta))
        self.request_handler.append_next_tokens(torch.tensor(next_tokens))
        return self.request_handler.update()

    def kill_workers(self) -> None:
        for w in self.workers:
            try:
                self._call(w, "shutdown")
                w.close()
            except Exception:
                pass
        self.workers = []
        for p in self.procs:
            p.join(timeout=10)
            if p.is_alive():
                p.terminate()
        self.procs = []

    def __del__(self):
        try:
            self.kill_workers()
        except Exception:
            pass
