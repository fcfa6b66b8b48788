"""Reference arm of bench.py: runs the UNMODIFIED reference (hpcaitech/ColossalAI 0.5.0 installed into baseline/_ref with
`pip install --no-deps --target baseline/_ref`) through its own public API (`colossalai.launch_from_torch`, `Booster`,
a stock plugin) on the same metric/config as our arm: Llama-3-8B shape, bf16, seq 4096, one sequence per GPU per step,
AdamW, synthetic tokens, random init; K device-timed steps, max over ranks.

What is and is not possible offline (recorded in DESIGN.md):
  * the reference hard-imports packages that are not in this image (peft, galore_torch, bitsandbytes, ...).  They are
    never exercised by the benchmark path, so this file registers EMPTY stub modules for them before importing the
    reference - the reference's own files are untouched;
  * the reference's Shardformer forwards are written against transformers 4.51.3 (not in the offline wheelhouse); the
    installed transformers 5.5 changed the `LlamaDecoderLayer.forward` signature / return type.
    `install_transformers_shims()` adapts the INSTALLED transformers class (not the reference) so the reference's own
    TP + sequence-parallel path runs (checked on the CPU/gloo tier with a tiny Llama: loss decreases);
  * the reference benchmark's optimizer `HybridAdam` needs two native extensions; `baseline/build_ref_ext.py` builds
    them ahead of time with the reference's own `build_aot()` recipe into `baseline/_ref/colossalai/_C/`.

Rows (`--parallelism tp|dp|both`, the same flag as our arm): `tp` = HybridParallelPlugin(tp=N, split_gather SP) with a
fallback ladder, `dp` = LowLevelZeroPlugin(stage=1) accumulating under `no_sync` (falls back to stage 2 / DDP).  Every
row reports the stock plugin that actually ran in `parallelism` / `skipped_plugins`.
"""
from __future__ import annotations

import contextlib
import json
import os
import sys
import time
import types

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
REF = os.path.join(ROOT, "baseline", "_ref")
STUBS = ["peft", "galore_torch", "bitsandbytes", "ray", "rpyc", "diffusers", "tensornvme", "apex", "xformers"]


class _Dummy:
    def __init__(self, *a, **k):
        pass

    def __call__(self, *a, **k):
        return _Dummy()

    def __getattr__(self, n):
        return _Dummy()


class _StubModule(types.ModuleType):
    def __getattr__(self, name):
        if name.startswith("__"):
            raise AttributeError(name)
        cls = type(name, (_Dummy,), {})
        setattr(self, name, cls)
        return cls


class _StubFinder:
    def find_spec(self, name, path, target=None):
        if name.split(".")[0] in STUBS:
            from importlib.machinery import ModuleSpec

            return ModuleSpec(name, self, is_package=True)
        return None

    def create_module(self, spec):
        m = _StubModule(spec.name)
        m.__path__ = []
        return m

    def exec_module(self, module):
        pass


def install_transformers_shims() -> None:
    """Environment shims on the INSTALLED transformers (5.x) so the unmodified reference, written against
    transformers 4.51.3, can run its own Shardformer TP/SP forwards.  Nothing under baseline/_ref is touched:

    * 4.51 exported `StaticCache/DynamicCache/Cache` from `modeling_llama`; 5.x keeps them in `cache_utils` only;
    * 4.51's `LlamaDecoderLayer.forward(hidden_states, attention_mask, position_ids, past_key_value,
      output_attentions, use_cache, cache_position, position_embeddings)` returned a TUPLE `(hidden_states, ...)`;
      5.x renamed `past_key_value`, dropped `output_attentions` / `cache_position` from the positional list and returns
      the bare tensor.  The reference's `llama_model_forward` calls the 4.51 signature and indexes `layer_outputs[0]`
      (`shardformer/modeling/llama.py:200-222`), so the class method is wrapped to accept the old call and return a
      tuple.  The math inside the layer is the installed transformers' own, with the reference's replaced attention
      forward and parallel linears, exactly as under 4.51.
    """
    try:
        import transformers.cache_utils as _cu
        import transformers.models.llama.modeling_llama as _ml
    except Exception:
        return
    for _n in ("StaticCache", "DynamicCache", "Cache"):
        if not hasattr(_ml, _n) and hasattr(_cu, _n):
            setattr(_ml, _n, getattr(_cu, _n))
    layer_cls = _ml.LlamaDecoderLayer
    if getattr(layer_cls, "_cb200_ref_shim", False):
        return
    import inspect

    params = inspect.signature(layer_cls.forward).parameters
    if "past_key_value" in params:          # a 4.x transformers: nothing to adapt
        return
    orig = layer_cls.forward

    def forward(self, hidden_states, attention_mask=None, position_ids=None, past_key_value=None,
                output_attentions=False, use_cache=False, cache_position=None, position_embeddings=None, **kwargs):
        if "past_key_values" in kwargs:
            # a call in the installed transformers' own convention (its stock `LlamaModel.forward`, used by the
            # reference's DDP / ZeRO plugins which do not replace the model forward): pass through untouched
            return orig(self, hidden_states, attention_mask=attention_mask, position_ids=position_ids,
                        use_cache=use_cache, position_embeddings=position_embeddings, **kwargs)
        out = orig(self, hidden_states, attention_mask=attention_mask, position_ids=position_ids,
                   past_key_values=past_key_value, use_cache=use_cache, position_embeddings=position_embeddings,
                   cache_position=cache_position, output_attentions=output_attentions, **kwargs)
        return out if isinstance(out, tuple) else (out,)

    layer_cls.forward = forward
    layer_cls._cb200_ref_shim = True


def _unavailable(why: str) -> None:
    if int(os.environ.get("RANK", "0")) == 0:
        print(json.dumps({"impl": "reference", "unavailable": why.replace("\n", " ")[:300]}), flush=True)


def run_reference_arm(args) -> None:
    if not os.path.isdir(os.path.join(REF, "colossalai")):
        _unavailable("baseline/_ref is missing (pip install --no-deps --target baseline/_ref <reference checkout> not done)")
        return
    # make sure OUR package is not importable by accident on this path
    sys.path[:] = [p for p in sys.path if os.path.abspath(p or ".") != ROOT]
    sys.path.insert(0, REF)
    for name in STUBS:
        try:
            __import__(name)
        except Exception:
            if not any(isinstance(f, _StubFinder) for f in sys.meta_path):
                sys.meta_path.append(_StubFinder())
    try:
        import torch
        import torch.distributed as dist
        import colossalai
        from colossalai.booster import Booster
    except Exception as e:
        _unavailable(f"reference import failed: {type(e).__name__}: {e}")
        return
    if not torch.cuda.is_available():
        _unavailable("no CUDA device")
        return

    if "RANK" not in os.environ:
        os.environ.update(RANK="0", LOCAL_RANK="0", WORLD_SIZE="1", MASTER_ADDR="127.0.0.1",
                          MASTER_PORT=str(29500 + os.getpid() % 2000))
    try:
        colossalai.launch_from_torch()
    except Exception as e:
        _unavailable(f"colossalai.launch_from_torch failed: {type(e).__name__}: {e}")
        return
    rank, world = dist.get_rank(), dist.get_world_size()
    dev = torch.device("cuda", torch.cuda.current_device())
    from transformers import LlamaConfig, LlamaForCausalLM

    shapes = {"llama3-8b": dict(vocab_size=128256, hidden_size=4096, intermediate_size=14336, num_hidden_layers=32,
                                num_attention_heads=32, num_key_value_heads=8, max_position_embeddings=8192,
                                rope_theta=500000.0)}
    hf_cfg = LlamaConfig(**shapes.get(args.model, shapes["llama3-8b"]))
    if args.layers:
        hf_cfg.num_hidden_layers = args.layers
    attn_impl = "sdpa"
    try:
        import flash_attn  # noqa: F401

        attn_impl = "flash_attention_2"
    except Exception:
        pass

    def build_model():
        torch.manual_seed(1234)
        with torch.device(dev):
            try:
                m = LlamaForCausalLM._from_config(hf_cfg, attn_implementation=attn_impl, torch_dtype=torch.bfloat16)
            except Exception:
                m = LlamaForCausalLM._from_config(hf_cfg, attn_implementation="sdpa", torch_dtype=torch.bfloat16)
        return m

    install_transformers_shims()

    import gc
    import traceback

    sys.path.insert(0, ROOT)            # only for the helpers shared with our arm (labels, clock sampler) in bench.py
    try:
        from bench import METRIC, ClockSampler, row_label, shared_config
    finally:
        sys.path[:] = [p for p in sys.path if os.path.abspath(p or ".") != ROOT]

    # ---- optimizer: the reference's own benchmark uses HybridAdam (examples/language/llama/benchmark.py); its two
    # native extensions are prebuilt by baseline/build_ref_ext.py.  Probe them in a child process first (a CPU-ISA
    # mismatch would kill the process, not raise).
    opt_name = "torch.optim.AdamW inside the reference's OptimizerWrapper"
    HybridAdam = None
    if os.environ.get("CB200_REF_OPTIM", "hybrid_adam") == "hybrid_adam":
        import subprocess

        probe = ("import sys; sys.path.insert(0, %r); sys.path.insert(0, %r); import reference_arm as ra; "
                 "sys.meta_path.append(ra._StubFinder()); import torch; from colossalai.nn.optimizer import HybridAdam; "
                 "p=[torch.nn.Parameter(torch.randn(64, 64)), torch.nn.Parameter(torch.randn(64, 64, device='cuda'))]; "
                 "o=HybridAdam(p, lr=1e-3); [setattr(q, 'grad', torch.randn_like(q)) for q in p]; o.step(); "
                 "torch.cuda.synchronize(); print('HYBRID_ADAM_OK')") % (REF, os.path.join(ROOT, "baseline"))
        ok = False
        if rank == 0:
            try:
                r = subprocess.run([sys.executable, "-c", probe], capture_output=True, text=True, timeout=600)
                ok = "HYBRID_ADAM_OK" in r.stdout
                if not ok:
                    print("[reference arm] HybridAdam probe failed: " + (r.stderr or r.stdout)[-400:], file=sys.stderr)
            except Exception as e:
                print(f"[reference arm] HybridAdam probe failed: {e}", file=sys.stderr)
        flag = torch.tensor([1 if ok else 0], device=dev)
        dist.broadcast(flag, 0)
        if int(flag.item()) == 1:
            from colossalai.nn.optimizer import HybridAdam

            opt_name = "colossalai.nn.optimizer.HybridAdam (the reference benchmark's optimizer)"

    def make_optimizer(params):
        if HybridAdam is not None:
            return HybridAdam(params, lr=1e-5, betas=(0.9, 0.95), weight_decay=0.1)
        return torch.optim.AdamW(params, lr=1e-5, betas=(0.9, 0.95), weight_decay=0.1)

    S = args.seq

    def measure(kind: str, steps: int, with_e2e: bool):
        """One row: walk the ladder of stock reference configurations for this layout, time the first that steps."""
        if kind == "tp":
            plans = [("hybrid_tp", False), ("hybrid_tp", True)]
            if world == 1:
                plans += [("zero1", False), ("zero2", False), ("zero2", True), ("ddp", False)]
        else:
            plans = [("zero1", False), ("zero2", False), ("zero2", True), ("ddp", False)]
        chosen = None
        model = optimizer = booster = plugin = None
        errors = []
        for plan, ckpt in plans:
            label = {"hybrid_tp": row_label("tp", world), "zero1": row_label("dp", world) if world > 1 else "zero1(dp1)",
                     "zero2": f"zero2(dp{world})", "ddp": f"ddp(dp{world})"}[plan] + ("+grad_ckpt" if ckpt else "")
            try:
                if plan == "hybrid_tp":
                    from colossalai.booster.plugin import HybridParallelPlugin

                    plugin = HybridParallelPlugin(tp_size=world, pp_size=1, precision="bf16", zero_stage=0,
                                                  enable_sequence_parallelism=world > 1,
                                                  sequence_parallelism_mode="split_gather" if world > 1 else None,
                                                  enable_flash_attention=True, enable_fused_normalization=False,
                                                  max_norm=1.0)
                elif plan in ("zero1", "zero2"):
                    from colossalai.booster.plugin import LowLevelZeroPlugin

                    plugin = LowLevelZeroPlugin(stage=1 if plan == "zero1" else 2, precision="bf16", max_norm=1.0)
                else:
                    from colossalai.booster.plugin import TorchDDPPlugin

                    plugin = TorchDDPPlugin()
                booster = Booster(plugin=plugin)
                model = build_model()
                if ckpt:
                    model.gradient_checkpointing_enable()
                model.train()
                optimizer = make_optimizer(model.parameters())
                model, optimizer, _, _, _ = booster.boost(model, optimizer)
                # one probing step
                nseq = args.mbs * (world if plan == "hybrid_tp" else 1)
                ids = torch.randint(0, hf_cfg.vocab_size, (nseq, S), device=dev)
                out = model(input_ids=ids, labels=ids)
                booster.backward(out.loss, optimizer)
                optimizer.step()
                optimizer.zero_grad()
                torch.cuda.synchronize()
                del out, ids
                chosen = (plan, label)
                break
            except Exception as e:  # try the next stock configuration
                msg = f"{label}: {type(e).__name__}: {str(e)[:200]}"
                errors.append(msg)
                if rank == 0:
                    print("[reference arm] " + msg, file=sys.stderr, flush=True)
                    if os.environ.get("CB200_REF_TRACE"):
                        traceback.print_exc()
                traceback.clear_frames(e.__traceback__)
                e = None
                model = optimizer = booster = plugin = None
                gc.collect()
                torch.cuda.empty_cache()
        if chosen is None:
            return None, errors
        tp_mode = chosen[0] == "hybrid_tp"
        # can gradient accumulation skip the per-micro-step gradient reduction?  (the reference forbids no_sync
        # under ZeRO-2; everything else supports it)
        use_no_sync = False
        try:
            use_no_sync = bool(plugin.support_no_sync()) and chosen[0] != "zero2" and args.accum > 1
        except Exception:
            use_no_sync = False

        # TP: every rank feeds the same global batch of mbs*world sequences (as our arm does); DP: mbs per rank.
        B = args.mbs * world if tp_mode else args.mbs
        tokens_per_step = args.mbs * world * S * args.accum
        gen = torch.Generator().manual_seed(4321 + (0 if tp_mode else rank))
        host_ids = [torch.randint(0, hf_cfg.vocab_size, (args.accum, B, S), generator=gen).pin_memory()
                    for _ in range(4)]
        dev_ids = [h.to(dev) for h in host_ids]

        def step(ids_dev):
            loss_acc = 0.0
            for a in range(args.accum):
                last = a == args.accum - 1
                ctx = booster.no_sync(model, optimizer) if (use_no_sync and not last) else contextlib.nullcontext()
                with ctx:
                    out = model(input_ids=ids_dev[a], labels=ids_dev[a])
                    loss = out.loss / args.accum
                    booster.backward(loss, optimizer)
                loss_acc = loss.detach() + loss_acc
            optimizer.step()
            optimizer.zero_grad()
            return loss_acc

        def timed(n, e2e):
            dist.barrier()
            torch.cuda.synchronize()
            s_ev, e_ev = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            t0 = time.perf_counter()
            s_ev.record()
            last = None
            for i in range(n):
                if e2e:
                    last = step(host_ids[i % 4].to(dev, non_blocking=True)).item()
                else:
                    last = step(dev_ids[i % 4])
            e_ev.record()
            torch.cuda.synchronize()
            dist.barrier()
            t = torch.tensor([s_ev.elapsed_time(e_ev), (time.perf_counter() - t0) * 1e3], device=dev,
                             dtype=torch.float64)
            dist.all_reduce(t, op=dist.ReduceOp.MAX)
            return t[0].item(), t[1].item(), (last.item() if torch.is_tensor(last) else last)

        torch.cuda.reset_peak_memory_stats()
        for i in range(max(args.warmup - 1, 0)):          # the probing step above was warm-up step 1
            step(dev_ids[i % 4])
        sampler = ClockSampler(torch.cuda.current_device()) if rank == 0 else None
        if sampler:
            sampler.start()
        ms, wall, loss_val = timed(steps, False)
        clocks = sampler.stop() if sampler else {}
        row = {"parallelism": chosen[1], "value": tokens_per_step * steps / (ms / 1e3), "unit": "tokens/s",
               "steps": steps, "ms_per_step": ms / steps, "wall_ms_per_step": wall / steps,
               "global_batch": args.mbs * world * args.accum, "reference_plugin": chosen[0],
               "no_sync_accumulation": use_no_sync, "skipped_plugins": errors, "loss": loss_val, "clocks": clocks,
               "peak_mem_mib": torch.cuda.max_memory_allocated() / 2**20}
        if with_e2e:
            ms_e, wall_e, _ = timed(steps, True)
            row["e2e"] = {"value": tokens_per_step * steps / (max(ms_e, wall_e) / 1e3), "unit": "tokens/s",
                          "h2d_bytes_per_step": host_ids[0].numel() * 8, "d2h_bytes_per_step": 4,
                          "ms_per_step": max(ms_e, wall_e) / steps}
        del model, optimizer, booster, plugin, dev_ids, host_ids, step, timed
        gc.collect()
        torch.cuda.empty_cache()
        return row, errors

    kinds = {"tp": ["tp"], "dp": ["dp"], "both": ["tp", "dp"]}[getattr(args, "parallelism", "both")]
    if world == 1:
        kinds = kinds[:1]
    rows, all_errors = [], []
    for i, kind in enumerate(kinds):
        steps = args.steps if i == 0 else max(3, args.steps // 2)
        row, errs = measure(kind, steps, not args.no_e2e)
        all_errors += errs
        if row is not None:
            rows.append(row)
        elif i == 0:
            # the named layout does not run on this stack: the companion layout becomes the headline
            continue
    if not rows:
        _unavailable("no stock plugin of the reference runs on this stack: " + " | ".join(e_[:120] for e_ in all_errors))
        return
    head = rows[0]
    res = {"metric": METRIC, "value": head["value"], "unit": "tokens/s", "n_gpus": world, "steps": head["steps"],
           "warmup": args.warmup, "ms_per_step": head["ms_per_step"], "higher_is_better": True, "scaling": "weak",
           "vs_baseline": None, "dtype": "bf16", "data": "synthetic tokens, random-init weights", "impl": "reference",
           "config": shared_config(args, world, head["parallelism"]),
           "detail": {"reference_plugin": head["reference_plugin"], "attn": attn_impl, "optimizer_impl": opt_name,
                      "no_sync_accumulation": head["no_sync_accumulation"], "skipped_plugins": all_errors,
                      "transformers_shim": "LlamaDecoderLayer.forward 4.51-style signature / tuple return (see "
                                           "baseline/reference_arm.py:install_transformers_shims)"},
           "clocks": head["clocks"], "gpu_launches": 0, "loss": head["loss"], "peak_mem_mib": head["peak_mem_mib"],
           "rows": rows}
    if "e2e" in head:
        res["e2e"] = head["e2e"]
    if rank == 0:
        print(json.dumps(res), flush=True)
    dist.barrier()
    dist.destroy_process_group()
