"""Decode / prefill throughput of the inference engine (reference: examples/inference/llama/benchmark_llama.py).

    python examples/inference/benchmark_llama.py -m llama3-8b -b 32 --in_len 512 --out_len 128 [--cuda_graph] [--layers 8]

Prints one JSON line: prefill tokens/s, decode tokens/s (device-timed with CUDA events), per-step latency."""
import argparse
import json
import os
import sys
import time

import torch

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), "..", ".."))

from colossalai_b200.inference import GenerationConfig, InferenceConfig, InferenceEngine  # noqa: E402
from colossalai_b200.kernel import loader  # noqa: E402
from colossalai_b200.lazy import LazyInitContext  # noqa: E402
from colossalai_b200.models import build_model, get_config  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("-m", "--model", default="llama3-8b")
    ap.add_argument("-b", "--batch_size", type=int, default=32)
    ap.add_argument("--in_len", type=int, default=512)
    ap.add_argument("--out_len", type=int, default=128)
    ap.add_argument("--layers", type=int, default=0, help="debug: override the layer count")
    ap.add_argument("--cuda_graph", action="store_true")
    ap.add_argument("--dtype", default="bf16")
    ap.add_argument("--profile", default="", help="write a per-kernel breakdown of 8 decode steps to this file")
    args = ap.parse_args()
    assert torch.cuda.is_available(), "this benchmark needs a GPU"
    cfg = get_config(args.model, **({"num_hidden_layers": args.layers} if args.layers else {}))
    torch.manual_seed(0)
    with LazyInitContext():
        model = build_model(cfg)
    LazyInitContext.materialize(model)
    icfg = InferenceConfig(max_batch_size=args.batch_size, max_input_len=args.in_len, max_output_len=args.out_len,
                           dtype=args.dtype, use_cuda_graph=args.cuda_graph, block_size=64, ignore_eos=True)
    engine = InferenceEngine(model, None, icfg)
    g = torch.Generator().manual_seed(1)
    prompts = torch.randint(3, cfg.vocab_size, (args.batch_size, args.in_len), generator=g).tolist()
    gen = GenerationConfig(max_new_tokens=args.out_len)
    eng = engine.engine
    eng.generation_config, eng.generation_config_dict = gen, gen.to_dict()

    def run():
        eng.add_request(prompts_token_ids=prompts, generation_config=gen)
        torch.cuda.synchronize()
        e0, e1, e2 = (torch.cuda.Event(enable_timing=True) for _ in range(3))
        e0.record()
        eng.step()                                  # prefill of the whole batch
        e1.record()
        steps = 1
        while eng.request_handler.check_unfinished_reqs():
            eng.step()
            steps += 1
        e2.record()
        torch.cuda.synchronize()
        return e0.elapsed_time(e1), e1.elapsed_time(e2), steps

    run()                                           # warm-up (graph capture, allocator)
    loader.launch_counter.reset()
    t_prefill, t_decode, steps = run()
    out = {"model": args.model + (f"[layers={args.layers}]" if args.layers else ""), "batch": args.batch_size,
           "in_len": args.in_len, "out_len": args.out_len, "cuda_graph": args.cuda_graph, "dtype": args.dtype,
           "prefill_ms": t_prefill, "prefill_tokens_per_s": args.batch_size * args.in_len / (t_prefill / 1e3),
           "decode_ms_per_step": t_decode / max(steps - 1, 1),
           "decode_tokens_per_s": args.batch_size * (steps - 1) / (t_decode / 1e3),
           "our_kernel_launches": loader.launch_counter.count,
           "peak_mem_gib": torch.cuda.max_memory_allocated() / 2**30}
    # decode is HBM-bound: every step streams all weights once plus the live KV cache; roofline = bytes / measured
    # copy bandwidth (MEASURED_PEAKS.json when present)
    hbm_gbs = 6555.8
    try:
        hbm_gbs = json.load(open(os.path.join(os.path.dirname(os.path.abspath(__file__)), "..", "..",
                                              "MEASURED_PEAKS.json")))["hbm_gbs"]
    except Exception:
        pass
    n_params = sum(p.numel() for p in model.parameters())
    w_bytes = n_params * 2
    ctx = args.in_len + args.out_len / 2
    kv_bytes = args.batch_size * ctx * 2 * cfg.num_hidden_layers * cfg.num_key_value_heads * cfg.head_dim * 2
    roof_ms = (w_bytes + kv_bytes) / (hbm_gbs * 1e9) * 1e3
    out.update({"params": n_params, "decode_hbm_roofline_ms": roof_ms,
                "decode_frac_of_measured_hbm_roofline": roof_ms / out["decode_ms_per_step"],
                "prefill_tflops": 2.0 * n_params * args.batch_size * args.in_len / (t_prefill / 1e3) / 1e12})
    print(json.dumps(out), flush=True)
    if args.profile:
        from torch.profiler import ProfilerActivity, profile

        eng.add_request(prompts_token_ids=prompts, generation_config=gen)
        eng.step()
        for _ in range(4):
            eng.step()
        torch.cuda.synchronize()
        import time
        t0 = time.perf_counter()
        with profile(activities=[ProfilerActivity.CUDA, ProfilerActivity.CPU]) as prof:
            for _ in range(8):
                eng.step()
            torch.cuda.synchronize()
        wall = (time.perf_counter() - t0) / 8 * 1e3
        while eng.request_handler.check_unfinished_reqs():
            eng.step()
        evs = [e for e in prof.key_averages() if e.device_time_total > 0 and str(e.device_type).endswith("CUDA")]
        tot = sum(e.device_time_total for e in evs) / 8 / 1e3
        with open(args.profile, "w") as f:
            f.write(f"# decode step: wall {wall:.3f} ms (under profiler), sum of GPU kernel time {tot:.3f} ms/step\n")
            for e in sorted(evs, key=lambda e: -e.device_time_total)[:25]:
                f.write(f"{e.device_time_total / 8 / 1e3:9.4f} ms/step  x{e.count / 8:7.1f}  {e.key[:110]}\n")


if __name__ == "__main__":
    main()
