"""Prefix caching on the GPU: the paged prefill kernel and the engine.

(a) Kernel.  `flash_prefill_paged` (new query rows against keys in a paged cache, block 16, blocks permuted) against
    the packed kernel (`flash_fwd(..., cu_seqlens=)`) recomputing the whole sequences from the same K/V gathered
    contiguous - what a prefill without a cache hit runs.  Attention shapes of Llama-3-8B (Hq 32, Hkv 8, D 128) and
    Llama-3.2-1B (Hq 32, Hkv 8, D 64); contexts (cached + new) of 1k / 4k / 16k tokens with 128 / 512 / 2048 new
    tokens, batch 1 and 8.  CUDA events after warm-up.  TFLOP/s from the causal FLOPs each kernel computes:
    4 * D * Hq * (keys seen) summed over its query rows.  At every shape the paged rows must equal the packed kernel's
    rows bit for bit.
(b) Engine.  A `llama3.2-1b`-shaped model with bf16 random weights, max_batch_size 8, no CUDA graphs (one new token per
    request, so no decode step).  Workload 1: 32 requests sharing a 2048-token prefix plus 64 distinct tokens each,
    max_new_tokens=1; workload 2: 32 distinct prompts of the same length.  Time to finish (host clock around
    `generate`, ended by a device synchronise), with prefix caching on and off, and the hit tokens.  Each engine is
    warmed up on two short prompts first.

Prints one JSON line with the card's name and power limit, read in the same run.  Needs a GPU.
"""
import argparse
import itertools
import json
import subprocess
import time

import torch

SHAPES = {"llama3-8b": (32, 8, 128), "llama3.2-1b": (32, 8, 64)}
CONTEXTS = [(1024, 128), (4096, 512), (16384, 2048)]
BLOCK = 16


def gpu_info():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
        name, power, clock = (s.strip() for s in out.split(","))
    except (OSError, IndexError, ValueError, subprocess.SubprocessError):
        name, power, clock = torch.cuda.get_device_name(), "unknown", "unknown"
    return {"gpu": name, "power_limit": power, "max_sm_clock": clock}


def cuda_ms(fn, min_window_s=0.2):
    for _ in range(3):
        fn()
    torch.cuda.synchronize()
    s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    n = 3
    while True:
        s.record()
        for _ in range(n):
            fn()
        e.record()
        e.synchronize()
        ms = s.elapsed_time(e)
        if ms >= min_window_s * 1e3:
            return ms / n
        n *= 2


def causal_flops(D, Hq, lens, new):
    """4 * D * Hq * sum over the query rows of the keys each row sees (rows at positions L - n .. L - 1)."""
    return sum(4 * D * Hq * (n * L - n * (n - 1) // 2) for L, n in zip(lens, new))


def kernel_rows():
    from colossalai_b200.ops import flash_attn_native as fa

    rows = []
    for (name, (Hq, Hkv, D)), (L, n), B in itertools.product(SHAPES.items(), CONTEXTS, (1, 8)):
        torch.manual_seed(0)
        dt = torch.bfloat16
        qf = torch.randn(B * L, Hq, D, device="cuda", dtype=dt)
        kf = torch.randn(B * L, Hkv, D, device="cuda", dtype=dt)
        vf = torch.randn(B * L, Hkv, D, device="cuda", dtype=dt)
        nblk = L // BLOCK
        perm = torch.randperm(B * nblk, device="cuda")
        tables = perm.view(B, nblk).to(torch.int32)
        kc = torch.empty(B * nblk, BLOCK, Hkv, D, device="cuda", dtype=dt)
        vc = torch.empty_like(kc)
        kc[perm] = kf.view(B * nblk, BLOCK, Hkv, D)
        vc[perm] = vf.view(B * nblk, BLOCK, Hkv, D)
        q = qf.view(B, L, Hq, D)[:, L - n:].reshape(B * n, Hq, D).contiguous()
        cu_full = torch.arange(B + 1, device="cuda", dtype=torch.int32) * L
        cu_new = torch.arange(B + 1, device="cuda", dtype=torch.int32) * n
        lens = torch.full((B,), L, device="cuda", dtype=torch.int32)
        scale = D ** -0.5

        def paged():
            return fa.flash_prefill_paged(q, kc, vc, tables, cu_new, lens, scale)

        def packed():
            return fa.flash_fwd(qf, kf, vf, 1, True, scale, cu_seqlens=cu_full)[0]

        bitwise = torch.equal(paged().view(B, n, Hq, D), packed().view(B, L, Hq, D)[:, L - n:])
        t_paged, t_packed = cuda_ms(paged), cuda_ms(packed)
        f_paged = causal_flops(D, Hq, [L] * B, [n] * B)
        f_packed = causal_flops(D, Hq, [L] * B, [L] * B)
        rows.append({"shape": name, "batch": B, "context": L, "new": n, "paged_ms": round(t_paged, 4),
                     "packed_full_ms": round(t_packed, 4), "speedup": round(t_packed / t_paged, 2),
                     "paged_tflops": round(f_paged / t_paged / 1e9, 1),
                     "packed_tflops": round(f_packed / t_packed / 1e9, 1), "bitwise_equal": bitwise})
        print(json.dumps(rows[-1]), flush=True)
        del qf, kf, vf, kc, vc, q
        torch.cuda.empty_cache()
    return rows


def engine_rows():
    from colossalai_b200.inference import InferenceConfig, InferenceEngine
    from colossalai_b200.inference.config import GenerationConfig
    from colossalai_b200.models import build_model, get_config

    torch.manual_seed(0)
    model = build_model(get_config("llama3.2-1b")).to(torch.bfloat16).cuda().eval()
    vocab = model.cfg.vocab_size
    g = torch.Generator().manual_seed(1)
    prefix = torch.randint(3, vocab, (2048,), generator=g).tolist()
    shared = [prefix + torch.randint(3, vocab, (64,), generator=g).tolist() for _ in range(32)]
    distinct = [torch.randint(3, vocab, (2112,), generator=g).tolist() for _ in range(32)]
    gen = GenerationConfig(max_new_tokens=1)
    rows = []
    for workload, prompts in (("shared_prefix", shared), ("distinct", distinct)):
        for caching in (False, True):
            eng = InferenceEngine(model, None, InferenceConfig(
                max_batch_size=8, max_input_len=2112, max_output_len=1, block_size=BLOCK, dtype="bf16",
                use_cuda_graph=False, ignore_eos=True, enable_prefix_caching=caching))
            eng.generate(prompts_token_ids=[[5, 6, 7], [8, 9]], generation_config=gen)       # warm-up
            torch.cuda.synchronize()
            stats0 = dict(eng.request_handler.cache_manager.prefix_cache_stats)
            t0 = time.perf_counter()
            eng.generate(prompts_token_ids=prompts, generation_config=gen)
            torch.cuda.synchronize()
            dt = time.perf_counter() - t0
            stats = eng.request_handler.cache_manager.prefix_cache_stats
            rows.append({"workload": workload, "prefix_caching": caching, "seconds": round(dt, 3),
                         "hit_tokens": stats["hit_tokens"] - stats0["hit_tokens"],
                         "queried_tokens": stats["queried_tokens"] - stats0["queried_tokens"]})
            print(json.dumps(rows[-1]), flush=True)
            del eng
            torch.cuda.empty_cache()
    return rows


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--skip-engine", action="store_true")
    args = ap.parse_args()
    assert torch.cuda.is_available(), "needs a GPU"
    result = {**gpu_info(), "kernel": kernel_rows()}
    if not args.skip_engine:
        result["engine"] = engine_rows()
    print(json.dumps(result))


if __name__ == "__main__":
    main()
