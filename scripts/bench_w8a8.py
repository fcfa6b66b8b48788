"""SmoothQuant W8A8 linears on the GPU: kernel times and one engine decode step.

(a) The Llama-3-8B linears (K -> N: qkv 4096->6144, o 4096->4096, gate_up 4096->28672, down 14336->4096) at
    M in {1, 16, 64, 256, 4096} tokens, bf16 activations, per-token activation scales, no bias.  Variants:
      native     `ops.w8a8.w8a8_linear`: the int8 per-token quantiser, then the int8 wgmma GEMM (split-K where the
                 launcher chooses it);
      gemm       the native GEMM alone on pre-quantised activations;
      torch      the previous PyTorch path of `W8A8Linear` (six quantisation ops, `torch._int_mm` for M > 16 or the
                 fp32 GEMM below, five epilogue ops);
      bf16       cuBLAS `F.linear` on the unquantised bf16 weight.
    Each timed call reads a different copy of the weight (enough copies to exceed 200 MB), so a decode-sized call reads
    its weight from HBM rather than the 50 MB L2, as it would in a model.  Share of peak: the least time the op needs
    (the larger of bytes / 3.35 TB/s and 2MNK / 1,979 int8 TOPS, or 989 bf16 TFLOP/s for bf16) over the measured time;
    the bound names which of the two it is.  Bytes: weight + bf16 activation + bf16 output.  At every shape, the native
    output must equal the PyTorch epilogue on the exact int32 product bit for bit; whether the previous path (whose
    fp32 GEMM at M <= 16 may round) gave the same bytes is reported.
(b) ms per decode step of a `llama3.2-1b`-shaped model (random weights; SmoothQuant on random calibration batches), batch
    16, prompts of 1024 tokens, CUDA graphs on, through `InferenceEngine`: W8A8 native, W8A8 on the previous path, bf16.
    A step = (time of generating 40 tokens - time of generating 8) / 32.

Kernel times are taken two ways: eager calls back to back (`us`, which at decode sizes measures the host-side cost of
a call as much as the GPU), and the same calls captured in a CUDA graph and replayed (`graph_us`, device time, as in
the engine's decode graphs).  Everything is measured twice in the same process; both runs and their spread are
reported.  Prints one JSON line.
Needs a GPU.
"""
import argparse
import contextlib
import copy
import json
import subprocess
import time

import torch
import torch.nn.functional as F

SHAPES = {"qkv": (4096, 6144), "o": (4096, 4096), "gate_up": (4096, 28672), "down": (14336, 4096)}
MS = [1, 16, 64, 256, 4096]
HBM_BPS, INT8_OPS, BF16_FLOPS = 3.35e12, 1979e12, 989e12


def gpu_info():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
        name, power, clock = (s.strip() for s in out.split(","))
    except (OSError, IndexError, ValueError, subprocess.SubprocessError):
        name, power, clock = torch.cuda.get_device_name(), "unknown", "unknown"
    return {"gpu": name, "power_limit": power, "max_sm_clock": clock}


def timeit(fn, n_variants, min_window_s=0.2):
    """µs per call; fn(i) uses weight copy i % n_variants."""
    for i in range(max(3, n_variants)):
        fn(i)
    torch.cuda.synchronize()
    s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    s.record()
    for i in range(5):
        fn(i)
    e.record()
    torch.cuda.synchronize()
    iters = max(20, min(2000, int(min_window_s * 1e3 / max(s.elapsed_time(e) / 5, 1e-3))))
    s.record()
    for i in range(iters):
        fn(i)
    e.record()
    torch.cuda.synchronize()
    return s.elapsed_time(e) / iters * 1e3


def graph_time(fn, n_variants, min_window_s=0.2):
    """Device µs per call: max(8, n_variants) calls captured in one CUDA graph, replayed (no host overhead)."""
    calls = max(8, n_variants)
    for i in range(calls):
        fn(i)
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        for i in range(calls):
            fn(i)
    for _ in range(3):
        g.replay()
    torch.cuda.synchronize()
    s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    s.record()
    g.replay()
    e.record()
    torch.cuda.synchronize()
    iters = max(10, min(1000, int(min_window_s * 1e3 / max(s.elapsed_time(e), 1e-3))))
    s.record()
    for _ in range(iters):
        g.replay()
    e.record()
    torch.cuda.synchronize()
    return s.elapsed_time(e) / (iters * calls) * 1e3


@contextlib.contextmanager
def previous_path():
    """W8A8Linear takes its PyTorch path (everything else stays native)."""
    from colossalai_b200.ops import w8a8

    orig = w8a8.supported
    w8a8.supported = lambda *a, **k: False
    try:
        yield
    finally:
        w8a8.supported = orig


def exact_reference(x, w_q, w_scale):
    from colossalai_b200.quantization.smoothquant import quantize_activation_per_token

    xq, sx = quantize_activation_per_token(x)
    M, N = xq.shape[0], w_q.shape[0]
    ap = torch.zeros(max(24, (M + 7) // 8 * 8), xq.shape[1], dtype=torch.int8, device=x.device)
    ap[:M] = xq
    acc = torch._int_mm(ap, w_q.t().contiguous())[:M]
    return (acc.float() * sx * w_scale[None, :]).to(x.dtype)


def kernel_times():
    from colossalai_b200.kernel import loader
    from colossalai_b200.ops import w8a8
    from colossalai_b200.quantization.smoothquant import W8A8Linear

    rows = []
    for name, (K, N) in SHAPES.items():
        torch.manual_seed(0)
        copies = max(1, -(-200_000_000 // (N * K)))
        lins, w16 = [], []
        for _ in range(copies):
            lin = torch.nn.Linear(K, N, bias=False, device="cuda", dtype=torch.bfloat16)
            torch.nn.init.normal_(lin.weight, 0, 0.02)
            lins.append(W8A8Linear.from_float(lin))
            w16.append(lin.weight.detach())
        w16 = w16[:max(1, -(-200_000_000 // (2 * N * K)))]
        for M in MS:
            x = torch.randn(M, K, device="cuda", dtype=torch.bfloat16)
            x[:, ::97] *= 20
            with torch.no_grad():
                xq, sx = w8a8.quantize_per_token(x)
                loader.launch_counter.reset()
                got = lins[0](x)
                branch = [k for k in loader.launch_counter.by_name if k.startswith("gemm_w8a8")]
                want = exact_reference(x, lins[0].weight, lins[0].weight_scale)
                assert torch.equal(got.view(torch.int16), want.view(torch.int16)), f"{name} M={M}: native != exact"
                with previous_path():
                    old = lins[0](x)
                old_equal = torch.equal(got.view(torch.int16), old.view(torch.int16))
                n = len(lins)
                variants = {
                    "native": (lambda i: lins[i % n](x), n),
                    "gemm": (lambda i: w8a8._gemm(xq, sx, True, lins[i % n].weight, lins[i % n].weight_scale, None,
                                                  torch.bfloat16), n),
                    "bf16": (lambda i: F.linear(x, w16[i % len(w16)]), len(w16)),
                }
                times = {k: timeit(fn, nv) for k, (fn, nv) in variants.items()}
                with previous_path():
                    times["torch"] = timeit(lambda i: lins[i % n](x), n)
                graph = {k: graph_time(fn, nv) for k, (fn, nv) in variants.items()}
                with previous_path():
                    graph["torch"] = graph_time(lambda i: lins[i % n](x), n)
            row = {"linear": name, "K": K, "N": N, "M": M, "branch": branch[0] if branch else None,
                   "old_path_bitwise_equal": old_equal}
            for k, us in times.items():
                wbytes = N * K * (2 if k == "bf16" else 1)
                t_bw = (wbytes + 2 * M * K + 2 * M * N) / HBM_BPS
                t_ops = 2 * M * N * K / (BF16_FLOPS if k == "bf16" else INT8_OPS)
                row[k] = {"us": round(us, 2), "share": round(max(t_bw, t_ops) / (us * 1e-6), 4),
                          "bound": "hbm" if t_bw >= t_ops else ("bf16_tflops" if k == "bf16" else "int8_tops")}
            row["graph_us"] = {k: round(v, 2) for k, v in graph.items()}
            rows.append(row)
        del lins, w16
        torch.cuda.empty_cache()
    return rows


def engine_steps():
    from colossalai_b200.inference import InferenceConfig, InferenceEngine
    from colossalai_b200.inference.config import GenerationConfig
    from colossalai_b200.models import build_model, get_config
    from colossalai_b200.quantization.smoothquant import smooth_and_quantize_model

    torch.manual_seed(0)
    with torch.device("cuda"):
        bf16 = build_model(get_config("llama3.2-1b")).to(torch.bfloat16).eval()
    q = copy.deepcopy(bf16)
    vocab = bf16.cfg.vocab_size
    smooth_and_quantize_model(q, [dict(input_ids=torch.randint(0, vocab, (2, 256), device="cuda")) for _ in range(2)])
    B, ctx = 16, 1024
    prompts = torch.randint(0, vocab, (B, ctx)).tolist()
    kw = dict(max_batch_size=B, max_input_len=ctx, max_output_len=48, block_size=16, dtype="bf16", ignore_eos=True,
              use_cuda_graph=True)
    out = {}
    for label, model, ctxm in (("w8a8_native", q, contextlib.nullcontext), ("w8a8_previous", q, previous_path),
                               ("bf16", bf16, contextlib.nullcontext)):
        with ctxm():
            eng = InferenceEngine(model, None, InferenceConfig(**kw))

            def gen(n):
                torch.cuda.synchronize()
                t = time.perf_counter()
                eng.generate(prompts_token_ids=prompts, return_token_ids=True,
                             generation_config=GenerationConfig(max_new_tokens=n))
                torch.cuda.synchronize()
                return time.perf_counter() - t

            gen(4)
            out[label] = round((gen(40) - gen(8)) / 32 * 1e3, 3)
            del eng
            torch.cuda.empty_cache()
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--runs", type=int, default=2)
    ap.add_argument("--skip-engine", action="store_true")
    args = ap.parse_args()
    assert torch.cuda.is_available(), "bench_w8a8.py measures on the GPU"
    import colossalai_b200  # noqa: F401

    result = {**gpu_info(), "runs": []}
    for _ in range(args.runs):
        run = {"kernels": kernel_times()}
        if not args.skip_engine:
            run["decode_step_ms"] = engine_steps()
        result["runs"].append(run)
    if args.runs > 1:
        spread = []
        for rows in zip(*(r["kernels"] for r in result["runs"])):
            for k in ("native", "gemm", "torch", "bf16"):
                us = [r[k]["us"] for r in rows]
                spread.append(max(us) / min(us) - 1)
        result["kernel_time_spread_max"] = round(max(spread), 4)
        result["kernel_time_spread_median"] = round(sorted(spread)[len(spread) // 2], 4)
    print(json.dumps(result))


if __name__ == "__main__":
    main()
