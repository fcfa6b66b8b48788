"""QLoRA on packed 4-bit base weights: kernel times and one optimizer step.

(a) M = 4096 tokens, bf16, nf4 with block 64, on the Llama-3.2-1B linears (qkv 2048->3072, o 2048->2048, gate_up
    2048->16384, down 8192->2048) and the Llama-3-8B linears (4096->6144, 4096->4096, 4096->28672, 14336->4096).  For
    each shape, the forward (NT: x W^T) and the input gradient (NN: dy W) of three variants:
      native    `ops/wq_gemm.py`: `cb_wq_dequantize` into a scratch bf16 weight, then the dense wgmma GEMM;
      torch     the PyTorch dequantize (indexing ops) followed by cuBLAS;
      bf16      cuBLAS on the unquantised bf16 weight.
    TFLOP/s = 2 M N K / time.
(b) One QLoRA optimizer step of the `llama3.2-1b` preset at sequence 4096 (batch 1), LoRA r 16 on qkv_proj, o_proj,
    gate_up_proj and down_proj, through TorchDDPPlugin: nf4 base weights against a bf16 base (LoRA), step time and peak
    memory.

Prints one JSON line.  Needs a GPU.
"""
import gc
import json
import subprocess
import time

import torch
import torch.nn as nn
import torch.nn.functional as F

M = 4096
SHAPES = {
    "llama3.2-1b": {"qkv": (2048, 3072), "o": (2048, 2048), "gate_up": (2048, 16384), "down": (8192, 2048)},
    "llama3-8b": {"qkv": (4096, 6144), "o": (4096, 4096), "gate_up": (4096, 28672), "down": (14336, 4096)},
}


def gpu_info():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
        name, power, clock = (s.strip() for s in out.split(","))
    except (OSError, IndexError, ValueError, subprocess.SubprocessError):
        name, power, clock = torch.cuda.get_device_name(), "unknown", "unknown"
    return {"gpu": name, "power_limit": power, "max_sm_clock": clock}


def timeit(fn, min_window_s=0.2):
    for _ in range(3):
        fn()
    torch.cuda.synchronize()
    s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    s.record()
    for _ in range(3):
        fn()
    e.record()
    torch.cuda.synchronize()
    iters = max(10, min(500, int(min_window_s * 1e3 / max(s.elapsed_time(e) / 3, 1e-3))))
    s.record()
    for _ in range(iters):
        fn()
    e.record()
    torch.cuda.synchronize()
    return s.elapsed_time(e) / iters * 1e3       # microseconds per call


def kernel_times():
    from colossalai_b200.ops import wq_gemm
    from colossalai_b200.quantization.bnb import Linear4bit

    rows = []
    for model, shapes in SHAPES.items():
        for name, (K, N) in shapes.items():
            torch.manual_seed(0)
            lin = nn.Linear(K, N, bias=False, device="cuda")
            with torch.no_grad():
                lin.weight.normal_(0, 0.02)
            w16 = lin.weight.detach().to(torch.bfloat16)
            layer = Linear4bit(lin, torch.bfloat16, "nf4", 64)
            del lin
            x = torch.randn(M, K, device="cuda", dtype=torch.bfloat16)
            dy = torch.randn(M, N, device="cuda", dtype=torch.bfloat16)
            variants = {
                "native": (lambda: wq_gemm.wq_linear(x, layer), lambda: wq_gemm.wq_matmul_nn(dy, layer)),
                "torch": (lambda: F.linear(x, layer.dequantize_reference()),
                          lambda: dy @ layer.dequantize_reference()),
                "bf16": (lambda: F.linear(x, w16), lambda: dy @ w16),
            }
            flop = 2.0 * M * N * K
            row = {"model": model, "linear": name, "K": K, "N": N}
            for v, (fwd, bwd) in variants.items():
                for tag, fn in (("fwd", fwd), ("dgrad", bwd)):
                    us = timeit(fn)
                    row[f"{v}_{tag}_us"] = round(us, 1)
                    row[f"{v}_{tag}_tflops"] = round(flop / us / 1e6, 1)
            rows.append(row)
            print("ROW " + json.dumps(row), flush=True)
            del layer, w16, x, dy, variants
            torch.cuda.empty_cache()
    return rows


def qlora_step(quantized: bool, seq=4096, steps=5, warmup=2):
    from colossalai_b200.booster import Booster
    from colossalai_b200.booster.lora import LoraConfig
    from colossalai_b200.booster.plugin import TorchDDPPlugin
    from colossalai_b200.models import build_model
    from colossalai_b200.quantization import BnbQuantizationConfig

    torch.manual_seed(0)
    model = build_model("llama3.2-1b").to(device="cuda", dtype=torch.bfloat16)
    booster = Booster(plugin=TorchDDPPlugin())
    lcfg = LoraConfig(r=16, lora_alpha=32, target_modules=["qkv_proj", "o_proj", "gate_up_proj", "down_proj"])
    qcfg = BnbQuantizationConfig(load_in_4bit=True, bnb_4bit_quant_type="nf4", bnb_4bit_compute_dtype="bf16") \
        if quantized else None
    model = booster.enable_lora(model, lora_config=lcfg, bnb_quantization_config=qcfg)
    opt = torch.optim.AdamW([p for p in model.parameters() if p.requires_grad], lr=1e-4)
    model, opt, *_ = booster.boost(model, opt)
    ids = torch.randint(0, 128256, (1, seq), device="cuda")
    gc.collect()
    torch.cuda.empty_cache()
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    times, losses = [], []
    for i in range(warmup + steps):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        loss = model(input_ids=ids, labels=ids)["loss"]
        booster.backward(loss, opt)
        opt.step()
        opt.zero_grad()
        torch.cuda.synchronize()
        if i >= warmup:
            times.append(time.perf_counter() - t0)
        losses.append(float(loss))
    res = {"step_ms": round(1e3 * sum(times) / len(times), 1), "step_ms_min": round(1e3 * min(times), 1),
           "peak_mem_gib": round(torch.cuda.max_memory_allocated() / 2**30, 2),
           "losses": [round(l, 4) for l in losses]}
    del model, opt, booster
    gc.collect()
    torch.cuda.empty_cache()
    return res


def main():
    import colossalai_b200
    from colossalai_b200.testing import free_port

    assert torch.cuda.is_available(), "bench_qlora.py measures GPU kernels and needs a GPU"
    info = gpu_info()
    print("GPU " + json.dumps(info), flush=True)
    rows = kernel_times()
    if not torch.distributed.is_initialized():
        colossalai_b200.launch(0, 1, "127.0.0.1", free_port(), verbose=False)
    step = {"qlora_nf4": qlora_step(True), "lora_bf16": qlora_step(False)}
    print(json.dumps({**info, "M": M, "kernels": rows, "step_llama3.2-1b_seq4096": step}), flush=True)


if __name__ == "__main__":
    main()
