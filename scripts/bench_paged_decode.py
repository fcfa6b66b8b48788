"""Paged decode attention with a bf16 vs an fp8 (e5m2) KV cache on the Llama-3-8B decode shape (Hq 32, Hkv 8, D 128,
block 16).  Decode is bound by HBM bandwidth, so the figure of merit is bytes read per second: the cache K+V at its
element size plus q, the output and the split-KV partials (written and read back).  The bf16 cache holds the decoded
fp8 cache, so both runs compute the same values and their outputs must be bitwise equal."""
import json
import subprocess

import torch

from colossalai_b200.ops import inference as iops

HBM_BYTES_PER_S = 3.35e12          # H100 SXM data sheet (HBM3)
HQ, HKV, D, BS = 32, 8, 128, 16


def gpu_info():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
        name, power, clock = (s.strip() for s in out.split(","))
    except (OSError, IndexError, ValueError, subprocess.SubprocessError):
        name, power, clock = torch.cuda.get_device_name(), "unknown", "unknown"
    return {"gpu": name, "power_limit": power, "max_sm_clock": clock}


def timeit(fn, min_window_s=0.3):
    for _ in range(10):
        fn()
    torch.cuda.synchronize()
    s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    s.record()
    for _ in range(10):
        fn()
    e.record()
    torch.cuda.synchronize()
    iters = max(20, min(5000, int(min_window_s * 1e3 / max(s.elapsed_time(e) / 10, 1e-3))))
    s.record()
    for _ in range(iters):
        fn()
    e.record()
    torch.cuda.synchronize()
    return s.elapsed_time(e) / iters * 1e3       # microseconds per call


def main():
    assert torch.cuda.is_available(), "bench_paged_decode.py measures the GPU kernels and needs a GPU"
    print("GPU " + json.dumps(gpu_info()), flush=True)
    dev = torch.device("cuda")
    sms = iops.sm_count(torch.cuda.current_device())
    for B in (1, 16, 64):
        for L in (1024, 4096, 16384):
            torch.manual_seed(0)
            nblk = L // BS
            tables = torch.randperm(B * nblk, device=dev).to(torch.int32).view(B, nblk).contiguous()
            kc8 = torch.randn(B * nblk, BS, HKV, D, device=dev, dtype=torch.bfloat16).to(torch.float8_e5m2)
            vc8 = torch.randn(B * nblk, BS, HKV, D, device=dev, dtype=torch.bfloat16).to(torch.float8_e5m2)
            kc16, vc16 = kc8.to(torch.bfloat16), vc8.to(torch.bfloat16)
            kc8, vc8 = kc8.view(torch.uint8), vc8.view(torch.uint8)
            lens = torch.full((B,), L, device=dev, dtype=torch.int32)
            q = torch.randn(B, HQ, D, device=dev, dtype=torch.bfloat16)
            splits, _ = iops.decode_splits(B, HKV, L, sms)
            other = 2 * B * HQ * D * 2 + 2 * B * HQ * splits * (D + 2) * 4     # q + out, partials written and read
            same = torch.equal(iops.paged_decode_attention(q, kc8, vc8, tables, lens),
                               iops.paged_decode_attention(q, kc16, vc16, tables, lens))
            row = {"batch": B, "context": L, "splits": splits, "bitwise_equal": same}
            for name, kc, vc in (("bf16", kc16, vc16), ("fp8", kc8, vc8)):
                us = timeit(lambda: iops.paged_decode_attention(q, kc, vc, tables, lens))
                nbytes = 2 * B * L * HKV * D * kc.element_size() + other
                row[name] = {"us": round(us, 2), "bytes": nbytes, "GB_per_s": round(nbytes / us / 1e3, 1),
                             "hbm_share": round(nbytes / us / 1e-6 / HBM_BYTES_PER_S, 3)}
            row["fp8_speedup"] = round(row["bf16"]["us"] / row["fp8"]["us"], 3)
            print("PAGED_DECODE " + json.dumps(row), flush=True)
            del kc8, vc8, kc16, vc16


if __name__ == "__main__":
    main()
