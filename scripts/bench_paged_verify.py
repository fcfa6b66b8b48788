"""Speculative verification attention on the Llama-3-8B shape (Hq 32, Hkv 8, D 128, block 16): one multi-query
`paged_decode_attention(..., q_len=n)` call against the per-position loop it replaces (n single-query decode calls,
each with its own sequence lengths).  Both are timed at every shape and must give bitwise equal outputs.  Bytes are
counted as in bench_paged_decode.py - the cache K+V once at its element size, plus q, the output and the split-KV
partials of all n query rows - so the loop's rate is the useful rate, not the bytes it actually moves (n times the
cache)."""
import json

import torch

from bench_paged_decode import BS, D, HBM_BYTES_PER_S, HKV, HQ, gpu_info, timeit
from colossalai_b200.ops import inference as iops


def per_position(q, kc, vc, tables, lens, q_len):
    n = lens.numel()
    qs = q.view(n, q_len, HQ, D)
    outs = [iops.paged_decode_attention(qs[:, j], kc, vc, tables, lens - (q_len - 1 - j)) for j in range(q_len)]
    return torch.stack(outs, 1).view(n * q_len, HQ, D)


def main():
    assert torch.cuda.is_available(), "bench_paged_verify.py measures the GPU kernels and needs a GPU"
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
            caches = {"bf16": (kc8.to(torch.bfloat16), vc8.to(torch.bfloat16)),
                      "fp8": (kc8.view(torch.uint8), vc8.view(torch.uint8))}
            lens = torch.full((B,), L, device=dev, dtype=torch.int32)
            splits, _ = iops.decode_splits(B, HKV, L, sms)
            for name, (kc, vc) in caches.items():
                for q_len in (1, 2, 4, 6):
                    q = torch.randn(B * q_len, HQ, D, device=dev, dtype=torch.bfloat16)
                    same = torch.equal(iops.paged_decode_attention(q, kc, vc, tables, lens, q_len=q_len),
                                       per_position(q, kc, vc, tables, lens, q_len))
                    rows = B * q_len
                    nbytes = (2 * B * L * HKV * D * kc.element_size() + 2 * rows * HQ * D * 2
                              + 2 * rows * HQ * splits * (D + 2) * 4)
                    row = {"batch": B, "context": L, "cache": name, "q_len": q_len, "splits": splits,
                           "bitwise_equal": same, "bytes": nbytes}
                    for impl, fn in (("native", lambda: iops.paged_decode_attention(q, kc, vc, tables, lens,
                                                                                    q_len=q_len)),
                                     ("loop", lambda: per_position(q, kc, vc, tables, lens, q_len))):
                        us = timeit(fn)
                        row[impl] = {"us": round(us, 2), "GB_per_s": round(nbytes / us / 1e3, 1),
                                     "hbm_share": round(nbytes / us / 1e-6 / HBM_BYTES_PER_S, 3)}
                    row["loop_over_native"] = round(row["loop"]["us"] / row["native"]["us"], 3)
                    print("PAGED_VERIFY " + json.dumps(row), flush=True)
            del kc8, vc8, caches


if __name__ == "__main__":
    main()
