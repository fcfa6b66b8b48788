"""Device-timed GEMM microbenchmark: our wgmma kernel vs cuBLAS (torch.matmul) on Llama-3 shapes.
Usage (on the GPU box): python tests/bench_gemm.py > gpurun_out/gemm_bench.json"""
import json
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from colossalai_b200.ops import gemm_native as g  # noqa: E402


def timeit(fn, iters=20, warmup=5):
    flush = torch.empty(256 << 20, dtype=torch.uint8, device="cuda")
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    ts = []
    for _ in range(iters):
        flush.zero_()                       # flush the 50 MB L2 between timed iterations
        s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        s.record()
        fn()
        e.record()
        torch.cuda.synchronize()
        ts.append(s.elapsed_time(e))
    ts.sort()
    return ts[len(ts) // 2]


def main():
    peaks = {}
    try:
        peaks = json.load(open(os.path.join(os.path.dirname(__file__), "..", "MEASURED_PEAKS.json")))
    except Exception:
        pass
    peak = peaks.get("bf16_tflops", 1590.0)
    M0 = int(os.environ.get("CB200_GEMM_BENCH_M", "8192"))     # tokens per micro-batch (4096 = the N=1 bench step)
    shapes = [(M0, 6144, 4096, "qkv fwd"), (M0, 4096, 4096, "o_proj fwd"), (M0, 28672, 4096, "gate_up fwd"),
              (M0, 4096, 14336, "down fwd"), (4096, 128256, 4096, "lm_head fwd"), (8192, 8192, 8192, "square")]
    out = []
    for M, N, K, name in shapes:
        x = torch.randn(M, K, device="cuda", dtype=torch.bfloat16)
        w = torch.randn(N, K, device="cuda", dtype=torch.bfloat16)
        dy = torch.randn(M, N, device="cuda", dtype=torch.bfloat16)
        fl = 2.0 * M * N * K
        row = {"shape": [M, N, K], "name": name}
        for label, ours, ref in [
            ("nt", lambda: g.gemm_nt(x, w), lambda: torch.nn.functional.linear(x, w)),
            ("nn", lambda: g.gemm_nn(dy, w), lambda: dy @ w),
            ("tn", lambda: g.gemm_tn(dy, x), lambda: dy.t() @ x),
        ]:
            t_o, t_r = timeit(ours), timeit(ref)
            row[label] = {"ours_ms": t_o, "cublas_ms": t_r, "ours_tflops": fl / t_o / 1e9, "cublas_tflops": fl / t_r / 1e9,
                          "frac_of_measured_peak": fl / t_o / 1e9 / peak}
        out.append(row)
        print(json.dumps(row), flush=True)


if __name__ == "__main__":
    main()
