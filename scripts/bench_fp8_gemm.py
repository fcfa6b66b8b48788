"""fp8 wgmma GEMM vs cuBLASLt `_scaled_mm` vs bf16 cuBLAS on the Llama-3-8B forward shapes (CUDA events, L2 flushed
by cycling through distinct operand buffers)."""
import json

import torch

from colossalai_b200.ops import gemm_native


def timeit(fn, iters=20):
    for _ in range(3):
        fn(0)
    torch.cuda.synchronize()
    s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    s.record()
    for i in range(iters):
        fn(i)
    e.record()
    torch.cuda.synchronize()
    return s.elapsed_time(e) / iters


def main():
    for (M, N, K) in [(4096, 6144, 4096), (4096, 28672, 4096), (4096, 4096, 14336), (8192, 4096, 4096),
                      (16384, 28672, 4096)]:
        nbuf = 4
        a8 = [torch.randn(M, K, device="cuda").to(torch.float8_e4m3fn) for _ in range(nbuf)]
        b8 = [torch.randn(N, K, device="cuda").to(torch.float8_e4m3fn) for _ in range(nbuf)]
        a16 = [t.to(torch.bfloat16) for t in a8]
        b16 = [t.to(torch.bfloat16) for t in b8]
        one = torch.ones(1, device="cuda")
        out = torch.empty(M, N, device="cuda", dtype=torch.bfloat16)
        t_nat = timeit(lambda i: gemm_native.gemm_fp8_nt(a8[i % nbuf], b8[i % nbuf], one, one, torch.bfloat16, out))
        t_lt = timeit(lambda i: torch._scaled_mm(a8[i % nbuf], b8[i % nbuf].t(), scale_a=one.reshape(()),
                                                 scale_b=one.reshape(()), out_dtype=torch.bfloat16))
        t_bf = timeit(lambda i: torch.mm(a16[i % nbuf], b16[i % nbuf].t(), out=out))
        fl = 2.0 * M * N * K
        print("FP8_GEMM " + json.dumps({"M": M, "N": N, "K": K, "native_ms": t_nat, "cublaslt_fp8_ms": t_lt,
                                        "cublas_bf16_ms": t_bf, "native_tflops": fl / t_nat / 1e9,
                                        "cublaslt_fp8_tflops": fl / t_lt / 1e9, "bf16_tflops": fl / t_bf / 1e9}),
              flush=True)


if __name__ == "__main__":
    main()
