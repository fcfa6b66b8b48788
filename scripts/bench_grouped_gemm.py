"""Grouped expert GEMMs: our wgmma kernel vs the library `torch._grouped_mm` vs a per-expert cuBLAS loop, on the
expert-MLP shapes of Mixtral-8x7B and a DeepSeekMoE-16B-class layer (tokens per rank 8192, balanced routing)."""
import json
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from colossalai_b200.moe import grouped_gemm as gg  # noqa: E402


def timeit(fn, iters=10):
    for _ in range(3):
        fn()
    torch.cuda.synchronize()
    s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    s.record()
    for _ in range(iters):
        fn()
    e.record()
    torch.cuda.synchronize()
    return s.elapsed_time(e) / iters


def main():
    cases = [("mixtral-8x7b gate_up (ep=1: 8 experts, top-2 of 8192 tokens)", 8, 16384, 4096, 28672),
             ("mixtral-8x7b down", 8, 16384, 14336, 4096),
             ("deepseek-moe-16b gate_up (64 experts, top-6 of 8192 tokens)", 64, 49152, 2048, 2816),
             ("deepseek-moe-16b down", 64, 49152, 1408, 2048)]
    for name, E, rows, K, N in cases:
        torch.manual_seed(0)
        # mildly unbalanced routing
        p = torch.rand(E) + 0.5
        counts = torch.floor(p / p.sum() * rows).long()
        counts[0] += rows - counts.sum()
        c = counts.cuda()
        x = torch.randn(rows, K, device="cuda", dtype=torch.bfloat16)
        w = torch.randn(E, N, K, device="cuda", dtype=torch.bfloat16) * 0.02
        offs = torch.cumsum(c, 0).int()
        fl = 2.0 * rows * K * N
        os.environ["CB200_GROUPED_GEMM"] = "native"
        t_nat = timeit(lambda: gg.grouped_linear(x, w, c))
        t_lib = timeit(lambda: torch._grouped_mm(x, w.transpose(-2, -1), offs=offs)) if hasattr(torch, "_grouped_mm") else None
        cl = counts.tolist()

        def loop():
            s = 0
            for e, n in enumerate(cl):
                torch.nn.functional.linear(x[s:s + n], w[e])
                s += n
        t_loop = timeit(loop)
        row = {"case": name, "E": E, "rows": rows, "K": K, "N": N, "native_ms": t_nat, "native_tflops": fl / t_nat / 1e9,
               "grouped_mm_ms": t_lib, "grouped_mm_tflops": fl / t_lib / 1e9 if t_lib else None,
               "cublas_loop_ms": t_loop, "cublas_loop_tflops": fl / t_loop / 1e9}
        # backward (dgrad + wgrad) through autograd
        if N % 128 == 0:
            xg = x.clone().requires_grad_(True)
            wg = w.clone().requires_grad_(True)
            dy = torch.randn(rows, N, device="cuda", dtype=torch.bfloat16)

            def fb():
                y = gg.grouped_linear(xg, wg, c)
                y.backward(dy)
                xg.grad = wg.grad = None
            try:
                row["native_fwd_bwd_ms"] = timeit(fb, 5)
                row["native_fwd_bwd_tflops"] = 3 * fl / row["native_fwd_bwd_ms"] / 1e9
            except Exception as e:
                row["native_fwd_bwd_error"] = f"{type(e).__name__}: {str(e)[:160]}"
            # the three GEMMs separately, on a 128-aligned group layout (what the fused EP dispatch produces)
            ca = (counts // 128 * 128)
            ca[0] += rows - ca.sum()
            offa = torch.cumsum(ca.cuda(), 0).int()
            try:
                row["native_dgrad_ms"] = timeit(lambda: gg._native_fwd(dy, w, offa, False))
                row["native_wgrad_ms"] = timeit(lambda: gg._native_wgrad(dy, x, offa, E, torch.bfloat16))
                row["native_wgrad_tflops"] = fl / row["native_wgrad_ms"] / 1e9
                row["native_wgrad_unaligned_ms"] = timeit(lambda: gg._GroupedLinearNative.backward(
                    type("C", (), {"saved_tensors": (x, w, c, offs), "aligned": False,
                                   "needs_input_grad": (False, True, False, False)})(), dy))
            except Exception as e:
                row["native_split_error"] = f"{type(e).__name__}: {str(e)[:160]}"
            if hasattr(torch, "_grouped_mm"):
                def fb_lib():
                    y = torch._grouped_mm(xg, wg.transpose(-2, -1), offs=offs)
                    y.backward(dy)
                    xg.grad = wg.grad = None
                try:
                    row["grouped_mm_fwd_bwd_ms"] = timeit(fb_lib, 5)
                except Exception as e:
                    row["grouped_mm_fwd_bwd_error"] = f"{type(e).__name__}: {str(e)[:160]}"
        print("GROUPED_GEMM " + json.dumps(row), flush=True)


if __name__ == "__main__":
    main()
