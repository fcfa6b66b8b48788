"""Expert-parallel MoE layer, device-timed (max over ranks): fused NVLink dispatch/combine + wgmma grouped GEMM vs the
NCCL all-to-all composition (+ library grouped GEMM), forward + backward, 8192 tokens per rank.

    python -m torch.distributed.run --nproc-per-node N scripts/bench_moe_ep.py      (BASELINE.json config 4)
"""
import json
import os
import sys

import torch
import torch.distributed as dist

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import colossalai_b200  # noqa: E402
from colossalai_b200.moe import dispatch_combine as dc  # noqa: E402
from colossalai_b200.moe.grouped_gemm import grouped_linear  # noqa: E402
from colossalai_b200 import ops  # noqa: E402


def timed(fn, group, iters=5, warmup=3):
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    dist.barrier(group=group)
    s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    s.record()
    for _ in range(iters):
        fn()
    e.record()
    torch.cuda.synchronize()
    t = torch.tensor([s.elapsed_time(e) / iters], device="cuda")
    dist.all_reduce(t, op=dist.ReduceOp.MAX, group=group)
    return t.item()


def main():
    # receive buffers of 2x the balanced load instead of the worst case (every token of every rank to one rank); an
    # overflow raises
    os.environ.setdefault("CB200_EP_CAPACITY_FACTOR", "2")
    colossalai_b200.launch_from_torch(verbose=False)
    rank, world = dist.get_rank(), dist.get_world_size()
    group = dist.group.WORLD
    T = int(os.environ.get("CB200_MOE_TOKENS", "8192"))
    models = [("mixtral-8x7b", 8, 2, 4096, 14336), ("deepseek-moe-16b-class", 64, 6, 2048, 1408)]
    for name, E, K, H, F in models:
        if E % world:
            continue
        n_local = E // world
        torch.manual_seed(7 + rank)
        w_up = (torch.randn(n_local, 2 * F, H, device="cuda") * 0.02).bfloat16().requires_grad_()
        w_down = (torch.randn(n_local, H, F, device="cuda") * 0.02).bfloat16().requires_grad_()
        x = torch.randn(T, H, device="cuda").bfloat16().requires_grad_()
        logits = torch.randn(T, E, device="cuda")
        tw, ti = logits.softmax(-1).topk(K, -1)
        tw = (tw / tw.sum(-1, keepdim=True)).bfloat16()
        dy = torch.randn(T, H, device="cuda").bfloat16()

        def experts(rows, counts):
            h = grouped_linear(rows, w_up, counts)
            h = ops.glu(h, "silu", valid_rows=counts.sum())
            return grouped_linear(h, w_down, counts)

        def identity(rows, counts):
            return rows

        res = {"model": name, "ep": world, "tokens_per_rank": T, "experts": E, "top_k": K, "hidden": H, "ffn": F}
        for backend, gg in (("fused", "native"), ("nccl", "lib")):
            os.environ["CB200_GROUPED_GEMM"] = gg
            dc.set_moe_backend(backend)

            def layer(fn=experts):
                y = dc.moe_forward(x, tw, ti, fn, E, group)
                y.backward(dy)
                x.grad = w_up.grad = w_down.grad = None

            try:
                res[f"{backend}_a2a_only_ms"] = timed(lambda: layer(identity), group)
                res[f"{backend}_layer_ms"] = timed(layer, group)
            except Exception as e:      # keep the other arm's numbers
                res[f"{backend}_error"] = f"{type(e).__name__}: {str(e)[:200]}"
        # mixed: fused dispatch/combine with the library grouped GEMM (isolates the GEMM's contribution)
        os.environ["CB200_GROUPED_GEMM"] = "lib"
        dc.set_moe_backend("fused")
        try:
            res["fused_a2a_lib_gemm_layer_ms"] = timed(lambda: layer(), group)
        except Exception as e:
            res["mixed_error"] = str(e)[:200]
        # roofline: expert FLOPs (3 GEMMs fwd, x3 for fwd+bwd) at the measured cuBLAS peak vs dispatch+combine bytes
        flops = 3 * 3 * 2.0 * T * K * H * F
        a2a_bytes = 4 * T * K * H * 2 * (world - 1) / world       # dispatch + combine, forward + backward
        res["roofline_ms"] = max(flops / 1676.7e9, a2a_bytes / 770e6)
        if "fused_layer_ms" in res:
            res["fused_frac_of_roofline"] = res["roofline_ms"] / res["fused_layer_ms"]
            res["fused_tflops_per_gpu"] = flops / res["fused_layer_ms"] / 1e9
        if rank == 0:
            print("MOE_EP " + json.dumps(res), flush=True)
        del w_up, w_down
        torch.cuda.empty_cache()
    dist.barrier()
    dist.destroy_process_group()


if __name__ == "__main__":
    main()
