"""Fused compute+collective kernels vs their NCCL + cuBLAS composition (needs >= 2 GPUs on one NVLink box).
Also times both (device-timed, max over ranks) and prints one JSON line per op for profiles/."""
import json
import os

import pytest
import torch
import torch.distributed as dist

import colossalai_b200
from colossalai_b200.testing import rerun_if_address_is_in_use, spawn

pytestmark = pytest.mark.gpu


def _time(fn, iters=10, warmup=3):
    for _ in range(warmup):
        fn()
    dist.barrier()
    torch.cuda.synchronize()
    s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    s.record()
    for _ in range(iters):
        fn()
    e.record()
    torch.cuda.synchronize()
    t = torch.tensor([s.elapsed_time(e) / iters], device="cuda")
    dist.all_reduce(t, op=dist.ReduceOp.MAX)
    return t.item()


def _worker(rank, world_size, port, timing=False):
    colossalai_b200.launch(rank, world_size, "127.0.0.1", port, backend="nccl", verbose=False)
    from colossalai_b200.parallel import comm, fused

    group = dist.group.WORLD
    assert fused.available(group), "fused backend must be available on a multi-GPU box"
    torch.manual_seed(100 + rank)
    results = []
    shapes = [(256, 512, 768), (1024, 4096, 6144 // world_size), (2048, 4096, 4096)]
    if timing:   # Llama-3-8B per-layer shapes at this TP degree (4096 tokens per rank)
        shapes += [(4096, 4096, 28672 // world_size), (4096, 14336 // world_size, 4096)]
        if world_size >= 4:   # the skinny projections of high TP degrees (qkv: small N, o_proj: small K)
            shapes += [(4096, 4096, 6144 // world_size), (4096, 4096 // world_size, 4096)]
    for (t, K, N) in shapes:
        T = t * world_size
        x_local = (torch.randn(t, K, device="cuda") * 0.5).bfloat16()
        torch.manual_seed(7)   # identical weights on every rank
        w = (torch.randn(N, K, device="cuda") * 0.05).bfloat16()
        w2 = (torch.randn(K, N, device="cuda") * 0.05).bfloat16()
        torch.manual_seed(100 + rank + t)
        # ---- all_gather
        ref_full = comm.all_gather(x_local, 0, group)
        got_full = fused.all_gather(x_local, group)
        torch.testing.assert_close(got_full, ref_full, atol=0, rtol=0)
        # ---- AG + GEMM (both weight layouts)
        y, gathered = fused.all_gather_gemm(x_local, w, group, transpose_b=True)
        torch.testing.assert_close(gathered, ref_full, atol=0, rtol=0)
        torch.testing.assert_close(y.float(), ref_full.float() @ w.float().t(), atol=0.08, rtol=2e-2)
        y2, _ = fused.all_gather_gemm(x_local, w2, group, transpose_b=False)
        torch.testing.assert_close(y2.float(), ref_full.float() @ w2.float(), atol=0.08, rtol=2e-2)
        # ---- GEMM + RS: every rank holds a different A (a K-shard of the activations)
        a = (torch.randn(T, K, device="cuda") * 0.5).bfloat16()
        ref = comm.reduce_scatter((a.float() @ w.float().t()), 0, group)
        ref2 = comm.reduce_scatter((a.float() @ w2.float()), 0, group)
        variants = ["fused"]
        for v in variants:      # fused GEMM + chunk reduction (in-switch multimem or P2P loads)
            got = fused.gemm_reduce_scatter(a, w, group, transpose_b=True, variant=v)
            torch.testing.assert_close(got.float(), ref, atol=0.15, rtol=3e-2, msg=lambda m: f"{v} NT {(t, K, N)}: {m}")
            got2 = fused.gemm_reduce_scatter(a, w2, group, transpose_b=False, variant=v)
            torch.testing.assert_close(got2.float(), ref2, atol=0.15, rtol=3e-2, msg=lambda m: f"{v} NN {(t, K, N)}: {m}")
        # autotuned dispatch (measures every candidate once on these tensors, then sticks to the fastest)
        got = fused.gemm_reduce_scatter(a, w, group, transpose_b=True)
        torch.testing.assert_close(got.float(), ref, atol=0.15, rtol=3e-2)
        # ---- GEMM + all-reduce in one kernel (in-switch reduce + multicast broadcast)
        ref_ar = (a.float() @ w.float().t())
        dist.all_reduce(ref_ar, group=group)
        got_ar = fused.gemm_all_reduce(a, w, group)
        torch.testing.assert_close(got_ar.float(), ref_ar, atol=0.15, rtol=3e-2, msg=lambda m: f"AR {(t, K, N)}: {m}")
        # block_n is accepted for interface stability (one 128 x 128 tile kernel on sm_90a)
        y1, _ = fused.all_gather_gemm(x_local, w, group, transpose_b=True, block_n=256)
        torch.testing.assert_close(y1.float(), ref_full.float() @ w.float().t(), atol=0.08, rtol=2e-2)
        got1 = fused.gemm_reduce_scatter(a, w, group, transpose_b=True, block_n=256)
        torch.testing.assert_close(got1.float(), ref, atol=0.15, rtol=3e-2)
        # repeated calls exercise buffer reuse / epoch guards
        for i in range(6):
            got = fused.gemm_reduce_scatter(a, w, group, transpose_b=True, variant=variants[i % len(variants)])
            y, _ = fused.all_gather_gemm(x_local, w, group, transpose_b=True)
            got_ar = fused.gemm_all_reduce(a, w, group)
        torch.testing.assert_close(got.float(), ref, atol=0.15, rtol=3e-2)
        torch.testing.assert_close(got_ar.float(), ref_ar, atol=0.15, rtol=3e-2)
        torch.testing.assert_close(y.float(), ref_full.float() @ w.float().t(), atol=0.08, rtol=2e-2)
        if timing and t >= 1024:
            def ar_lib():
                y_ = torch.nn.functional.linear(a, w)
                dist.all_reduce(y_, group=group)
                return y_

            r = {"world": world_size, "t_local": t, "K": K, "N": N,
                 "ag_gemm_fused_ms": _time(lambda: fused.all_gather_gemm(x_local, w, group)),
                 "ag_gemm_nccl_cublas_ms": _time(lambda: torch.nn.functional.linear(comm.all_gather(x_local, 0, group), w)),
                 "gemm_rs_fused_ms": _time(lambda: fused.gemm_reduce_scatter(a, w, group, variant="fused")),
                 "gemm_rs_nccl_cublas_ms": _time(lambda: fused.gemm_reduce_scatter(a, w, group, variant="lib")),
                 "gemm_ar_fused_ms": _time(lambda: fused.gemm_all_reduce(a, w, group)),
                 "gemm_ar_nccl_cublas_ms": _time(ar_lib)}
            r["rs_autotuned"] = fused.rs_variant(a, w, group, True)
            results.append(r)
    # ---- Ulysses layout switch (q | k | v segments in one pull kernel) vs the NCCL all_to_all composition
    B, Sl, hq, hkv, D = 2, 192, 4 * world_size, 2 * world_size, 128
    torch.manual_seed(300 + rank)
    qkv = torch.randn(B * Sl, (hq + 2 * hkv) * D, device="cuda").bfloat16().requires_grad_(True)
    got = fused.ulysses_all_to_all(qkv, group, True, B, Sl, [hq // world_size * D, hkv // world_size * D, hkv // world_size * D])
    parts = []
    for t, nh in zip(qkv.detach().split([hq * D, hkv * D, hkv * D], dim=-1), (hq, hkv, hkv)):
        r = comm.all_to_all_single(t.reshape(B, Sl, nh, D), 2, 1, group)
        parts.append(r.reshape(B * Sl * world_size, nh // world_size * D))
    ref = torch.cat(parts, -1)
    torch.testing.assert_close(got, ref, atol=0, rtol=0)
    gw = torch.randn_like(got)
    got.backward(gw)                                       # backward = the inverse switch of the gradient
    back = []
    off = 0
    for nh in (hq, hkv, hkv):
        w = nh // world_size * D
        g = comm.all_to_all_single(gw[:, off:off + w].reshape(B, Sl * world_size, nh // world_size, D), 1, 2, group)
        back.append(g.reshape(B * Sl, nh * D))
        off += w
    torch.testing.assert_close(qkv.grad, torch.cat(back, -1), atol=0, rtol=0)
    o = torch.randn(B * Sl * world_size, hq // world_size * D, device="cuda").bfloat16()
    got_o = fused.ulysses_all_to_all(o, group, False, B, Sl, [hq // world_size * D])
    ref_o = comm.all_to_all_single(o.reshape(B, Sl * world_size, hq // world_size, D), 1, 2, group).reshape(B * Sl, hq * D)
    torch.testing.assert_close(got_o, ref_o, atol=0, rtol=0)
    if timing:
        Bt, St = 1, 16384 // world_size
        x = torch.randn(Bt * St, (32 + 16) * 128, device="cuda").bfloat16()
        t_f = _time(lambda: fused.ulysses_all_to_all(x, group, True, Bt, St, [32 // world_size * 128] + [8 // world_size * 128] * 2)) \
            if 8 % world_size == 0 else None

        def lib():
            outs = []
            for t, nh in zip(x.split([32 * 128, 8 * 128, 8 * 128], dim=-1), (32, 8, 8)):
                outs.append(comm.all_to_all_single(t.reshape(Bt, St, nh, 128), 2, 1, group).reshape(Bt * St * world_size, -1))
            return torch.cat(outs, -1)
        t_n = _time(lib) if 8 % world_size == 0 else None
        results.append({"world": world_size, "op": "ulysses_qkv_a2a", "tokens_local": St, "fused_ms": t_f, "nccl_ms": t_n})
    assert fused.stats["ag_gemm"] > 0 and fused.stats["gemm_rs"] > 0, fused.stats
    if rank == 0:
        for r in results:
            print("FUSED_TIMING " + json.dumps(r), flush=True)
        print("FUSED_STATS " + json.dumps(fused.stats), flush=True)
        for r in fused.rs_tuning_log:
            print("RS_TUNING " + json.dumps(r), flush=True)
    dist.barrier()
    dist.destroy_process_group()


@pytest.mark.dist
@rerun_if_address_is_in_use()
def test_fused_comm_kernels():
    n = torch.cuda.device_count()
    if n < 2:
        pytest.skip("needs >= 2 GPUs")
    spawn(_worker, 2)


if __name__ == "__main__":
    n = int(os.environ.get("NGPU", torch.cuda.device_count()))
    spawn(_worker, n, timing=True)
