"""Zigzag ring attention == full causal attention (values and gradients).  CPU tier on gloo; GPU tier exercises the
library flash kernel with LSE + the P2P KV gather / fused reduce-scatter path (reference:
tests/test_shardformer/test_layer/test_ring_attn.py)."""
import os

import pytest
import torch
import torch.distributed as dist

import colossalai_b200
from colossalai_b200.ops.attention import attention_ref
from colossalai_b200.shardformer.layer._operation import split_batch_zigzag
from colossalai_b200.shardformer.layer.attn import RingAttention
from colossalai_b200.testing import rerun_if_address_is_in_use, spawn


def _check(device, dtype, B, S, Hq, Hkv, D, tol):
    sp, r = dist.get_world_size(), dist.get_rank()
    torch.manual_seed(0)
    q = torch.randn(B, S, Hq, D, device=device, dtype=dtype)
    k = torch.randn(B, S, Hkv, D, device=device, dtype=dtype)
    v = torch.randn(B, S, Hkv, D, device=device, dtype=dtype)
    do = torch.randn(B, S, Hq, D, device=device, dtype=dtype)
    # oracle on the full sequence (fp32)
    qf, kf, vf = (t.float().reshape(B * S, t.shape[2], D).requires_grad_() for t in (q, k, v))
    ref = attention_ref(qf, kf, vf, batch=B, causal=True)
    ref.backward(do.float().reshape(B * S, Hq, D))
    # local zigzag shards
    ql, kl, vl, dol = (split_batch_zigzag(t, dist.group.WORLD, seq_dim=1).contiguous() for t in (q, k, v, do))
    Sl = S // sp
    ql, kl, vl = (t.reshape(B * Sl, t.shape[2], D).requires_grad_() for t in (ql, kl, vl))
    out = RingAttention.attention(ql, kl, vl, dist.group.WORLD, batch=B)
    out.backward(dol.reshape(B * Sl, Hq, D))

    def shard(full, H):
        return split_batch_zigzag(full.view(B, S, H, D), dist.group.WORLD, seq_dim=1).reshape(B * Sl, H, D)

    torch.testing.assert_close(out.float(), shard(ref.detach(), Hq), **tol)
    torch.testing.assert_close(ql.grad.float(), shard(qf.grad, Hq), **tol)
    torch.testing.assert_close(kl.grad.float(), shard(kf.grad, Hkv), **tol)
    torch.testing.assert_close(vl.grad.float(), shard(vf.grad, Hkv), **tol)


def _cpu_worker(rank, world_size, port):
    colossalai_b200.launch(rank, world_size, "127.0.0.1", port, backend="gloo", verbose=False)
    _check("cpu", torch.float32, B=2, S=32, Hq=4, Hkv=2, D=16, tol=dict(rtol=1e-4, atol=1e-5))
    dist.barrier()
    dist.destroy_process_group()


@rerun_if_address_is_in_use()
def test_ring_attention_cpu():
    spawn(_cpu_worker, 2)


def _gpu_worker(rank, world_size, port):
    colossalai_b200.launch(rank, world_size, "127.0.0.1", port, backend="nccl", verbose=False)
    from colossalai_b200.parallel import fused

    from colossalai_b200.shardformer.layer import ring_attn_fused as rf

    tol = dict(rtol=3e-2, atol=3e-2)
    # fused ring attention (default on sm_90a): KV tiles TMA-loaded from the owner's HBM inside the kernel, in-kernel
    # softmax-state merge, dK / dV reduced into the owner's accumulators.  GQA, batch > 1, repeated layers (buffer reuse)
    for (B, S, Hq, Hkv) in [(2, 1024, 8, 2), (1, 2048 * world_size, 8, 2), (1, 512, 4, 4)]:
        for _ in range(2):
            _check("cuda", torch.bfloat16, B=B, S=S, Hq=Hq, Hkv=Hkv, D=128, tol=tol)
    assert rf.stats["layers_fwd"] >= 6 and rf.stats["layers_bwd"] >= 6, rf.stats
    os.environ["CB200_RING_ATTN"] = "python"
    _check("cuda", torch.bfloat16, B=2, S=1024, Hq=8, Hkv=2, D=128, tol=tol)      # P2P gather + fused RS path
    assert fused.stats.get("reduce_scatter", 0) > 0 and fused.stats["all_gather"] > 0, fused.stats
    os.environ["CB200_RING_ATTN_P2P"] = "0"
    _check("cuda", torch.bfloat16, B=1, S=2048, Hq=8, Hkv=8, D=64, tol=tol)       # NCCL ring path
    # stand-alone fused reduce-scatter, both element types
    for dt in (torch.float32, torch.bfloat16):
        torch.manual_seed(5 + rank)
        x = torch.randn(world_size * 300, 64, device="cuda").to(dt)
        ref = x.float().clone()
        dist.all_reduce(ref)
        got = fused.reduce_scatter(x, dist.group.WORLD)
        torch.testing.assert_close(got.float(), ref[rank * 300:(rank + 1) * 300], rtol=2e-2, atol=2e-2)
    dist.barrier()
    if os.environ.get("CB200_RING_ATTN_TIMING", "0") == "1":
        _timing(rank, world_size)
    if rank == 0:
        print("RING_ATTN_GPU_OK", flush=True)
    dist.destroy_process_group()


def _timing(rank, world_size):
    """Device-timed fwd+bwd of one attention layer (Llama-3-8B heads) at 16k local tokens per rank (= 128k context at
    sp = 8): fused ring vs the python ring of library flash calls (P2P gather) vs NCCL ring."""
    import json

    from colossalai_b200.shardformer.layer import ring_attn_fused as rf

    Sl = int(os.environ.get("CB200_RING_LOCAL_TOKENS", "16384"))
    Hq, Hkv, D = 32, 8, 128
    torch.manual_seed(rank)
    q, k, v = (torch.randn(Sl, h, D, device="cuda", dtype=torch.bfloat16, requires_grad=True) for h in (Hq, Hkv, Hkv))
    do = torch.randn(Sl, Hq, D, device="cuda", dtype=torch.bfloat16)

    def run():
        out = RingAttention.attention(q, k, v, dist.group.WORLD, batch=1)
        out.backward(do)
        q.grad = k.grad = v.grad = None

    res = {"world": world_size, "local_tokens": Sl, "context": Sl * world_size}
    for mode, env in (("fused", dict(CB200_RING_ATTN="fused")),
                      ("python_p2p_gather", dict(CB200_RING_ATTN="python", CB200_RING_ATTN_P2P="1")),
                      ("python_nccl_ring", dict(CB200_RING_ATTN="python", CB200_RING_ATTN_P2P="0"))):
        os.environ.update(env)
        for _ in range(2):
            run()
        torch.cuda.synchronize()
        dist.barrier()
        s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        s.record()
        for _ in range(3):
            run()
        e.record()
        torch.cuda.synchronize()
        t = torch.tensor([s.elapsed_time(e) / 3], device="cuda")
        dist.all_reduce(t, op=dist.ReduceOp.MAX)
        res[mode + "_ms"] = t.item()
    # causal attention FLOPs of this rank's share: fwd 4 S^2 H D / 2 / sp, bwd 2.5x
    S = Sl * world_size
    res["fused_tflops_per_gpu"] = 3.5 * 4.0 * S * S * Hq * D / 2 / world_size / res["fused_ms"] / 1e9
    if rank == 0:
        print("RING_TIMING " + json.dumps(res), flush=True)


@pytest.mark.gpu
@rerun_if_address_is_in_use()
def test_ring_attention_gpu():
    if torch.cuda.device_count() < 2:
        pytest.skip("needs >= 2 GPUs")
    spawn(_gpu_worker, 2)


if __name__ == "__main__":
    spawn(_gpu_worker, int(os.environ.get("NGPU", "2")))
