"""Long-context training with zigzag ring attention (context parallelism): every rank holds 1 / sp of the sequence,
attention runs blockwise against the K/V of all ranks (fused NVLink path on sm_90a, python ring elsewhere), everything
else is sequence-local.  BASELINE config 5 is `--model llama3-8b --seq 131072 --sp 8 --zero 1 --grad-ckpt` on 8 GPUs
(not measured on H100).

    torchrun --nproc-per-node 8 --master-addr 127.0.0.1 examples/language/long_context/train_ring_attention.py \\
        --model llama3-8b --seq 131072 --sp 8 --zero 1 --grad-ckpt
    torchrun --nproc-per-node 2 --master-addr 127.0.0.1 examples/language/long_context/train_ring_attention.py   # CPU smoke

Reference counterpart: `examples/language/llama/benchmark.py -p 3d --sp N --sp_mode ring_attn`."""
import argparse
import os
import sys
import time

import torch
import torch.distributed as dist

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), "..", "..", ".."))
import colossalai_b200  # noqa: E402
from colossalai_b200.booster import Booster  # noqa: E402
from colossalai_b200.booster.plugin import HybridParallelPlugin  # noqa: E402
from colossalai_b200.lazy import LazyInitContext  # noqa: E402
from colossalai_b200.models import build_model, get_config  # noqa: E402
from colossalai_b200.nn.optimizer import HybridAdam  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--model", default="llama-tiny")
    ap.add_argument("--seq", type=int, default=256, help="tokens of ONE sequence (split over the sp ranks)")
    ap.add_argument("--batch", type=int, default=1)
    ap.add_argument("--sp", type=int, default=0, help="context-parallel size (default: all ranks)")
    ap.add_argument("--zero", type=int, default=0)
    ap.add_argument("--grad-ckpt", action="store_true")
    ap.add_argument("--steps", type=int, default=3)
    args = ap.parse_args()
    colossalai_b200.launch_from_torch()
    world, rank = dist.get_world_size(), dist.get_rank()
    sp = args.sp or world
    cuda = torch.cuda.is_available()
    cfg = get_config(args.model, **({"max_position_embeddings": max(args.seq, 256)} if args.model == "llama-tiny" else {}))
    assert args.seq % (2 * sp) == 0, "the zigzag layout needs seq divisible by 2 * sp"
    plugin = HybridParallelPlugin(tp_size=1, pp_size=1, sp_size=sp, enable_sequence_parallelism=True,
                                  sequence_parallelism_mode="ring_attn", zero_stage=args.zero,
                                  precision="bf16" if cuda or args.zero else "fp32", max_norm=1.0)
    booster = Booster(plugin=plugin)
    with LazyInitContext():
        model = build_model(cfg)
    if args.grad_ckpt:
        model.gradient_checkpointing_enable()
    optimizer = HybridAdam(model.parameters(), lr=1e-5, weight_decay=0.1)
    model, optimizer, *_ = booster.boost(model, optimizer)
    dev = colossalai_b200.accelerator.get_accelerator().get_current_device()
    g = torch.Generator().manual_seed(rank // sp)                 # the ranks of one sp group see the same sequence
    for step in range(args.steps):
        ids = torch.randint(0, cfg.vocab_size, (args.batch, args.seq), generator=g).to(dev)
        t0 = time.perf_counter()
        loss = model(input_ids=ids, labels=ids)["loss"]           # the plugin splits the sequence (zigzag) internally
        booster.backward(loss, optimizer)
        optimizer.step()
        optimizer.zero_grad()
        if cuda:
            torch.cuda.synchronize()
        dt = time.perf_counter() - t0
        if rank == 0:
            print(f"step {step}: loss {loss.item():.4f}  {dt * 1e3:.1f} ms  "
                  f"({args.batch * args.seq * (world // sp) / dt:,.0f} tokens/s, seq {args.seq}, sp {sp})")
    dist.barrier()
    colossalai_b200.initialize.shutdown()


if __name__ == "__main__":
    main()
