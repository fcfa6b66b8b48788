"""MoE training throughput through the Booster API with expert parallelism (reference:
examples/language/mixtral/benchmark.py and examples/language/deepseek/benchmark.py).

    torchrun --nproc-per-node 8 examples/language/mixtral/benchmark.py -c mixtral-8x7b --layers 4 --ep 8 --zero 1 -b 2 -l 4096

Prints device-timed tokens/s (max over ranks), the MoE back ends in use (fused NVLink dispatch/combine + wgmma grouped
GEMM vs NCCL all-to-all + library grouped GEMM: `--moe_backend`, `--grouped_gemm`) and peak memory.  `--layers` cuts the
depth so the full-width model fits one box without pipeline stages (Mixtral-8x7B is 47 B parameters); the per-layer
expert shapes - which is what the EP kernels see - are unchanged.
"""
import argparse
import json
import os
import sys

import torch
import torch.distributed as dist

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), "..", "..", ".."))

import colossalai_b200  # noqa: E402
from colossalai_b200.booster import Booster  # noqa: E402
from colossalai_b200.booster.plugin import MoeHybridParallelPlugin  # noqa: E402
from colossalai_b200.kernel import launch_counter  # noqa: E402
from colossalai_b200.lazy import LazyInitContext  # noqa: E402
from colossalai_b200.models import build_model, get_config  # noqa: E402
from colossalai_b200.moe import dispatch_combine as dc  # noqa: E402
from colossalai_b200.nn.optimizer import FusedAdam  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("-c", "--config", default="mixtral-8x7b")
    ap.add_argument("--layers", type=int, default=0)
    ap.add_argument("--ep", type=int, default=0, help="expert parallel size (default: world size)")
    ap.add_argument("--tp", type=int, default=1)
    ap.add_argument("--zero", type=int, default=1)
    ap.add_argument("-b", "--batch_size", type=int, default=2, help="sequences per rank per step")
    ap.add_argument("-l", "--max_length", type=int, default=4096)
    ap.add_argument("-s", "--num_steps", type=int, default=6)
    ap.add_argument("-i", "--ignore_steps", type=int, default=3)
    ap.add_argument("--moe_backend", default="auto", choices=["auto", "fused", "nccl"])
    ap.add_argument("--grouped_gemm", default="native", choices=["native", "lib"])
    args = ap.parse_args()
    os.environ["CB200_GROUPED_GEMM"] = args.grouped_gemm
    os.environ.setdefault("CB200_EP_CAPACITY_FACTOR", "2")      # receive buffers: 2x the balanced load (overflow raises)
    colossalai_b200.launch_from_torch(verbose=False)
    rank, world = dist.get_rank(), dist.get_world_size()
    dc.set_moe_backend(args.moe_backend)
    cfg = get_config(args.config, **({"num_hidden_layers": args.layers} if args.layers else {}))
    plugin = MoeHybridParallelPlugin(ep_size=args.ep or world, tp_size=args.tp, pp_size=1, zero_stage=args.zero,
                                     precision="bf16", max_norm=1.0)
    booster = Booster(plugin=plugin)
    torch.manual_seed(1234)
    with LazyInitContext():
        model = build_model(cfg)
    optimizer = FusedAdam(model.parameters(), lr=1e-5, weight_decay=0.1)
    model, optimizer, *_ = booster.boost(model, optimizer)
    dev = torch.device("cuda", torch.cuda.current_device())
    g = torch.Generator().manual_seed(4321 + plugin.pg_mesh.axis_rank("dp"))
    batches = [torch.randint(0, cfg.vocab_size, (args.batch_size, args.max_length), generator=g).to(dev) for _ in range(4)]
    times = []
    launch_counter.reset()
    for step in range(args.num_steps):
        ids = batches[step % 4]
        ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        ev0.record()
        out = model(input_ids=ids, labels=ids)
        loss = out["loss"]
        aux = [m.aux_loss for m in model.unwrap().modules() if getattr(m, "aux_loss", None) is not None]
        if aux:
            loss = loss + sum(aux)
        booster.backward(loss, optimizer)
        optimizer.step()
        optimizer.zero_grad()
        ev1.record()
        torch.cuda.synchronize()
        if step >= args.ignore_steps:
            times.append(ev0.elapsed_time(ev1) / 1e3)
        if rank == 0:
            print(f"step {step}: loss {loss.item():.4f}  {ev0.elapsed_time(ev1):.1f} ms", flush=True)
    t = torch.tensor(sum(times) / max(len(times), 1), device=dev)
    dist.all_reduce(t, op=dist.ReduceOp.MAX)
    tok = args.batch_size * world * args.max_length / t.item()
    if rank == 0:
        print(f"throughput: {tok:,.0f} tokens/s (max over ranks), {t.item() * 1e3:.1f} ms/step")
        print("MOE_BENCH " + json.dumps({
            "model": args.config + (f"[layers={args.layers}]" if args.layers else ""), "ep": args.ep or world,
            "tokens_per_s": tok, "ms_per_step": t.item() * 1e3, "moe_backend": dc.get_moe_backend(),
            "grouped_gemm": args.grouped_gemm, "launches_by_kernel": dict(launch_counter.by_name),
            "peak_mem_gib": torch.cuda.max_memory_allocated() / 2**30}), flush=True)
    dist.barrier()
    colossalai_b200.initialize.shutdown()


if __name__ == "__main__":
    main()
