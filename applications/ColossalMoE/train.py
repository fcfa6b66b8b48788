"""Mixtral-style sparse-MoE training with expert parallelism.

    torchrun --nproc-per-node 8 --master-addr 127.0.0.1 applications/ColossalMoE/train.py --model mixtral-8x7b \
        --ep 8 --zero 1 --batch_size 1 --max_length 4096 --steps 100 --save_dir ckpt --save_interval 50
    torchrun --nproc-per-node 2 --master-addr 127.0.0.1 applications/ColossalMoE/train.py --model mixtral-tiny --ep 2 --steps 10

Experts are sharded over the `--ep` group (dropless dispatch, grouped wgmma GEMMs, fused NVLink dispatch / combine on an
NVSwitch node), attention / dense layers over `--tp`, layers over `--pp`; the remaining ranks are data parallel (`--zero`).
The loss adds the routers' load-balancing terms; every `--log_interval` steps the expert load share is printed (max share
x experts: 1.0 = balanced).  `--pretrained` imports a HuggingFace Mixtral / DeepSeek-MoE directory (`models.hf_io`),
`--load_checkpoint` resumes.  Data: jsonl `{"text": ...}` via `--dataset`, else random tokens.

Parity: reference `applications/ColossalMoE/train.py:1-290` (+ `train.sh`).
"""
import argparse
import json
import os
import sys

import torch
import torch.distributed as dist

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
sys.path.insert(0, os.path.join(HERE, "..", ".."))

import colossalai_b200  # noqa: E402
from colossalai_b200.booster import Booster  # noqa: E402
from colossalai_b200.booster.plugin import MoeHybridParallelPlugin  # noqa: E402
from colossalai_b200.cluster import DistCoordinator  # noqa: E402
from colossalai_b200.models import build_model, get_config  # noqa: E402
from colossalai_b200.nn.lr_scheduler import CosineAnnealingWarmupLR  # noqa: E402
from colossalai_b200.nn.optimizer import HybridAdam  # noqa: E402
from utils import ExpertLoadMonitor, load_checkpoint, save_checkpoint  # noqa: E402


def batches(args, vocab: int, dp_rank: int, dev):
    if args.dataset:
        rows = []
        for path in args.dataset:
            with open(path) as f:
                rows += [[3 + b for b in json.loads(l)["text"].encode()][: args.max_length] for l in f if l.strip()]
        rows = [r + [0] * (args.max_length - len(r)) for r in rows]
        i = dp_rank * args.batch_size
        while True:
            ids = torch.tensor([rows[(i + j) % len(rows)] for j in range(args.batch_size)], device=dev)
            i += args.batch_size * args.dp_size
            yield {"input_ids": ids, "labels": ids.masked_fill(ids == 0, -100)}
    g = torch.Generator().manual_seed(1234 + dp_rank)
    while True:
        ids = torch.randint(0, vocab, (args.batch_size, args.max_length), generator=g).to(dev)
        yield {"input_ids": ids, "labels": ids}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--model", default="mixtral-tiny")
    ap.add_argument("--pretrained", default=None)
    ap.add_argument("--dataset", nargs="*", default=None)
    ap.add_argument("--ep", type=int, default=2)
    ap.add_argument("--tp", type=int, default=1)
    ap.add_argument("--pp", type=int, default=1)
    ap.add_argument("--zero", type=int, default=1)
    ap.add_argument("--microbatch_size", type=int, default=1)
    ap.add_argument("--batch_size", type=int, default=2)
    ap.add_argument("--max_length", type=int, default=128)
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--lr", type=float, default=1e-4)
    ap.add_argument("--weight_decay", type=float, default=0.01)
    ap.add_argument("--warmup_steps", type=int, default=2)
    ap.add_argument("--log_interval", type=int, default=5)
    ap.add_argument("--save_dir", default=None)
    ap.add_argument("--save_interval", type=int, default=0)
    ap.add_argument("--load_checkpoint", default=None)
    args = ap.parse_args()
    colossalai_b200.launch_from_torch(backend="nccl" if torch.cuda.is_available() else "gloo")
    coordinator = DistCoordinator()
    dev = colossalai_b200.accelerator.get_accelerator().get_current_device()
    torch.manual_seed(42)
    if args.pretrained:
        from colossalai_b200.models.hf_io import load_hf_checkpoint

        model = load_hf_checkpoint(args.pretrained)
    else:
        model = build_model(get_config(args.model))
    cfg = model.cfg
    plugin = MoeHybridParallelPlugin(ep_size=args.ep, tp_size=args.tp, pp_size=args.pp, zero_stage=args.zero,
                                     precision="bf16", max_norm=1.0,
                                     microbatch_size=args.microbatch_size if args.pp > 1 else None)
    booster = Booster(plugin=plugin)
    optimizer = HybridAdam(model.parameters(), lr=args.lr, weight_decay=args.weight_decay)
    scheduler = CosineAnnealingWarmupLR(optimizer, total_steps=args.steps, warmup_steps=args.warmup_steps)
    model, optimizer, _, _, scheduler = booster.boost(model, optimizer, lr_scheduler=scheduler)
    monitor = ExpertLoadMonitor(model.unwrap())
    args.dp_size = plugin.dp_size
    data = batches(args, cfg.vocab_size, plugin.pg_mesh.axis_rank("dp"), dev)
    start = 0
    if args.load_checkpoint:
        _, start, _ = load_checkpoint(args.load_checkpoint, booster, model, optimizer, scheduler)
        coordinator.print_on_master(f"resumed from {args.load_checkpoint} at step {start}")
        for _ in range(start):
            next(data)

    def with_aux(out, batch=None):
        loss = out["loss"]
        aux = [m.aux_loss for m in model.unwrap().modules() if getattr(m, "aux_loss", None) is not None]
        return loss + sum(aux) if aux else loss

    for step in range(start, args.steps):
        batch = next(data)
        if args.pp > 1:
            out = booster.execute_pipeline(iter([batch]), model, with_aux, optimizer, return_loss=True)
            loss = out["loss"]
        else:
            loss = with_aux(model(**batch))
            booster.backward(loss, optimizer)
        optimizer.step()
        optimizer.zero_grad()
        scheduler.step()
        val = torch.full((1,), float("-inf"), device=dev) if loss is None else loss.detach().float().reshape(1)
        dist.all_reduce(val, op=dist.ReduceOp.MAX)
        if (step + 1) % args.log_interval == 0 or step + 1 == args.steps:
            share = monitor.fractions()
            monitor.reset()
            coordinator.print_on_master(
                f"step {step + 1}: loss {val.item():.4f} lr {optimizer.param_groups[0]['lr']:.3g} expert load "
                f"{[round(x, 3) for x in share.tolist()] if share is not None else 'n/a'} "
                f"(imbalance {float(share.max() * share.numel()) if share is not None else float('nan'):.2f})")
        if args.save_dir and args.save_interval and (step + 1) % args.save_interval == 0:
            path = save_checkpoint(args.save_dir, booster, model, optimizer, scheduler, 0, step + 1,
                                   args.batch_size * plugin.dp_size, coordinator.is_master())
            coordinator.print_on_master(f"saved {path}")
    dist.barrier()
    dist.destroy_process_group()


if __name__ == "__main__":
    main()
