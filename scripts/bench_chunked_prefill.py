"""Chunked prefill on the GPU: the decode streams' inter-token latency while long prompts arrive.

Engine: a `llama3.2-1b`-shaped model with bf16 random weights, CUDA graphs on, max_batch_size 16, block 16.
Workload: 12 streams with 32-token prompts decode 256 tokens each.  Once every stream has 16 tokens, four
8192-token prompts arrive together (8 new tokens each).  `prefill_ratio` is 0 so that the unchunked engine prefills
arriving prompts at its next step; with its default, 1.2, it would hold them back until the streams end.  Chunked
steps do not use it.

For `max_num_batched_tokens` None, 512 and 2048 the script reports:
- the streams' inter-token latency (time between consecutive tokens of a stream): p50, p99 and max.  Every `step()`
  is timed on the host and ended by a device synchronise;
- the time from the long prompts' arrival to each one's first token;
- the total time of the workload.
Each configuration runs the whole workload once untimed first.  Prints one JSON line with the card's name and power
limit, read in the same run.  Needs a GPU.
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

STREAMS, STREAM_PROMPT, STREAM_TOKENS = 12, 32, 256
LONG, LONG_PROMPT, LONG_TOKENS = 4, 8192, 8
ARRIVE_AFTER = 16                    # stream tokens before the long prompts arrive
BUDGETS = [None, 512, 2048]


def gpu_info():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
        name, power, clock = (s.strip() for s in out.split(","))
    except (OSError, IndexError, ValueError, subprocess.SubprocessError):
        name, power, clock = torch.cuda.get_device_name(), "unknown", "unknown"
    return {"gpu": name, "power_limit": power, "max_sm_clock": clock}


def run_workload(eng, streams, longs):
    """Returns (stream inter-token latencies in s, long prompts' times to first token in s, total s)."""
    from colossalai_b200.inference.config import GenerationConfig

    rh = eng.request_handler
    eng.add_request(request_ids=list(range(STREAMS)), prompts_token_ids=streams,
                    generation_config=GenerationConfig(max_new_tokens=STREAM_TOKENS))
    seqs = {rid: rh._find_sequence(rid) for rid in range(STREAMS)}
    stamps = {rid: [] for rid in seqs}
    long_ids = list(range(STREAMS, STREAMS + LONG))
    arrived = None
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    while rh.check_unfinished_reqs():
        if arrived is None and all(seqs[r].output_len >= ARRIVE_AFTER for r in range(STREAMS)):
            eng.add_request(request_ids=long_ids, prompts_token_ids=longs,
                            generation_config=GenerationConfig(max_new_tokens=LONG_TOKENS))
            seqs.update({rid: rh._find_sequence(rid) for rid in long_ids})
            stamps.update({rid: [] for rid in long_ids})
            arrived = time.perf_counter()
        eng.step()
        torch.cuda.synchronize()
        now = time.perf_counter()
        for rid, s in seqs.items():
            while len(stamps[rid]) < s.output_len:
                stamps[rid].append(now)
    total = time.perf_counter() - t0
    itl = [b - a for rid in range(STREAMS) for a, b in zip(stamps[rid], stamps[rid][1:])]
    ttft = [stamps[rid][0] - arrived for rid in long_ids]
    assert all(seqs[r].output_len == STREAM_TOKENS for r in range(STREAMS))
    return itl, ttft, total


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--model", default="llama3.2-1b")
    args = ap.parse_args()
    assert torch.cuda.is_available(), "needs a GPU"
    from colossalai_b200.inference import InferenceConfig, InferenceEngine
    from colossalai_b200.models import build_model, get_config

    torch.manual_seed(0)
    model = build_model(get_config(args.model)).to(torch.bfloat16).cuda().eval()
    vocab = model.cfg.vocab_size
    g = torch.Generator().manual_seed(1)
    streams = [torch.randint(3, vocab, (STREAM_PROMPT,), generator=g).tolist() for _ in range(STREAMS)]
    longs = [torch.randint(3, vocab, (LONG_PROMPT,), generator=g).tolist() for _ in range(LONG)]
    rows = []
    for budget in BUDGETS:
        eng = InferenceEngine(model, None, InferenceConfig(
            max_batch_size=16, max_input_len=LONG_PROMPT, max_output_len=STREAM_TOKENS, block_size=16, dtype="bf16",
            use_cuda_graph=True, ignore_eos=True, prefill_ratio=0.0, max_num_batched_tokens=budget))
        run_workload(eng, streams, longs)                                # warm-up: every shape of the timed run
        itl, ttft, total = run_workload(eng, streams, longs)
        ms = np.array(itl) * 1e3
        rows.append({"max_num_batched_tokens": budget, "itl_ms_p50": round(float(np.percentile(ms, 50)), 2),
                     "itl_ms_p99": round(float(np.percentile(ms, 99)), 2), "itl_ms_max": round(float(ms.max()), 2),
                     "long_ttft_s": [round(t, 3) for t in ttft], "total_s": round(total, 3)})
        print(json.dumps(rows[-1]), flush=True)
        del eng
        torch.cuda.empty_cache()
    print(json.dumps({**gpu_info(), "model": args.model, "streams": STREAMS, "stream_tokens": STREAM_TOKENS,
                      "long_prompts": LONG, "long_prompt_tokens": LONG_PROMPT, "results": rows}))


if __name__ == "__main__":
    main()
