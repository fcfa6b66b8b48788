"""Chunked prefill on the GPU: the mixed step of `PagedKVRuntime` (prompt chunks through the paged prefill, decode rows
through the split-KV paged decode) and bf16 engines with chunking on and off.

A chunk's rows must be bitwise equal to the same rows of the packed kernel over the whole prompt (the paged prefill's
own guarantee, see test_paged_prefill.py), and the mixed step bitwise equal to the two calls made separately on the
same cache."""
import itertools

import pytest
import torch

pytestmark = pytest.mark.gpu

DTYPES = [torch.bfloat16, torch.float16]


def _build(dtype, D, G, bs, chunks, decode_lens, seed, Hkv=2):
    """A paged cache, NaN everywhere but the cached positions of every sequence (in permuted blocks).  `chunks`:
    (cached, new) per prompt; `decode_lens`: the length, this step's token included, of every decoding sequence.  The
    step's K/V are returned apart, for the runtime to write."""
    g = torch.Generator(device="cuda").manual_seed(seed)
    Hq = Hkv * G
    lens = [c + n for c, n in chunks] + list(decode_lens)
    new = [n for _, n in chunks] + [1] * len(decode_lens)
    nblk = [(L + bs - 1) // bs for L in lens]
    num_blocks = sum(nblk) + 5
    perm = torch.randperm(num_blocks, generator=torch.Generator().manual_seed(seed)).tolist()
    tables = torch.full((len(lens), max(nblk) + 1), -1, dtype=torch.int32)
    kc = torch.full((num_blocks, bs, Hkv, D), float("nan"), dtype=dtype, device="cuda")
    vc = torch.full_like(kc, float("nan"))
    full, step = [], []
    at = 0
    for b, (L, n) in enumerate(zip(lens, new)):
        ids = perm[at:at + nblk[b]]
        at += nblk[b]
        tables[b, :nblk[b]] = torch.tensor(ids, dtype=torch.int32)
        q, k, v = (torch.randn(L, h, D, generator=g, device="cuda").to(dtype) for h in (Hq, Hkv, Hkv))
        rows = torch.tensor(ids, device="cuda").repeat_interleave(bs)[: L - n], torch.arange(L - n, device="cuda") % bs
        kc[rows], vc[rows] = k[: L - n], v[: L - n]
        full.append((q, k, v))
        step.append((q[L - n:], k[L - n:], v[L - n:]))
    q, k, v = (torch.cat(t) for t in zip(*step))
    return dict(q=q, k=k, v=v, kc=kc, vc=vc, tables=tables.cuda(), lens=torch.tensor(lens, dtype=torch.int32),
                cached=[c for c, _ in chunks], full=full[: len(chunks)], chunks=chunks)


def _mixed(case, slopes=None, window=None):
    from colossalai_b200.inference.modeling import PagedKVRuntime

    rt = PagedKVRuntime([case["kc"]], [case["vc"]], case["kc"].shape[1])
    rt.set_chunked_step(case["tables"], case["lens"], case["cached"], "cuda")
    kw = {} if slopes is None else {"alibi_slopes": slopes}
    if window:
        kw["sliding_window"] = window
    return rt, rt.attend(0, case["q"], case["k"], case["v"], None, case["q"].shape[-1] ** -0.5, **kw)


@pytest.mark.parametrize("bs", [16, 64])
@pytest.mark.parametrize("G", [1, 4])
@pytest.mark.parametrize("D", [64, 128])
@pytest.mark.parametrize("dtype", DTYPES)
def test_mixed_step_equals_separate_calls_and_packed_prefill(dtype, D, G, bs):
    idx = DTYPES.index(dtype) * 8 + [64, 128].index(D) * 4 + [1, 4].index(G) * 2 + [16, 64].index(bs)
    chunks = [(0, 2 * bs), (bs, 17), (3 * bs, 130), (0, 5)][: 1 + idx % 4]      # chunks end mid-block or on a boundary
    decode_lens = [[1, 40, 300, 1030], [7], [], [bs + 1, 2 * bs]][idx % 4]
    case = _build(dtype, D, G, bs, chunks, decode_lens, seed=idx)
    Hq = case["q"].shape[1]
    slopes = torch.tensor([2 ** (-(i + 1) / 2) for i in range(Hq)], device="cuda")
    # the step's K/V writes are the same in every variant, so one cache serves them all
    for window, alibi in itertools.product((None, 48), (None, slopes)):
        _check_mixed(case, chunks, decode_lens, alibi, window)


def _check_mixed(case, chunks, decode_lens, slopes, window):
    from colossalai_b200.ops import flash_attn_native as fa
    from colossalai_b200.ops import inference as iops

    D = case["q"].shape[-1]
    rt, got = _mixed(case, slopes, window)
    torch.cuda.synchronize()
    assert torch.isfinite(got.float()).all()
    scale = D ** -0.5
    bp, tp = len(chunks), sum(n for _, n in chunks)
    lens = case["lens"].cuda()
    if window is not None and int(lens.max()) <= window:           # the runtime drops a window nothing exceeds
        window = None
    cu = torch.tensor([0] + list(itertools.accumulate(n for _, n in chunks)), dtype=torch.int32, device="cuda")
    sep = [iops.paged_prefill_attention(case["q"][:tp], case["kc"], case["vc"], case["tables"][:bp], cu, lens[:bp],
                                        scale, alibi_slopes=slopes, window=window)]
    if decode_lens:
        sep.append(iops.paged_decode_attention(case["q"][tp:], case["kc"], case["vc"], case["tables"][bp:],
                                               lens[bp:], scale, alibi_slopes=slopes, window=window))
    assert torch.equal(got, torch.cat(sep))
    # the chunk rows against the packed prefill over each whole prompt
    qf, kf, vf = (torch.cat(t) for t in zip(*case["full"]))
    cu_full = torch.tensor([0] + list(itertools.accumulate(c + n for c, n in chunks)), dtype=torch.int32,
                           device="cuda")
    if window or slopes is not None:
        ref = fa.flash_prefill(qf, kf, vf, cu_full, scale, window=window or 0, alibi_slopes=slopes)
    else:
        ref = fa.flash_fwd(qf, kf, vf, 1, True, scale, cu_seqlens=cu_full)[0]
    ref = torch.cat([ref[int(cu_full[b]) + c: int(cu_full[b + 1])] for b, (c, _) in enumerate(chunks)])
    assert torch.equal(got[:tp], ref), f"max |diff| {(got[:tp].float() - ref.float()).abs().max().item()}"


@pytest.mark.parametrize("decode", [True, False])
def test_launches_per_layer(decode):
    from colossalai_b200.kernel import launch_counter

    case = _build(torch.bfloat16, 128, 4, 16, [(16, 40), (0, 9)], [33, 100] if decode else [], seed=3)
    launch_counter.reset()
    _mixed(case)
    want = {"kv_cache_write": 1, "flash_attn_paged_prefill": 1}
    if decode:
        want["paged_decode_attention"] = 2
    assert dict(launch_counter.by_name) == want


# ---------------------------------------------------------------------------------------------------- engines
PREFIX = [(7 * i + 3) % 500 + 3 for i in range(72)]


def _engine_run(model, cfg_kw, prompts, n_new, budget):
    """Greedy tokens, the first-token logits of every prompt, and per step whether it held chunks and decode rows."""
    import colossalai_b200.inference.core.llm_engine as le
    from colossalai_b200.inference import InferenceConfig, InferenceEngine
    from colossalai_b200.inference.config import GenerationConfig

    eng = InferenceEngine(model, None, InferenceConfig(max_num_batched_tokens=budget, **cfg_kw))
    firsts = {}
    orig = le.search_tokens
    keys = {tuple(p) for p in prompts}

    def spy(gen, logits, is_prompt, batch_token_ids=None, **kw):
        for row, ids in zip(logits, batch_token_ids):
            if tuple(ids) in keys:
                firsts[tuple(ids)] = row.float().clone()
        return orig(gen, logits, is_prompt, batch_token_ids=batch_token_ids, **kw)

    steps = []
    rt = eng.kv_runtime
    set_chunked = rt.set_chunked_step

    def spy_chunked(tables, lens, cached, device):
        steps.append(("chunks", len(lens) - len(cached)))
        return set_chunked(tables, lens, cached, device)

    rt.set_chunked_step = spy_chunked
    replays = []
    for bs, runner in list(eng.graph_runners.items()):
        def counted(runner=runner, bs=bs, **kw):
            replays.append(bs)
            return runner(**kw)
        eng.graph_runners[bs] = counted
    rh = eng.request_handler
    schedule = rh.schedule

    def spy_schedule():
        batch = schedule()
        if batch is rh.running_bb and not batch.is_empty:
            steps.append(("decode", batch.current_batch_size))
        return batch

    rh.schedule = spy_schedule
    le.search_tokens = spy
    try:
        toks = eng.generate(prompts_token_ids=prompts, return_token_ids=True,
                            generation_config=GenerationConfig(max_new_tokens=n_new))[1]
    finally:
        le.search_tokens = orig
    return eng, toks, torch.stack([firsts[tuple(p)] for p in prompts]), steps, replays


def _clear_prompts(model, pool, n_new, tol, k):
    """The first `k` prompts of `pool` (all of one length) whose every greedy step of full recomputation has a top-2
    logit margin above `tol`.  The pool decodes as one batch."""
    ids = torch.tensor(pool, device="cuda")
    ok = torch.ones(len(pool), dtype=torch.bool, device="cuda")
    for _ in range(n_new):
        B, S = ids.shape
        with torch.no_grad():
            lg = model(input_ids=ids)["logits"].reshape(B, S, -1)[:, -1, : model.cfg.vocab_size].float()
        top = lg.topk(2, dim=-1).values
        ok &= (top[:, 0] - top[:, 1]) > tol
        ids = torch.cat([ids, lg.argmax(-1, keepdim=True)], 1)
    return [p for p, good in zip(pool, ok.tolist()) if good][:k]


@pytest.mark.parametrize("name,kw", [
    ("llama-tiny", dict(head_dim=64, num_attention_heads=2, num_key_value_heads=2)),
    ("llama-tiny", dict(head_dim=128, num_attention_heads=4, num_key_value_heads=1)),
    ("mistral-tiny", dict(head_dim=64, sliding_window=40)),
    ("baichuan-tiny", dict(head_dim=64)),
], ids=["llama-d64", "llama-d128-gqa", "sliding-window", "alibi"])
def test_engine_chunked_matches_unchunked(name, kw):
    from colossalai_b200.kernel import launch_counter
    from colossalai_b200.models import build_model, get_config

    torch.manual_seed(0)
    model = build_model(get_config(name, **kw)).eval()
    if name == "baichuan-tiny":
        model.fold_norm_head()
    model = model.to(torch.bfloat16).cuda()
    n_new = 4
    with torch.no_grad():
        scale = model(input_ids=torch.tensor([PREFIX], device="cuda"))["logits"].float().abs().max().item()
    tol = 0.02 * scale                                             # bf16 tolerance of the first-token logits
    pool = [PREFIX + [400 + i, (401 + 2 * i) % 500 + 3, (402 + 3 * i) % 500 + 3] for i in range(64)]   # vocab 512
    prompts = _clear_prompts(model, pool, n_new, 2 * tol, 6)
    assert len(prompts) >= 5, "not enough prompts with a clear greedy choice"
    # ALiBi models copy their slopes to the device in every forward, which a CUDA-graph capture refuses.  A captured
    # decode graph keeps the attention branch taken at capture, when no sequence exceeds the window, so a
    # sliding-window model decodes without its window under graphs while chunked steps (eager) apply it.  Both decode
    # eagerly here.
    graphs = name not in ("baichuan-tiny", "mistral-tiny")
    cfg_kw = dict(max_batch_size=4, max_input_len=96, max_output_len=n_new, block_size=16, dtype="bf16",
                  use_cuda_graph=graphs, ignore_eos=True)
    _, off_toks, off_logits, _, _ = _engine_run(model, cfg_kw, prompts, n_new, None)
    launch_counter.reset()
    eng, on_toks, on_logits, steps, replays = _engine_run(model, cfg_kw, prompts, n_new, 32)
    assert launch_counter.by_name.get("flash_attn_paged_prefill", 0) > 0
    assert any(kind == "chunks" and n_dec > 0 for kind, n_dec in steps), "no mixed step"
    assert (on_logits - off_logits).abs().max().item() <= tol
    assert on_toks == off_toks
    # every pure decode step at a captured batch size replays its CUDA graph
    decode_steps = [n for kind, n in steps if kind == "decode" and n in eng.graph_runners]
    assert replays == (decode_steps if graphs else [])
    assert not graphs or decode_steps
