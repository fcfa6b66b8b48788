"""Paged prefill on the wgmma flash kernel: new query rows attending over keys held in a paged KV cache.

Every output row must be bitwise equal to the same row of the packed kernel run over the whole sequence gathered
contiguous (`flash_fwd(..., cu_seqlens=)`, or `flash_prefill` with a window / ALiBi): both kernels walk key tiles that
start at key 0, every row sees the same absolute positions, and a key tile that is fully masked for a row leaves its
online-softmax state unchanged.  Each case is also checked against the float64 reference."""
import itertools

import pytest
import torch

pytestmark = pytest.mark.gpu

DTYPES = [torch.bfloat16, torch.float16]
NEW_LENS = [1, 17, 128, 129, 300]


def _cached_lens(bs):
    return [0, bs, 3 * bs, (136 + bs - 1) // bs * bs]          # none, one block, several blocks, more than 128


def _build(dtype, D, G, bs, cached, new, seed, Hkv=2):
    """A paged cache holding each sequence's K/V in permuted blocks; unreferenced blocks are NaN, the unwritten tail
    slots of each last block finite stale values, table tails -1.  Returns the paged tensors and the contiguous
    full-sequence tensors of the packed reference."""
    g = torch.Generator(device="cuda").manual_seed(seed)
    Hq = Hkv * G
    lens = [c + n for c, n in zip(cached, new)]
    nblk = [(L + bs - 1) // bs for L in lens]
    num_blocks = sum(nblk) + 7
    perm = torch.randperm(num_blocks, generator=torch.Generator().manual_seed(seed)).tolist()
    max_blocks = max(nblk) + 2
    tables = torch.full((len(lens), max_blocks), -1, dtype=torch.int32)
    kc = torch.full((num_blocks, bs, Hkv, D), float("nan"), dtype=dtype, device="cuda")
    vc = torch.full_like(kc, float("nan"))
    qf, kf, vf, qn = [], [], [], []
    at = 0
    for b, (L, c) in enumerate(zip(lens, cached)):
        ids = perm[at:at + nblk[b]]
        at += nblk[b]
        tables[b, :nblk[b]] = torch.tensor(ids, dtype=torch.int32)
        k = torch.randn(nblk[b] * bs, Hkv, D, generator=g, device="cuda").to(dtype)    # tail rows: stale, finite
        v = torch.randn(nblk[b] * bs, Hkv, D, generator=g, device="cuda").to(dtype)
        kc[ids] = k.view(nblk[b], bs, Hkv, D)
        vc[ids] = v.view(nblk[b], bs, Hkv, D)
        q = torch.randn(L, Hq, D, generator=g, device="cuda").to(dtype)
        qf.append(q)
        kf.append(k[:L])
        vf.append(v[:L])
        qn.append(q[c:])
    cu_new = torch.tensor([0] + list(itertools.accumulate(new)), dtype=torch.int32, device="cuda")
    cu_full = torch.tensor([0] + list(itertools.accumulate(lens)), dtype=torch.int32, device="cuda")
    return dict(q=torch.cat(qn), kc=kc, vc=vc, tables=tables.cuda(), cu_new=cu_new,
                lens=torch.tensor(lens, dtype=torch.int32, device="cuda"), qf=torch.cat(qf), kf=torch.cat(kf),
                vf=torch.cat(vf), cu_full=cu_full, cached=cached, new=new)


def _new_rows(t, case):
    return torch.cat([t[int(case["cu_full"][b]) + c: int(case["cu_full"][b + 1])]
                      for b, c in enumerate(case["cached"])])


def _check(case, window=0, slopes=None):
    from colossalai_b200.ops import flash_attn_native as fa
    from colossalai_b200.ops import inference as iops

    D = case["q"].shape[-1]
    scale = D ** -0.5
    got = fa.flash_prefill_paged(case["q"], case["kc"], case["vc"], case["tables"], case["cu_new"], case["lens"], scale,
                                 window=window, alibi_slopes=slopes)
    if window or slopes is not None:
        ref = fa.flash_prefill(case["qf"], case["kf"], case["vf"], case["cu_full"], scale, window=window,
                               alibi_slopes=slopes)
    else:
        ref = fa.flash_fwd(case["qf"], case["kf"], case["vf"], 1, True, scale, cu_seqlens=case["cu_full"])[0]
    torch.cuda.synchronize()
    ref = _new_rows(ref, case)
    assert torch.isfinite(got.float()).all()
    assert torch.equal(got, ref), f"max |diff| {(got.float() - ref.float()).abs().max().item()}"
    # float64 reference
    r64 = iops.paged_prefill_attention_ref(case["q"].double(), case["kc"].double(), case["vc"].double(),
                                           case["tables"], case["cu_new"], case["lens"], scale,
                                           None if slopes is None else slopes.double(), window or None)
    tol = 1.5e-2 if case["q"].dtype == torch.bfloat16 else 2e-3
    torch.testing.assert_close(got.double(), r64, atol=tol, rtol=tol)


@pytest.mark.parametrize("bs", [8, 16, 64, 128])
@pytest.mark.parametrize("G", [1, 4, 8])
@pytest.mark.parametrize("D", [64, 128])
@pytest.mark.parametrize("dtype", DTYPES)
def test_paged_prefill_bitwise_equals_packed_kernel(dtype, D, G, bs):
    idx = DTYPES.index(dtype) * 24 + [64, 128].index(D) * 12 + [1, 4, 8].index(G) * 4 + [8, 16, 64, 128].index(bs)
    nseq = 1 + idx % 4                                              # 1-4 sequences of unequal lengths
    cached = [_cached_lens(bs)[(idx + i) % 4] for i in range(nseq)]
    new = [NEW_LENS[(idx + 2 * i) % 5] for i in range(nseq)]
    _check(_build(dtype, D, G, bs, cached, new, seed=idx))
    # every cached length against every new length once per (dtype, D): one batch of 20 sequences
    if G == 4 and bs == 16:
        pairs = list(itertools.product(_cached_lens(bs), NEW_LENS))
        _check(_build(dtype, D, G, bs, [c for c, _ in pairs], [n for _, n in pairs], seed=1000 + idx))


@pytest.mark.parametrize("D", [64, 128])
@pytest.mark.parametrize("dtype", DTYPES)
def test_paged_prefill_window_and_alibi(dtype, D):
    Hkv, G, bs = 2, 4, 16
    cached, new = [0, 16, 320, 512], [129, 300, 17, 128]
    slopes = torch.tensor([2 ** (-(i + 1) / 2) for i in range(Hkv * G)], device="cuda")
    case = _build(dtype, D, G, bs, cached, new, seed=7, Hkv=Hkv)
    for window in (40, 200, 4096):       # smaller than the cached prefix (leading tiles skipped) ... beyond the context
        _check(case, window=window)
        _check(case, window=window, slopes=slopes)
    _check(case, slopes=slopes)


@pytest.mark.parametrize("dtype", DTYPES)
def test_paged_prefill_long_context_few_new_tokens(dtype):
    case = _build(dtype, 128, 4, 16, [16384 - 8], [8], seed=11)
    _check(case)


def test_one_native_launch_per_call():
    from colossalai_b200.kernel import launch_counter
    from colossalai_b200.ops import inference as iops

    case = _build(torch.bfloat16, 128, 4, 16, [32, 0], [17, 40], seed=3)
    launch_counter.reset()
    iops.paged_prefill_attention(case["q"], case["kc"], case["vc"], case["tables"], case["cu_new"], case["lens"])
    assert dict(launch_counter.by_name) == {"flash_attn_paged_prefill": 1}


@pytest.mark.parametrize("what", ["fp32", "fp8 cache", "head_dim 32", "cache dtype differs"])
def test_outside_the_envelope_takes_the_reference(what):
    from colossalai_b200.kernel import launch_counter
    from colossalai_b200.ops import inference as iops

    case = _build(torch.bfloat16, 32 if what == "head_dim 32" else 64, 2, 16, [32, 16], [5, 20], seed=5)
    q, kc, vc = case["q"], case["kc"], case["vc"]
    if what == "fp32":
        q, kc, vc = q.float(), kc.float(), vc.float()
    elif what == "fp8 cache":
        kc, vc = (c.to(torch.float8_e5m2).view(torch.uint8) for c in (kc, vc))
    elif what == "cache dtype differs":
        q = q.half()
    args = (q, kc, vc, case["tables"], case["cu_new"], case["lens"])
    launch_counter.reset()
    got = iops.paged_prefill_attention(*args)
    assert launch_counter.by_name.get("flash_attn_paged_prefill", 0) == 0
    assert torch.equal(got, iops.paged_prefill_attention_ref(*args))


def test_launcher_rejects_bad_arguments_and_launches_nothing():
    from colossalai_b200.ops import flash_attn_native as fa

    case = _build(torch.bfloat16, 128, 4, 16, [32, 16], [5, 20], seed=9)
    T, Hq, D = case["q"].shape
    nb, bs, Hkv, _ = case["kc"].shape
    out = torch.full_like(case["q"], float("nan"))
    o_state = torch.full((T, Hq, D), float("nan"), device="cuda")
    lse = torch.full((T, Hq), float("nan"), device="cuda")
    good = dict(q=case["q"].data_ptr(), k=case["kc"].data_ptr(), v=case["vc"].data_ptr(), out=out.data_ptr(), lse=0,
                batch=2, seqlen_q=0, seqlen_k=0, hq=Hq, hkv=Hkv, d=D, causal=True, scale=D ** -0.5,
                dtype=torch.bfloat16, cu_seqlens=case["cu_new"].data_ptr(), total_tokens=T,
                block_tables=case["tables"].data_ptr(), seq_lens=case["lens"].data_ptr(), block_size=bs,
                max_blocks=case["tables"].shape[1], num_blocks=nb)
    rejected = {
        "block_size 24": dict(good, block_size=24),
        "block_size 0": dict(good, block_size=0),
        "block_size 256": dict(good, block_size=256),
        "not causal": dict(good, causal=False),
        "without cu_seqlens": dict(good, cu_seqlens=0, seqlen_q=T, seqlen_k=T, batch=1),
        "with o_state": dict(good, o_state=o_state.data_ptr(), lse=lse.data_ptr()),
        "null seq_lens": dict(good, seq_lens=0),
        "seq_lens without block_tables": dict(good, block_tables=0),
        "max_blocks 0": dict(good, max_blocks=0),
        "num_blocks 0": dict(good, num_blocks=0),
        "cache rows past int32": dict(good, num_blocks=2 ** 27),
        "head_dim 96": dict(good, d=96),
        "fp32": dict(good, dtype=torch.float32),
    }
    for name, args in rejected.items():
        with pytest.raises(RuntimeError, match=r"CUDA error 1$"):
            fa._fwd(name, **args)
    torch.cuda.synchronize()
    for t in (out, o_state, lse):
        assert torch.isnan(t).all(), "a rejected call wrote its output"
    fa._fwd("paged", **good)
    torch.cuda.synchronize()
    assert torch.isfinite(out.float()).all()


# ---------------------------------------------------------------------------------------------------- engines
SHARED = [(7 * i + 3) % 500 + 3 for i in range(70)]                # a 70-token prefix: 4 full blocks of 16


def _engine_run(model, cfg_kw, waves, n_new, caching):
    """Greedy tokens and the per-step logits (prefill steps' last-token rows, then decode steps) of every wave."""
    import colossalai_b200.inference.core.llm_engine as le
    from colossalai_b200.inference import InferenceConfig, InferenceEngine
    from colossalai_b200.inference.config import GenerationConfig

    eng = InferenceEngine(model, None, InferenceConfig(enable_prefix_caching=caching, **cfg_kw))
    firsts = []
    orig = le.search_tokens

    def spy(gen, logits, is_prompt, **kw):
        if is_prompt:
            firsts.append(logits.float().clone())
        return orig(gen, logits, is_prompt, **kw)

    le.search_tokens = spy
    try:
        toks = [eng.generate(prompts_token_ids=w, return_token_ids=True,
                             generation_config=GenerationConfig(max_new_tokens=n_new))[1] for w in waves]
    finally:
        le.search_tokens = orig
    return eng, toks, torch.cat(firsts)


def _margins_ok(model, prompts, n_new, tol):
    """Top-2 logit margin of every greedy step of the full-recompute model on these prompts exceeds `tol`."""
    for p in prompts:
        ids = list(p)
        for _ in range(n_new):
            with torch.no_grad():
                lg = model(input_ids=torch.tensor([ids], device="cuda"))["logits"][-1, : model.cfg.vocab_size].float()
            top = lg.topk(2).values
            if float(top[0] - top[1]) <= tol:
                return False
            ids.append(int(lg.argmax()))
    return True


@pytest.mark.parametrize("name,kw", [
    ("llama-tiny", dict(head_dim=64, num_attention_heads=2, num_key_value_heads=2)),
    ("llama-tiny", dict(head_dim=128, num_attention_heads=4, num_key_value_heads=1)),
    ("mistral-tiny", dict(head_dim=64, sliding_window=40)),
    ("baichuan-tiny", dict(head_dim=64)),
], ids=["llama-d64", "llama-d128-gqa", "sliding-window", "alibi"])
def test_engine_prefix_caching_matches_no_caching(name, kw):
    from colossalai_b200.kernel import launch_counter
    from colossalai_b200.models import build_model, get_config

    torch.manual_seed(0)
    model = build_model(get_config(name, **kw)).eval()
    if name == "baichuan-tiny":
        model.fold_norm_head()
    model = model.to(torch.bfloat16).cuda()
    n_new = 3
    with torch.no_grad():
        scale = model(input_ids=torch.tensor([SHARED], device="cuda"))["logits"].float().abs().max().item()
    tol = 0.02 * scale                                             # bf16 tolerance of the first-token logits
    pool = [SHARED + [400 + i, (401 + 2 * i) % 500 + 3, (402 + 3 * i) % 500 + 3] for i in range(64)]   # vocab 512
    prompts = [p for p in pool if _margins_ok(model, [p], n_new, 2 * tol)][:5]
    assert len(prompts) >= 3, "not enough prompts with a clear greedy choice"
    waves = [prompts[:1], prompts[1:]]
    # ALiBi models copy their slopes to the device in every forward, which a CUDA-graph capture refuses: they decode
    # eagerly
    cfg_kw = dict(max_batch_size=4, max_input_len=96, max_output_len=n_new, block_size=16, dtype="bf16",
                  use_cuda_graph=name != "baichuan-tiny", ignore_eos=True)
    _, off_toks, off_logits = _engine_run(model, cfg_kw, waves, n_new, False)
    launch_counter.reset()
    eng, on_toks, on_logits = _engine_run(model, cfg_kw, waves, n_new, True)
    assert eng.request_handler.cache_manager.prefix_cache_stats["hit_tokens"] > 0
    assert launch_counter.by_name.get("flash_attn_paged_prefill", 0) > 0
    assert (on_logits - off_logits).abs().max().item() <= tol
    assert on_toks == off_toks
