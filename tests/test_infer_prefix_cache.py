"""Prefix caching in the paged inference engine (CPU tier): the block index of `KVCacheManager`, the paged prefill
reference op, and engines whose greedy tokens with caching equal those without it."""
import pytest
import torch

from colossalai_b200.inference import InferenceConfig, InferenceEngine
from colossalai_b200.inference.config import GenerationConfig
from colossalai_b200.inference.core.llm_engine import prefix_caching_unsupported
from colossalai_b200.inference.kv_cache import KVCacheManager
from colossalai_b200.models import build_model, get_config
from colossalai_b200.ops import inference as iops
from colossalai_b200.ops.attention import attention_ref

BS = 8


def _mgr(**kw):
    cfg = InferenceConfig(max_batch_size=2, max_input_len=32, max_output_len=8, block_size=BS, dtype="fp32",
                          enable_prefix_caching=True, **kw)
    return KVCacheManager(cfg, get_config("llama-tiny"))


def _table(mgr):
    return torch.full((mgr.get_max_blocks_per_sequence(),), -1, dtype=torch.int32)


def _serve(mgr, tokens, written=None):
    """Admit a prompt, index its written blocks, free it; returns (cached tokens, block ids)."""
    t = _table(mgr)
    c = mgr.allocate_context_with_prefix(t, tokens)
    ids = t[t >= 0].tolist()
    mgr.register_prefix_blocks(t, tokens, len(tokens) if written is None else written)
    mgr.free_block_table(t)
    return c, ids


# ---------------------------------------------------------------------------------------------------- manager
def test_match_is_capped_so_the_last_prompt_token_is_computed():
    mgr = _mgr()
    p = list(range(100, 124))                                       # exactly 3 blocks
    assert _serve(mgr, p)[0] == 0
    t = _table(mgr)
    assert mgr.allocate_context_with_prefix(t, p) == 2 * BS         # (24 - 1) // 8 = 2 blocks
    t2 = _table(mgr)
    assert mgr.allocate_context_with_prefix(t2, p + [7]) == 3 * BS
    assert t[:2].tolist() == t2[:2].tolist() and t[2] != t2[2]
    assert mgr.prefix_cache_stats == {"queried_tokens": 24 + 24 + 25, "hit_tokens": 40}


def test_matching_compares_every_token_of_the_chain():
    mgr = _mgr()
    p = list(range(100, 120))
    _serve(mgr, p)
    q = list(p)
    q[3] += 1                                                      # first block differs -> nothing matches
    assert mgr.match_prefix(q) == []
    r = list(p)
    r[BS + 1] += 1                                                 # second block differs -> first block only
    assert len(mgr.match_prefix(r)) == 1


def test_reference_counts_available_counts_and_lru_eviction_order():
    mgr = _mgr()
    total = mgr.num_available_blocks
    a = [1] * BS + [2] * BS + [3]
    b = [4] * BS + [5] * BS + [6]
    _, ids_a = _serve(mgr, a)
    _, ids_b = _serve(mgr, b)
    assert mgr.num_available_blocks == total                       # cached-free blocks count as available
    # a hit takes a cached-free block back (0 -> 1 reference) and a second hit shares it (1 -> 2)
    t1, t2 = _table(mgr), _table(mgr)
    assert mgr.allocate_context_with_prefix(t1, a) == 2 * BS
    assert mgr.allocate_context_with_prefix(t2, a) == 2 * BS
    assert [mgr._cache_blocks[i].ref_count for i in ids_a[:2]] == [2, 2]
    assert mgr.num_available_blocks == total - 2 - 2               # two shared blocks + one fresh tail each
    mgr.free_block_table(t1)
    assert [mgr._cache_blocks[i].ref_count for i in ids_a[:2]] == [1, 1]
    mgr.free_block_table(t2)
    assert mgr.num_available_blocks == total
    # once the never-indexed free blocks are used up, cached-free blocks are evicted least recently freed first: b's
    # (freed before a's were freed a second time)
    n_plain = int(mgr._block_states.sum())
    assert n_plain == total - 4
    assert not set(mgr._take_free_blocks(n_plain)) & set(ids_a[:2] + ids_b[:2])
    assert mgr._take_free_blocks(1) == [ids_b[0]]
    assert mgr.match_prefix(b) == []                               # its entry is gone with it
    assert mgr.match_prefix(a) == ids_a[:2]


def test_evicted_parent_block_reused_for_other_content_does_not_revive_its_child():
    mgr = _mgr()
    a = [1] * BS + [2] * BS + [3]
    _, ids = _serve(mgr, a)
    parent = ids[0]
    mgr._take_free_blocks(int(mgr._block_states.sum()))
    assert mgr._take_free_blocks(1) == [parent]                    # freed first, evicted first; its child stays
    # the parent's block now holds other tokens and is indexed under them
    t = _table(mgr)
    t[0] = parent
    mgr._cache_blocks[parent].add_ref()
    mgr.register_prefix_blocks(t, [9] * BS + [3], BS)
    assert mgr.match_prefix([9] * BS + [2] * BS + [3]) == [parent]  # the old child must not match under the new parent
    assert mgr.match_prefix(a) == []


def test_only_written_positions_are_indexed():
    mgr = _mgr()
    p = list(range(50, 50 + 3 * BS))
    t = _table(mgr)
    mgr.allocate_context_with_prefix(t, p)
    mgr.register_prefix_blocks(t, p, 2 * BS - 1)                   # block 1 lacks its last position
    assert len(mgr.match_prefix(p + [1])) == 1
    mgr.register_prefix_blocks(t, p, 2 * BS)
    assert len(mgr.match_prefix(p + [1])) == 2


def test_prefix_caching_off_keeps_plain_allocation():
    cfg = InferenceConfig(max_batch_size=2, max_input_len=32, max_output_len=8, block_size=BS, dtype="fp32")
    mgr = KVCacheManager(cfg, get_config("llama-tiny"))
    p = list(range(20))
    t = _table(mgr)
    mgr.allocate_context_from_block_table(t, len(p))
    mgr.register_prefix_blocks(t, p, len(p))
    mgr.free_block_table(t)
    assert mgr.match_prefix(p) == [] and bool(mgr._block_states.all())


# ---------------------------------------------------------------------------------------------------- reference op
@pytest.mark.parametrize("fp8", [False, True])
@pytest.mark.parametrize("alibi", [False, True])
@pytest.mark.parametrize("window", [None, 5, 40])
def test_paged_prefill_reference_matches_per_row_decode_reference(fp8, alibi, window):
    torch.manual_seed(0)
    bs, Hkv, G, D, nb = 4, 2, 2, 16, 24
    kc, vc = torch.randn(nb, bs, Hkv, D), torch.randn(nb, bs, Hkv, D)
    if fp8:
        kc, vc = (c.to(torch.float8_e5m2).view(torch.uint8) for c in (kc, vc))
    tables = torch.randperm(nb)[:18].to(torch.int32).view(3, 6)
    lens = torch.tensor([9, 21, 4], dtype=torch.int32)
    new = [3, 13, 4]
    cu = torch.tensor([0, 3, 16, 20], dtype=torch.int32)
    q = torch.randn(20, Hkv * G, D)
    kw = dict(window=window)
    if alibi:
        kw["alibi_slopes"] = torch.tensor([2 ** (-(i + 1)) for i in range(Hkv * G)])
    got = iops.paged_prefill_attention(q, kc, vc, tables, cu, lens, **kw)         # CPU: the reference path
    assert torch.equal(got, iops.paged_prefill_attention_ref(q, kc, vc, tables, cu, lens, **kw))
    # row by row: a decode query at position p sees positions 0..p
    rows, row_lens, row_tables = [], [], []
    for b in range(3):
        for j in range(new[b]):
            row_lens.append(int(lens[b]) - new[b] + j + 1)
            row_tables.append(tables[b])
    ref = iops.paged_decode_attention_ref(q, kc, vc, torch.stack(row_tables), torch.tensor(row_lens), **kw)
    torch.testing.assert_close(got, ref, atol=1e-5, rtol=1e-5)


def test_paged_prefill_reference_matches_attention_ref_on_gathered_kv():
    torch.manual_seed(1)
    bs, Hkv, G, D, nb = 8, 2, 3, 16, 10
    kc, vc = torch.randn(nb, bs, Hkv, D), torch.randn(nb, bs, Hkv, D)
    tables = torch.tensor([[7, 2, 5, -1]], dtype=torch.int32)
    L, n = 21, 6
    q = torch.randn(n, Hkv * G, D)
    got = iops.paged_prefill_attention(q, kc, vc, tables, torch.tensor([0, n], dtype=torch.int32),
                                       torch.tensor([L], dtype=torch.int32))
    k = iops.gather_paged_kv(kc, tables[0], L)
    v = iops.gather_paged_kv(vc, tables[0], L)
    q_full = torch.cat([torch.zeros(L - n, Hkv * G, D), q])
    ref = attention_ref(q_full, k, v, batch=1, causal=True)[L - n:]
    torch.testing.assert_close(got, ref, atol=1e-5, rtol=1e-5)


# ---------------------------------------------------------------------------------------------------- engines
def _naive_greedy(model, prompt, n_new):
    ids = list(prompt)
    for _ in range(n_new):
        with torch.no_grad():
            logits = model(input_ids=torch.tensor([ids]))["logits"]
        ids.append(int(logits[-1, : model.cfg.vocab_size].argmax()))
    return ids


def _gen(eng, prompts, n_new):
    _, ids = eng.generate(prompts_token_ids=prompts, return_token_ids=True,
                          generation_config=GenerationConfig(max_new_tokens=n_new))
    return ids


def _both(model, kw, waves, n_new, drafter=None):
    """Run `waves` (lists of prompts, one generate call each) with caching on and off; returns (on, off, engine)."""
    outs = []
    for on in (True, False):
        eng = InferenceEngine(model, None, InferenceConfig(enable_prefix_caching=on, **kw))
        if drafter is not None:
            eng.enable_spec_dec(drafter, n_spec_tokens=3)
        outs.append([_gen(eng, w, n_new) for w in waves])
        if on:
            eng_on = eng
    return outs[0], outs[1], eng_on


SYS = [5, 9, 13, 200, 7, 21, 22, 23, 24, 25, 26, 27, 28, 29, 30, 31, 32, 33]     # > 2 blocks of 8


def test_engine_shared_system_prompt_continuous_batching():
    torch.manual_seed(0)
    model = build_model("llama-tiny").float().eval()
    kw = dict(max_batch_size=3, max_input_len=40, max_output_len=6, block_size=BS, dtype="fp32", ignore_eos=True)
    waves = [[SYS + [40, 41]], [SYS + [50 + i, 60 + i, 70] for i in range(5)]]
    on, off, eng = _both(model, kw, waves, 6)
    assert on == off
    for w, got in zip(waves, on):
        for p, g in zip(w, got):
            assert g == _naive_greedy(model, p, 6)
    assert eng.request_handler.cache_manager.prefix_cache_stats["hit_tokens"] > 0


def test_engine_two_turn_chat_hits_the_first_turn():
    torch.manual_seed(0)
    model = build_model("llama-tiny").float().eval()
    kw = dict(max_batch_size=2, max_input_len=64, max_output_len=8, block_size=BS, dtype="fp32", ignore_eos=True)
    eng = InferenceEngine(model, None, InferenceConfig(enable_prefix_caching=True, **kw))
    turn1 = _gen(eng, [SYS + [40, 41, 42]], 8)[0]
    mgr = eng.request_handler.cache_manager
    before = mgr.prefix_cache_stats["hit_tokens"]
    turn2 = turn1 + [77, 78, 79]
    got = _gen(eng, [turn2], 6)[0]
    # every full block of turn 1 but the one holding its last sampled token is cached
    assert mgr.prefix_cache_stats["hit_tokens"] - before == (len(turn1) - 1) // BS * BS
    assert got == _naive_greedy(model, turn2, 6)


def test_engine_speculative_decoding_with_prefix_caching():
    torch.manual_seed(0)
    model = build_model("llama-tiny").float().eval()
    torch.manual_seed(1)
    drafter = build_model(get_config("llama-tiny", num_hidden_layers=1)).float().eval()
    kw = dict(max_batch_size=2, max_input_len=48, max_output_len=10, block_size=BS, dtype="fp32", ignore_eos=True,
              max_n_spec_tokens=4)
    waves = [[SYS + [40]], [SYS + [41, 42], SYS + [43]]]
    on, off, eng = _both(model, kw, waves, 10, drafter=drafter)
    for a, b in zip(on, off):
        for x, y in zip(a, b):
            assert x[:len(y)] == y[:len(x)]
    for w, got in zip(waves, on):
        for p, g in zip(w, got):
            ref = _naive_greedy(model, p, 10)
            assert g[:len(ref)] == ref
    assert eng.request_handler.cache_manager.prefix_cache_stats["hit_tokens"] > 0


def test_engine_sliding_window_with_prefix_caching():
    torch.manual_seed(0)
    model = build_model(get_config("mistral-tiny", sliding_window=6)).float().eval()
    kw = dict(max_batch_size=2, max_input_len=40, max_output_len=6, block_size=BS, dtype="fp32", ignore_eos=True)
    waves = [[SYS + [40, 41]], [SYS + [50, 51, 52], SYS + [53]]]
    on, off, eng = _both(model, kw, waves, 6)
    assert on == off
    for w, got in zip(waves, on):
        for p, g in zip(w, got):
            assert g == _naive_greedy(model, p, 6)
    assert eng.request_handler.cache_manager.prefix_cache_stats["hit_tokens"] > 0


def test_engine_alibi_with_prefix_caching():
    torch.manual_seed(0)
    model = build_model("baichuan-tiny").float().eval()
    model.fold_norm_head()
    kw = dict(max_batch_size=2, max_input_len=40, max_output_len=5, block_size=BS, dtype="fp32", ignore_eos=True)
    waves = [[SYS + [40, 41]], [SYS + [50, 51, 52], SYS + [53]]]
    on, off, eng = _both(model, kw, waves, 5)
    assert on == off
    for w, got in zip(waves, on):
        for p, g in zip(w, got):
            assert g == _naive_greedy(model, p, 5)
    assert eng.request_handler.cache_manager.prefix_cache_stats["hit_tokens"] > 0


def test_engine_oversubscribed_cache_recycles_and_rehits():
    """A cache with fewer free blocks than the running sequences grow into: sequences are recycled, their written
    blocks indexed on the way out and hit again when they are re-admitted."""
    torch.manual_seed(0)
    model = build_model("llama-tiny").float().eval()
    kw = dict(max_batch_size=3, max_input_len=32, max_output_len=9, block_size=BS, dtype="fp32", ignore_eos=True)
    prompts = [SYS[:16] + [40 + i] for i in range(3)]
    eng = InferenceEngine(model, None, InferenceConfig(enable_prefix_caching=True, **kw))
    mgr = eng.request_handler.cache_manager
    mgr._take_free_blocks(mgr.num_available_blocks - 9)       # 9 blocks left: the three prompts fill them
    recycled = []
    orig = eng.request_handler._recycle_last

    def spy():
        recycled.append(1)
        orig()

    eng.request_handler._recycle_last = spy
    got = _gen(eng, prompts, 9)
    plain = InferenceEngine(model, None, InferenceConfig(**kw))
    plain.request_handler.cache_manager._take_free_blocks(plain.request_handler.cache_manager.num_available_blocks - 9)
    assert got == _gen(plain, prompts, 9)
    for p, g in zip(prompts, got):
        ref = _naive_greedy(model, p, 9)      # a recycled sequence starts a new generation budget when re-admitted
        assert g[:len(ref)] == ref
    assert recycled, "the cache was not over-subscribed"
    assert mgr.prefix_cache_stats["hit_tokens"] > 0


def test_shared_blocks_are_immutable():
    torch.manual_seed(0)
    model = build_model("llama-tiny").float().eval()
    kw = dict(max_batch_size=2, max_input_len=40, max_output_len=6, block_size=BS, dtype="fp32", ignore_eos=True)
    eng = InferenceEngine(model, None, InferenceConfig(enable_prefix_caching=True, **kw))
    _gen(eng, [SYS + [40, 41]], 6)
    mgr = eng.request_handler.cache_manager
    indexed = sorted(mgr._block_entry)
    assert indexed
    k_caches, v_caches = mgr.get_kv_cache()
    snap = [(k[indexed].clone(), v[indexed].clone()) for k, v in zip(k_caches, v_caches)]
    _gen(eng, [SYS + [50, 51, 52], SYS + [53]], 6)
    assert mgr.prefix_cache_stats["hit_tokens"] > 0
    for (k0, v0), k, v in zip(snap, k_caches, v_caches):
        assert torch.equal(k[indexed], k0) and torch.equal(v[indexed], v0)


# ---------------------------------------------------------------------------------------------------- rejections
def test_prefix_caching_rejects_streamingllm():
    with pytest.raises(AssertionError, match="enable_streamingllm"):
        InferenceConfig(enable_prefix_caching=True, enable_streamingllm=True, block_size=8, generated_token_size=16)


def test_rpc_engine_rejects_prefix_caching():
    from colossalai_b200.inference.core.rpc_engine import RPCInferenceEngine

    cfg = InferenceConfig(max_batch_size=2, max_input_len=16, max_output_len=6, block_size=8, dtype="fp32",
                          enable_prefix_caching=True)
    with pytest.raises(ValueError, match="RPC"):
        RPCInferenceEngine("llama-tiny", None, cfg)


def test_cuda_envelope_of_prefix_caching():
    """What a CUDA engine refuses at construction (the check itself needs no GPU)."""
    llama = get_config("llama-tiny", head_dim=64)
    ok = InferenceConfig(dtype="bf16", enable_prefix_caching=True)
    assert prefix_caching_unsupported(ok, llama) is None
    assert prefix_caching_unsupported(InferenceConfig(dtype="fp16"), get_config("llama-tiny", head_dim=128)) is None
    assert "kv_cache_dtype" in prefix_caching_unsupported(InferenceConfig(dtype="bf16", kv_cache_dtype="fp8"), llama)
    assert "fp16 or bf16" in prefix_caching_unsupported(InferenceConfig(dtype="fp32"), llama)
    assert "MLA" in prefix_caching_unsupported(ok, get_config("deepseek_v3-tiny"))
    assert "head_dim" in prefix_caching_unsupported(ok, get_config("llama-tiny"))         # head_dim 16
