"""fp8 (e5m2) paged KV cache through the engine (CPU tier): the cache stores K/V rounded to e5m2, prefill attends over
the step's exact K/V, and everything read back from the cache is the decoded e5m2 value.  The oracle is an engine with
a full-precision cache whose writes store `k.to(float8_e5m2)` values: its greedy tokens must be identical."""
import pytest
import torch

from colossalai_b200.inference import InferenceConfig, InferenceEngine
from colossalai_b200.inference.config import GenerationConfig
from colossalai_b200.models import build_model, get_config
from colossalai_b200.ops import inference as iops


def _generate(model, cfg_kw, prompts, n_new):
    eng = InferenceEngine(model, None, InferenceConfig(**cfg_kw))
    _, ids = eng.generate(prompts_token_ids=prompts, return_token_ids=True,
                          generation_config=GenerationConfig(max_new_tokens=n_new))
    return eng, ids


def _rounded_write_oracle(monkeypatch, model, cfg_kw, prompts, n_new):
    """Tokens of a default-cache engine whose cache writes store the e5m2-rounded K/V values."""
    write = iops.kv_cache_write

    def rounded_write(k, v, k_cache, v_cache, *args):
        write(k.to(torch.float8_e5m2).to(k.dtype), v.to(torch.float8_e5m2).to(v.dtype), k_cache, v_cache, *args)

    with monkeypatch.context() as m:
        m.setattr(iops, "kv_cache_write", rounded_write)
        return _generate(model, cfg_kw, prompts, n_new)[1]


def _assert_fp8_matches_oracle(monkeypatch, model, cfg_kw, prompts, n_new):
    eng, got = _generate(model, dict(cfg_kw, kv_cache_dtype="fp8"), prompts, n_new)
    k_caches, _ = eng.request_handler.get_kvcache()
    assert k_caches[0].dtype == torch.uint8 and k_caches[0].any()
    ref = _rounded_write_oracle(monkeypatch, model, cfg_kw, prompts, n_new)
    assert got == ref
    return got


def test_fp8_engine_matches_rounded_write_oracle_with_continuous_batching(monkeypatch):
    torch.manual_seed(0)
    model = build_model("llama-tiny").float().eval()
    cfg_kw = dict(max_batch_size=3, max_input_len=24, max_output_len=8, block_size=8, dtype="fp32",
                  use_cuda_graph=False, ignore_eos=True)
    prompts = [[5, 9, 13, 200, 7], [11, 3], [400, 401, 402, 403, 404, 405, 406, 407, 408, 409], [17] * 6, [99, 98, 97]]
    got = _assert_fp8_matches_oracle(monkeypatch, model, cfg_kw, prompts, 8)
    assert all(len(g) == len(p) + 8 for p, g in zip(prompts, got))


def test_fp8_engine_sliding_window_matches_rounded_write_oracle(monkeypatch):
    torch.manual_seed(0)
    model = build_model(get_config("mistral-tiny", sliding_window=6)).float().eval()
    cfg_kw = dict(max_batch_size=2, max_input_len=16, max_output_len=10, block_size=8, dtype="fp32",
                  use_cuda_graph=False, ignore_eos=True)
    prompts = [[5, 9, 13, 200, 7, 21, 22, 23, 24, 25, 26], [11, 3, 8]]
    _assert_fp8_matches_oracle(monkeypatch, model, cfg_kw, prompts, 10)


def test_fp8_engine_alibi_matches_rounded_write_oracle(monkeypatch):
    torch.manual_seed(0)
    model = build_model("baichuan-tiny").float().eval()
    model.fold_norm_head()
    cfg_kw = dict(max_batch_size=2, max_input_len=16, max_output_len=6, block_size=8, dtype="fp32",
                  use_cuda_graph=False, ignore_eos=True)
    prompts = [[5, 9, 13, 200, 7, 8, 9, 10, 11], [11, 3, 77]]
    _assert_fp8_matches_oracle(monkeypatch, model, cfg_kw, prompts, 6)


def test_fp8_speculative_decoding_matches_plain_greedy(monkeypatch):
    torch.manual_seed(0)
    model = build_model("llama-tiny").float().eval()
    torch.manual_seed(1)
    drafter = build_model(get_config("llama-tiny", num_hidden_layers=1)).float().eval()
    cfg_kw = dict(max_batch_size=2, max_input_len=16, max_output_len=8, block_size=8, dtype="fp32",
                  max_n_spec_tokens=4)
    cfg = InferenceConfig(kv_cache_dtype="fp8", **cfg_kw)
    prompts = [[5, 9, 13, 200, 7], [11, 3, 4]]
    gen = GenerationConfig(max_new_tokens=8)
    _, ref_ids = InferenceEngine(model, None, cfg).generate(prompts_token_ids=prompts, return_token_ids=True,
                                                            generation_config=gen)
    assert ref_ids == _rounded_write_oracle(monkeypatch, model, cfg_kw, prompts, 8)
    spec = InferenceEngine(model, None, cfg)
    spec.enable_spec_dec(drafter, n_spec_tokens=3)
    _, got_ids = spec.generate(prompts_token_ids=prompts, return_token_ids=True, generation_config=gen)
    for r, g in zip(ref_ids, got_ids):
        n = min(len(r), len(g))
        assert r[:n] == g[:n], (r, g)


def _fp8_cache(shape, seed):
    torch.manual_seed(seed)
    x = torch.randn(shape) * 3
    return x.to(torch.float8_e5m2).view(torch.uint8), x.to(torch.float8_e5m2).float()


def test_gather_paged_kv_decodes_fp8_cache():
    from colossalai_b200.inference.modeling.models.glide_llama import gather_paged_kv

    cache_u8, values = _fp8_cache((5, 4, 2, 16), 0)
    table = torch.tensor([3, 0, 4], dtype=torch.int32)
    got = gather_paged_kv(cache_u8, table, 10, torch.float32)
    want = values[table.long()].reshape(-1, 2, 16)[:10]
    assert got.dtype == torch.float32 and torch.equal(got, want)
    assert torch.equal(gather_paged_kv(cache_u8, table, 10).float(), want)           # default: e5m2 values
    assert torch.equal(gather_paged_kv(values, table, 10), want)                      # float caches: as stored


def test_glide_glimpse_reads_fp8_cache_values():
    """The GLIDE drafter's cross-attention over an fp8 target cache equals the one over the decoded cache."""
    from colossalai_b200.inference.modeling.models import GlideLlamaConfig, GlideLlamaForCausalLM
    from colossalai_b200.inference.spec import GlideInput

    gcfg = GlideLlamaConfig(vocab_size=512, hidden_size=32, intermediate_size=64, num_hidden_layers=1,
                            num_attention_heads=2, num_key_value_heads=2, max_position_embeddings=256,
                            large_hidden_size=64, large_num_attention_heads=4, large_num_key_value_heads=2,
                            large_head_dim=16)
    torch.manual_seed(1)
    drafter = GlideLlamaForCausalLM(gcfg).float().eval()
    k_u8, k_val = _fp8_cache((4, 8, 2, 16), 2)
    v_u8, v_val = _fp8_cache((4, 8, 2, 16), 3)
    tables, lens = torch.tensor([[2, 0]], dtype=torch.int32), torch.tensor([11])
    ids = torch.tensor([[5, 6, 7]])

    def glide(kc, vc):
        g = GlideInput(block_tables=tables, large_k_cache=kc, large_v_cache=vc, sequence_lengths=lens,
                       n_spec_tokens=3)
        with torch.no_grad():
            return drafter(input_ids=ids, glide_input=g)["logits"]

    torch.testing.assert_close(glide(k_u8, v_u8), glide(k_val, v_val), atol=0, rtol=0)


@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16, torch.float16])
def test_reference_paths_roundtrip_e5m2(dtype):
    """Reference write stores torch.float8_e5m2 bytes; reference decode attention on the fp8 cache equals it on the
    decoded cache."""
    torch.manual_seed(0)
    bs, Hkv, D, nb = 4, 2, 16, 6
    kc, vc = torch.zeros(nb, bs, Hkv, D, dtype=torch.uint8), torch.zeros(nb, bs, Hkv, D, dtype=torch.uint8)
    tables = torch.tensor([[4, 1], [0, 5]], dtype=torch.int32)
    lens = [7, 5]
    seq = torch.repeat_interleave(torch.arange(2), torch.tensor(lens)).int()
    pos = torch.cat([torch.arange(n) for n in lens]).int()
    k, v = torch.randn(sum(lens), Hkv, D, dtype=dtype), torch.randn(sum(lens), Hkv, D, dtype=dtype)
    iops.kv_cache_write(k, v, kc, vc, tables, seq, pos)
    blk, slot = tables[seq.long(), (pos // bs).long()].long(), (pos % bs).long()
    assert torch.equal(kc[blk, slot], k.to(torch.float8_e5m2).view(torch.uint8))
    assert torch.equal(vc[blk, slot], v.to(torch.float8_e5m2).view(torch.uint8))
    q = torch.randn(2, 4, D, dtype=dtype)
    seq_lens = torch.tensor(lens, dtype=torch.int32)
    out = iops.paged_decode_attention(q, kc, vc, tables, seq_lens)
    deq_k, deq_v = (c.view(torch.float8_e5m2).to(dtype) for c in (kc, vc))
    assert torch.equal(out, iops.paged_decode_attention_ref(q, deq_k, deq_v, tables, seq_lens))
