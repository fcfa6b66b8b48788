"""Speculative verification in one paged-attention pass (CPU tier): `paged_decode_attention(..., q_len=n)` attends n
query tokens per sequence, each over the cache up to its own position, and the engine verifies drafted tokens with it -
including ALiBi models, which could not speculate before, and sliding-window models."""
import pytest
import torch

from colossalai_b200.inference import InferenceConfig, InferenceEngine
from colossalai_b200.inference.config import GenerationConfig
from colossalai_b200.models import build_model, get_config
from colossalai_b200.ops import inference as iops


def _per_row_reference(q, kc, vc, tables, lens, q_len, **kw):
    """The verification the runtime used to run: one single-query reference call per query position."""
    n = lens.numel()
    qs = q.view(n, q_len, *q.shape[1:])
    outs = [iops.paged_decode_attention_ref(qs[:, j].contiguous(), kc, vc, tables, lens - (q_len - 1 - j), **kw)
            for j in range(q_len)]
    return torch.stack(outs, 1).reshape(q.shape)


@pytest.mark.parametrize("fp8", [False, True])
@pytest.mark.parametrize("alibi", [False, True])
@pytest.mark.parametrize("window", [None, 3, 9])
@pytest.mark.parametrize("q_len", [1, 2, 4])
def test_reference_q_len_equals_per_row_loop(fp8, alibi, window, q_len):
    torch.manual_seed(q_len)
    bs, Hkv, G, D, nb = 4, 2, 3, 16, 12
    kc, vc = torch.randn(nb, bs, Hkv, D), torch.randn(nb, bs, Hkv, D)
    if fp8:
        kc, vc = (c.to(torch.float8_e5m2).view(torch.uint8) for c in (kc, vc))
    tables = torch.randperm(nb)[:9].to(torch.int32).view(3, 3)
    lens = torch.tensor([q_len, 7, 12], dtype=torch.int32)
    q = torch.randn(3 * q_len, Hkv * G, D)
    kw = dict(window=window)
    if alibi:
        kw["alibi_slopes"] = torch.tensor([2 ** (-(i + 1)) for i in range(Hkv * G)])
    got = iops.paged_decode_attention(q, kc, vc, tables, lens, q_len=q_len, **kw)       # CPU: the reference path
    assert torch.equal(got, iops.paged_decode_attention_ref(q, kc, vc, tables, lens, q_len=q_len, **kw))
    assert torch.equal(got, _per_row_reference(q, kc, vc, tables, lens, q_len, **kw))


# (num_seqs, kv_heads, max_len) -> (splits, part_len) on 132 SMs (H100 SXM), as computed by the native
# `cb_decode_num_splits` that `decode_splits` replaces.  A verify pass uses the decode step's splits, which keeps each
# of its rows bitwise equal to the single-query result.
_SPLITS_132_SMS = {
    (1, 8, 1): (1, 32), (1, 8, 31): (1, 32), (1, 8, 100): (2, 64), (1, 8, 1000): (16, 64), (1, 8, 4096): (64, 64),
    (1, 8, 4097): (65, 64), (1, 8, 16384): (256, 64), (1, 16, 16384): (128, 128),
    (16, 8, 1): (1, 32), (16, 8, 31): (1, 32), (16, 8, 100): (2, 64), (16, 8, 1000): (16, 64),
    (16, 8, 4096): (16, 256), (16, 8, 4097): (17, 256), (16, 8, 16384): (17, 992), (16, 16, 4096): (9, 480),
    (64, 8, 1): (1, 32), (64, 8, 31): (1, 32), (64, 8, 100): (2, 64), (64, 8, 1000): (5, 224),
    (64, 8, 4096): (5, 832), (64, 8, 4097): (5, 832), (64, 8, 16384): (5, 3296), (64, 16, 1000): (3, 352),
}


@pytest.mark.parametrize("shape", sorted(_SPLITS_132_SMS))
def test_decode_splits_pinned_table(shape):
    assert iops.decode_splits(*shape, 132) == _SPLITS_132_SMS[shape]


def _spec_vs_plain(model, cfg_kw, prompts, n_new, n_spec):
    torch.manual_seed(1)
    drafter = build_model(get_config("llama-tiny", num_hidden_layers=1)).float().eval()
    gen = GenerationConfig(max_new_tokens=n_new)
    _, ref_ids = InferenceEngine(model, None, InferenceConfig(**cfg_kw)).generate(
        prompts_token_ids=prompts, return_token_ids=True, generation_config=gen)
    spec = InferenceEngine(model, None, InferenceConfig(**cfg_kw))
    spec.enable_spec_dec(drafter, n_spec_tokens=n_spec)
    _, got_ids = spec.generate(prompts_token_ids=prompts, return_token_ids=True, generation_config=gen)
    for p, r, g in zip(prompts, ref_ids, got_ids):
        assert len(g) >= len(p) + n_new
        assert g[: len(r)] == r, (r, g)


def test_alibi_engine_speculative_decoding_matches_plain_greedy():
    torch.manual_seed(0)
    model = build_model("baichuan-tiny").float().eval()
    model.fold_norm_head()
    cfg_kw = dict(max_batch_size=2, max_input_len=16, max_output_len=10, block_size=8, dtype="fp32",
                  use_cuda_graph=False, ignore_eos=True, max_n_spec_tokens=4)
    _spec_vs_plain(model, cfg_kw, [[5, 9, 13, 200, 7, 8, 9, 10, 11], [11, 3, 77]], 8, 3)


def test_sliding_window_engine_speculative_decoding_matches_plain_greedy():
    torch.manual_seed(0)
    model = build_model(get_config("mistral-tiny", sliding_window=6)).float().eval()
    cfg_kw = dict(max_batch_size=2, max_input_len=16, max_output_len=14, block_size=8, dtype="fp32",
                  use_cuda_graph=False, ignore_eos=True, max_n_spec_tokens=4)
    _spec_vs_plain(model, cfg_kw, [[5, 9, 13, 200, 7, 21, 22, 23, 24, 25, 26], [11, 3, 8]], 10, 4)
