"""Speculative verification on the native kernel: `paged_decode_attention(..., q_len=n)` with n query tokens per
sequence is one tensor-core pass over the cache whose rows are (query token, q head) pairs.  Without a window every row
must be bitwise the single-query decode kernel's result for that token (same tile bases, splits and reduce; masked
positions add p = 0); the oracle is the per-position decode loop the runtime used to run."""
import ctypes

import pytest
import torch

from colossalai_b200.kernel import loader
from colossalai_b200.ops import inference as iops
from colossalai_b200.ops._dtypes import code

pytestmark = pytest.mark.gpu
CUDA_ERROR_INVALID_VALUE = 1


def _per_position(q, kc, vc, tables, lens, q_len, decode=None, **kw):
    """One single-query decode call per query position: query j of a sequence sees lens - (q_len - 1 - j) tokens."""
    decode = decode or iops.paged_decode_attention
    n = lens.numel()
    qs = q.view(n, q_len, *q.shape[1:])
    outs = [decode(qs[:, j].contiguous(), kc, vc, tables, lens - (q_len - 1 - j), **kw) for j in range(q_len)]
    return torch.stack(outs, 1).reshape(q.shape)


def _dense_ref(q, kc, vc, tables, lens, q_len, alibi_slopes=None, window=None):
    """fp32 reference over every sequence's whole block table, each query row masked to the positions it sees."""
    n, mb = tables.shape
    _, bs, Hkv, D = kc.shape
    Hq = q.shape[1]

    def values(c):
        c = c.view(torch.float8_e5m2) if c.dtype == torch.uint8 else c
        return c[tables.long()].float().reshape(n, mb * bs, Hkv, D).repeat_interleave(Hq // Hkv, dim=2)

    k, v = values(kc), values(vc)
    s = torch.einsum("njhd,nlhd->njhl", q.float().view(n, q_len, Hq, D), k) * D ** -0.5
    pos = torch.arange(mb * bs, device=q.device)
    len_j = lens.long()[:, None] - (q_len - 1 - torch.arange(q_len, device=q.device))[None]        # [n, q_len]
    if alibi_slopes is not None:
        s = s + alibi_slopes.float()[None, None, :, None] * (pos - (len_j[:, :, None, None] - 1))
    keep = pos < len_j[:, :, None]
    if window:
        keep &= pos >= len_j[:, :, None] - window
    s = s.masked_fill(~keep[:, :, None, :], float("-inf"))
    return torch.einsum("njhl,nlhd->njhd", s.softmax(-1), v).reshape(n * q_len, Hq, D)


def _caches(n_seqs, max_len, bs, Hkv, D, dev):
    max_blocks = (max_len + bs - 1) // bs
    nb = n_seqs * max_blocks + 3
    tables = torch.randperm(nb, device=dev)[: n_seqs * max_blocks].to(torch.int32).view(n_seqs, max_blocks).contiguous()
    return torch.randn(nb, bs, Hkv, D, device=dev), torch.randn(nb, bs, Hkv, D, device=dev), tables


def _as_cache(x, dtype, fp8):
    return x.to(torch.float8_e5m2).view(torch.uint8) if fp8 else x.to(dtype)


def _check(q, kc, vc, tables, lens, q_len, bitwise=True, **kw):
    out = iops.paged_decode_attention(q, kc, vc, tables, lens, q_len=q_len, **kw)
    loop = _per_position(q, kc, vc, tables, lens, q_len, **kw)
    if bitwise:
        assert torch.equal(out, loop)
    else:
        torch.testing.assert_close(out, loop, atol=2e-2, rtol=2e-2)
    torch.testing.assert_close(out.float(), _dense_ref(q, kc, vc, tables, lens, q_len, **kw), atol=2e-2, rtol=2e-2)


@pytest.mark.parametrize("bsz", [1, 7, 32])
@pytest.mark.parametrize("bs", [8, 16, 32])
@pytest.mark.parametrize("max_blocks", [1, 8, 67])
@pytest.mark.parametrize("group", [1, 4, 8])
@pytest.mark.parametrize("D", [64, 128])
@pytest.mark.parametrize("q_len", [2, 3, 4, 6, 9])
@pytest.mark.parametrize("same_len", [True, False])
def test_paged_verify_grid(bsz, bs, max_blocks, group, D, q_len, same_len):
    """q_len * group > 16 (e.g. group 4 with 6 tokens) spreads a kv head's rows over sibling warps."""
    max_len = bs * max_blocks
    if max_len < q_len:
        pytest.skip("context shorter than the verified tokens")
    dev = torch.device("cuda")
    torch.manual_seed(bsz * 131 + bs * 17 + max_blocks + group + D + q_len)
    Hkv = 2
    k, v, tables = _caches(bsz, max_len, bs, Hkv, D, dev)
    if same_len:
        lens = torch.full((bsz,), max_len, dtype=torch.int32)
    else:
        lens = torch.randint(q_len, max_len + 1, (bsz,)).int()
        lens[0] = q_len                                    # the whole sequence is the verified tokens
    lens = lens.to(dev)
    for dtype in (torch.bfloat16, torch.float16):
        q = torch.randn(bsz * q_len, Hkv * group, D, device=dev, dtype=dtype)
        for fp8 in (False, True):
            _check(q, _as_cache(k, dtype, fp8), _as_cache(v, dtype, fp8), tables, lens, q_len)


@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16])
@pytest.mark.parametrize("fp8", [False, True])
def test_paged_verify_alibi(dtype, fp8):
    dev = torch.device("cuda")
    torch.manual_seed(2)
    k, v, tables = _caches(3, 256, 16, 2, 128, dev)
    lens = torch.tensor([5, 100, 256], device=dev, dtype=torch.int32)
    slopes = torch.tensor([2 ** (-(i + 1)) for i in range(8)], device=dev, dtype=torch.float32)
    q = torch.randn(3 * 5, 8, 128, device=dev, dtype=dtype)
    _check(q, _as_cache(k, dtype, fp8), _as_cache(v, dtype, fp8), tables, lens, 5, alibi_slopes=slopes)


@pytest.mark.parametrize("window", [1, 16, 100, 4096])
@pytest.mark.parametrize("alibi", [False, True])
@pytest.mark.parametrize("fp8", [False, True])
def test_paged_verify_sliding_window(window, alibi, fp8):
    """A window starts the shared tile grid at the first row's window start: equal to the loop up to rounding."""
    dev = torch.device("cuda")
    torch.manual_seed(3)
    k, v, tables = _caches(5, 3000, 16, 4, 128, dev)
    lens = torch.tensor([5, 15, 100, 1025, 3000], device=dev, dtype=torch.int32)
    slopes = torch.tensor([2 ** (-(i + 1) / 2) for i in range(16)], device=dev, dtype=torch.float32) if alibi else None
    q = torch.randn(5 * 5, 16, 128, device=dev, dtype=torch.bfloat16)
    _check(q, _as_cache(k, torch.bfloat16, fp8), _as_cache(v, torch.bfloat16, fp8), tables, lens, 5, bitwise=False,
           alibi_slopes=slopes, window=window)


@pytest.mark.parametrize("fp8", [False, True])
@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16])
def test_paged_verify_long_context_split_kv(dtype, fp8):
    """8192-token split-KV; some rows of a sequence end below the start of a split its last row reaches."""
    dev = torch.device("cuda")
    torch.manual_seed(1)
    _, P = iops.decode_splits(3, 8, 8192, iops.sm_count(torch.cuda.current_device()))
    k, v, tables = _caches(3, 8192, 16, 8, 128, dev)
    lens = torch.tensor([8192, 2 * P + 1, 3 * P + 2], device=dev, dtype=torch.int32)
    q = torch.randn(3 * 6, 32, 128, device=dev, dtype=dtype)
    _check(q, _as_cache(k, dtype, fp8), _as_cache(v, dtype, fp8), tables, lens, 6)


@pytest.mark.parametrize("fp8", [False, True])
@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16])
def test_paged_verify_cuda_core_shapes_run_the_loop(dtype, fp8):
    """Head_dim 256, which only the CUDA-core kernel serves, runs one decode call per query position: exactly the
    loop's output.  The native launcher itself refuses q_len > 1 there and launches nothing."""
    D = 256
    dev = torch.device("cuda")
    torch.manual_seed(4)
    k, v, tables = _caches(4, 300, 16, 2, D, dev)
    kc, vc = _as_cache(k, dtype, fp8), _as_cache(v, dtype, fp8)
    lens = torch.tensor([3, 17, 200, 300], device=dev, dtype=torch.int32)
    q = torch.randn(4 * 3, 8, D, device=dev, dtype=dtype)
    loader.launch_counter.reset()
    out = iops.paged_decode_attention(q, kc, vc, tables, lens, q_len=3)
    assert loader.launch_counter.by_name["paged_decode_attention"] == 2 * 3
    assert torch.equal(out, _per_position(q, kc, vc, tables, lens, 3))

    q2, out2 = q[: 4 * 2].contiguous(), torch.zeros(4 * 2, 8, D, device=dev, dtype=dtype)
    o_part, ml_part = torch.empty(4 * 2, 8, 1, D, device=dev), torch.empty(4 * 2, 8, 1, 2, device=dev)
    err = iops._get_lib().cb_paged_decode_attention(
        loader.ptr(q2), loader.ptr(kc), loader.ptr(vc), loader.ptr(tables), loader.ptr(lens), loader.ptr(out2),
        loader.ptr(o_part), loader.ptr(ml_part), 4, 2, 8, 2, D, 16, tables.shape[1], 1, 320, ctypes.c_float(D ** -0.5),
        loader.ptr(None), ctypes.c_int64(q2.stride(0)), ctypes.c_int64(out2.stride(0)), code(dtype),
        iops._cache_code(kc), 0, loader.stream_ptr())
    torch.cuda.synchronize()
    assert err == CUDA_ERROR_INVALID_VALUE
    assert not out2.any()


def test_paged_verify_is_one_native_call():
    dev = torch.device("cuda")
    torch.manual_seed(5)
    k, v, tables = _caches(4, 512, 16, 8, 128, dev)
    lens = torch.tensor([4, 60, 300, 512], device=dev, dtype=torch.int32)
    q = torch.randn(4 * 4, 32, 128, device=dev, dtype=torch.bfloat16)
    loader.launch_counter.reset()
    iops.paged_decode_attention(q, k.bfloat16(), v.bfloat16(), tables, lens, q_len=4)
    assert loader.launch_counter.by_name["paged_decode_attention"] == 2


@pytest.mark.parametrize("fp8", [False, True])
@pytest.mark.parametrize("name,overrides", [
    ("llama-tiny", dict(hidden_size=256, intermediate_size=512)),                                   # D 64, G 2
    ("llama-tiny", dict(hidden_size=512, num_key_value_heads=1, intermediate_size=512)),            # D 128, G 4
    ("baichuan-tiny", dict(hidden_size=256, intermediate_size=512)),                                # ALiBi, D 64
])
def test_engine_speculative_verify_is_one_pass(monkeypatch, name, overrides, fp8):
    """bf16 engines with a 1-layer drafter: the tokens equal those of the same engine verifying with the
    per-position loop, and a verify pass issues 2 decode-attention launches per layer instead of 2 x (n + 1)."""
    from colossalai_b200.inference import InferenceConfig, InferenceEngine
    from colossalai_b200.inference.config import GenerationConfig
    from colossalai_b200.models import build_model, get_config

    torch.manual_seed(0)
    model = build_model(get_config(name, **overrides)).to(torch.bfloat16).cuda().eval()
    if name == "baichuan-tiny":
        model.fold_norm_head()
    torch.manual_seed(1)
    drafter = build_model(get_config("llama-tiny", num_hidden_layers=1, hidden_size=256, intermediate_size=512))
    drafter = drafter.to(torch.bfloat16).cuda().eval()
    layers, n_spec = model.cfg.num_hidden_layers, 4
    prompts = [[5, 9, 13, 200, 7], [11, 3], [400, 401, 402, 403, 404, 405, 406, 407, 408, 409]]
    cfg = InferenceConfig(max_batch_size=4, max_input_len=32, max_output_len=20, block_size=16, dtype="bf16",
                          use_cuda_graph=False, ignore_eos=True, kv_cache_dtype="fp8" if fp8 else None)

    def run():
        eng = InferenceEngine(model, None, cfg)
        eng.enable_spec_dec(drafter, n_spec_tokens=n_spec)
        verify = []
        set_step = eng.kv_runtime.set_step

        def spy(block_tables, seq_lens, is_prompt, device, q_per_seq=1):
            if not is_prompt:
                verify.append(q_per_seq)
            return set_step(block_tables, seq_lens, is_prompt, device, q_per_seq)

        eng.kv_runtime.set_step = spy
        loader.launch_counter.reset()
        _, ids = eng.generate(prompts_token_ids=prompts, return_token_ids=True,
                              generation_config=GenerationConfig(max_new_tokens=16))
        assert verify and set(verify) == {n_spec + 1}
        return ids, len(verify), loader.launch_counter.by_name.get("paged_decode_attention", 0)

    ids, passes, launches = run()
    assert launches == 2 * layers * passes
    single = iops.paged_decode_attention

    def per_position(q, kc, vc, tables, lens, scale=None, alibi_slopes=None, window=None, q_len=1):
        return _per_position(q, kc, vc, tables, lens, q_len, decode=single, scale=scale, alibi_slopes=alibi_slopes,
                             window=window)

    monkeypatch.setattr(iops, "paged_decode_attention", per_position)
    loop_ids, loop_passes, loop_launches = run()
    assert loop_ids == ids
    assert loop_launches == 2 * layers * (n_spec + 1) * loop_passes
    for p, g in zip(prompts, ids):
        assert len(g) >= len(p) + 16
