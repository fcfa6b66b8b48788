"""fp8 (e5m2) paged KV cache on the native kernels: `cb_kv_cache_write` stores the bytes torch.float8_e5m2 would, and
`cb_paged_decode_attention` on an fp8 cache is bitwise the 16-bit kernel on the decoded cache (same tiles, lanes and
summation order; e5m2 decodes exactly to fp16 / bf16)."""
import pytest
import torch

from colossalai_b200.ops import inference as iops

pytestmark = pytest.mark.gpu


def _e5m2(x):
    return x.to(torch.float8_e5m2).view(torch.uint8)


def _mk_fp8_cache(n_seqs, max_len, bs, Hkv, D, dev):
    max_blocks = (max_len + bs - 1) // bs
    nb = n_seqs * max_blocks + 3
    tables = torch.randperm(nb, device=dev)[: n_seqs * max_blocks].to(torch.int32).view(n_seqs, max_blocks).contiguous()
    kc = _e5m2(torch.randn(nb, bs, Hkv, D, device=dev))
    vc = _e5m2(torch.randn(nb, bs, Hkv, D, device=dev))
    return kc, vc, tables


def _check_decode(q, kc, vc, tables, lens, **kw):
    """fp8 kernel == 16-bit kernel on the decoded cache (bitwise), and close to the fp32 reference."""
    kd, vd = (c.view(torch.float8_e5m2).to(q.dtype) for c in (kc, vc))
    out = iops.paged_decode_attention(q, kc, vc, tables, lens, **kw)
    assert torch.equal(out, iops.paged_decode_attention(q, kd, vd, tables, lens, **kw))
    ref = iops.paged_decode_attention_ref(q.float(), kd.float(), vd.float(), tables, lens, **kw)
    torch.testing.assert_close(out.float(), ref, atol=2e-2, rtol=2e-2)


@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16])
@pytest.mark.parametrize("tokens,Hkv,D", [(1, 8, 128), (33, 2, 64), (4096, 8, 128), (515, 4, 256)])
def test_kv_cache_write_fp8_vectorised(tokens, Hkv, D, dtype):
    dev = torch.device("cuda")
    torch.manual_seed(tokens)
    bs = 16
    n_seqs = max(1, tokens // 100)
    per = (tokens + n_seqs - 1) // n_seqs
    seq = (torch.arange(tokens, device=dev) // per).int()
    pos = (torch.arange(tokens, device=dev) % per).int()
    kc, vc, tables = _mk_fp8_cache(n_seqs, per, bs, Hkv, D, dev)
    fused = torch.randn(tokens, 3 * Hkv * D, device=dev, dtype=dtype) * 4
    k = fused[:, Hkv * D: 2 * Hkv * D].view(tokens, Hkv, D)          # row stride 3 * Hkv * D
    v = fused[:, 2 * Hkv * D:].view(tokens, Hkv, D)
    kc.zero_(); vc.zero_()
    iops.kv_cache_write(k, v, kc, vc, tables, seq, pos)
    blk = tables[seq.long(), (pos // bs).long()].long()
    assert torch.equal(kc[blk, (pos % bs).long()], _e5m2(k))
    assert torch.equal(vc[blk, (pos % bs).long()], _e5m2(v))


@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16])
def test_kv_cache_write_fp8_scalar_fallback(dtype):
    dev = torch.device("cuda")
    torch.manual_seed(3)
    bs, Hkv, D = 16, 4, 128
    kc, vc, tables = _mk_fp8_cache(3, 64, bs, Hkv, D, dev)
    kc0, vc0 = kc.clone(), vc.clone()
    lens = [5, 33, 64]
    seq = torch.repeat_interleave(torch.arange(3), torch.tensor(lens)).to(dev, torch.int32)
    pos = torch.cat([torch.arange(n) for n in lens]).to(dev, torch.int32)
    T = sum(lens)
    kv = torch.randn(T, 2 * Hkv * D + 7, device=dev, dtype=dtype)   # row stride not a multiple of 8: scalar kernel
    k = kv[:, : Hkv * D].view(T, Hkv, D)
    v = kv[:, Hkv * D: 2 * Hkv * D].view(T, Hkv, D)
    iops.kv_cache_write(k, v, kc, vc, tables, seq, pos)
    blk, slot = tables[seq.long(), (pos // bs).long()].long(), (pos % bs).long()
    kc0[blk, slot] = _e5m2(k)
    vc0[blk, slot] = _e5m2(v)
    assert torch.equal(kc, kc0) and torch.equal(vc, vc0)


@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16])
@pytest.mark.parametrize("bsz", [1, 7, 32])
@pytest.mark.parametrize("bs", [8, 16, 32])
@pytest.mark.parametrize("max_blocks", [1, 8, 67])
@pytest.mark.parametrize("group", [1, 4, 8])
@pytest.mark.parametrize("D", [64, 128, 256])
@pytest.mark.parametrize("same_len", [True, False])
def test_paged_decode_fp8_grid(bsz, bs, max_blocks, group, D, same_len, dtype):
    dev = torch.device("cuda")
    torch.manual_seed(bsz * 131 + bs * 17 + max_blocks + group + D)
    Hkv = 2
    max_len = bs * max_blocks
    kc, vc, tables = _mk_fp8_cache(bsz, max_len, bs, Hkv, D, dev)
    lens = torch.full((bsz,), max_len, dtype=torch.int32) if same_len else torch.randint(1, max_len + 1, (bsz,)).int()
    q = torch.randn(bsz, Hkv * group, D, device=dev, dtype=dtype)
    _check_decode(q, kc, vc, tables, lens.to(dev))


def test_paged_decode_fp8_long_context_split_kv():
    dev = torch.device("cuda")
    torch.manual_seed(1)
    kc, vc, tables = _mk_fp8_cache(2, 8192, 16, 8, 128, dev)
    lens = torch.tensor([8192, 4097], device=dev, dtype=torch.int32)
    _check_decode(torch.randn(2, 32, 128, device=dev, dtype=torch.bfloat16), kc, vc, tables, lens)


@pytest.mark.parametrize("D", [128, 256])          # tensor-core and CUDA-core kernels
@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16])
def test_paged_decode_fp8_alibi(dtype, D):
    dev = torch.device("cuda")
    torch.manual_seed(2)
    kc, vc, tables = _mk_fp8_cache(3, 256, 16, 8, D, dev)
    lens = torch.tensor([5, 100, 256], device=dev, dtype=torch.int32)
    slopes = torch.tensor([2 ** (-(i + 1)) for i in range(8)], device=dev, dtype=torch.float32)
    _check_decode(torch.randn(3, 8, D, device=dev, dtype=dtype), kc, vc, tables, lens, alibi_slopes=slopes)


@pytest.mark.parametrize("D", [128, 256])          # tensor-core and CUDA-core kernels
@pytest.mark.parametrize("window", [1, 16, 100, 4096])
@pytest.mark.parametrize("alibi", [False, True])
def test_paged_decode_fp8_sliding_window(window, alibi, D):
    dev = torch.device("cuda")
    torch.manual_seed(3)
    kc, vc, tables = _mk_fp8_cache(5, 3000, 16, 4, D, dev)
    lens = torch.tensor([1, 15, 100, 1025, 3000], device=dev, dtype=torch.int32)
    slopes = torch.tensor([2 ** (-(i + 1) / 2) for i in range(16)], device=dev, dtype=torch.float32) if alibi else None
    _check_decode(torch.randn(5, 16, D, device=dev, dtype=torch.bfloat16), kc, vc, tables, lens,
                  alibi_slopes=slopes, window=window)


@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16])
@pytest.mark.parametrize("group", [1, 4, 8])
def test_paged_decode_fp8_simt_kernel(dtype, group):
    """The CUDA-core kernel (head_dim 256) around block and partition boundaries."""
    dev = torch.device("cuda")
    torch.manual_seed(4)
    kc, vc, tables = _mk_fp8_cache(7, 700, 16, 2, 256, dev)
    lens = torch.tensor([1, 15, 16, 17, 300, 699, 700], device=dev, dtype=torch.int32)
    _check_decode(torch.randn(7, 2 * group, 256, device=dev, dtype=dtype), kc, vc, tables, lens)


def test_engine_fp8_cache_native_graphs_and_rounded_write_oracle(monkeypatch):
    """bf16 model + fp8 cache: CUDA-graph decode == eager decode == a bf16-cache engine storing e5m2-rounded K/V, with
    the decode step on the native kernels (no conversion launches)."""
    from colossalai_b200.inference import InferenceConfig, InferenceEngine
    from colossalai_b200.inference.config import GenerationConfig
    from colossalai_b200.kernel import loader
    from colossalai_b200.models import build_model, get_config

    torch.manual_seed(0)
    model = build_model(get_config("llama-tiny", hidden_size=256, intermediate_size=512)).to(torch.bfloat16).cuda().eval()
    prompts = [[5, 9, 13, 200, 7], [11, 3], [400, 401, 402, 403, 404, 405, 406, 407, 408, 409]]
    kw = dict(max_batch_size=4, max_input_len=32, max_output_len=12, block_size=16, dtype="bf16", ignore_eos=True)

    def run(**extra):
        eng = InferenceEngine(model, None, InferenceConfig(**kw, **extra))
        _, ids = eng.generate(prompts_token_ids=prompts, return_token_ids=True,
                              generation_config=GenerationConfig(max_new_tokens=12))
        return eng, ids

    loader.launch_counter.reset()
    eng, eager = run(kv_cache_dtype="fp8", use_cuda_graph=False)
    counts = dict(loader.launch_counter.by_name)
    assert eng.request_handler.get_kvcache()[0][0].dtype == torch.uint8
    assert counts.get("paged_decode_attention", 0) > 0 and counts.get("kv_cache_write", 0) > 0
    assert counts.get("convert_fp8", 0) == 0
    eng, graphed = run(kv_cache_dtype="fp8", use_cuda_graph=True)
    assert eng.use_cuda_graph and eng.graph_runners
    assert graphed == eager

    write = iops.kv_cache_write

    def rounded_write(k, v, k_cache, v_cache, *args):
        write(k.to(torch.float8_e5m2).to(k.dtype), v.to(torch.float8_e5m2).to(v.dtype), k_cache, v_cache, *args)

    monkeypatch.setattr(iops, "kv_cache_write", rounded_write)
    _, oracle = run(use_cuda_graph=False)
    assert eager == oracle
