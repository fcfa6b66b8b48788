"""Paged-KV inference kernels vs fp32 PyTorch references (reference: tests/test_infer/test_kernels/cuda/
test_{kv_cache_memcpy,flash_decoding_attention,convert_fp8}.py)."""
import pytest
import torch

from colossalai_b200.ops import inference as iops

pytestmark = pytest.mark.gpu


def _mk_cache(n_seqs, max_len, bs, Hkv, D, dtype, dev):
    max_blocks = (max_len + bs - 1) // bs
    nb = n_seqs * max_blocks + 3
    perm = torch.randperm(nb, device=dev)[: n_seqs * max_blocks].to(torch.int32)
    tables = perm.view(n_seqs, max_blocks).contiguous()
    kc = torch.randn(nb, bs, Hkv, D, device=dev, dtype=dtype)
    vc = torch.randn(nb, bs, Hkv, D, device=dev, dtype=dtype)
    return kc, vc, tables


@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16])
@pytest.mark.parametrize("D", [64, 128])
@pytest.mark.parametrize("Hq,Hkv", [(8, 8), (32, 8), (16, 2)])
@pytest.mark.parametrize("bs", [16, 64])
def test_paged_decode_attention(dtype, D, Hq, Hkv, bs):
    dev = torch.device("cuda")
    torch.manual_seed(0)
    n, max_len = 7, 700
    kc, vc, tables = _mk_cache(n, max_len, bs, Hkv, D, dtype, dev)
    lens = torch.tensor([1, 15, 16, 17, 300, 699, 700], device=dev, dtype=torch.int32)
    q = torch.randn(n, Hq, D, device=dev, dtype=dtype)
    out = iops.paged_decode_attention(q, kc, vc, tables, lens)
    ref = iops.paged_decode_attention_ref(q.float(), kc.float(), vc.float(), tables, lens)
    torch.testing.assert_close(out.float(), ref, atol=2e-2, rtol=2e-2)


def test_paged_decode_long_context_split_kv():
    dev = torch.device("cuda")
    torch.manual_seed(1)
    kc, vc, tables = _mk_cache(2, 8192, 16, 8, 128, torch.bfloat16, dev)
    lens = torch.tensor([8192, 4097], device=dev, dtype=torch.int32)
    q = torch.randn(2, 32, 128, device=dev, dtype=torch.bfloat16)
    out = iops.paged_decode_attention(q, kc, vc, tables, lens)
    ref = iops.paged_decode_attention_ref(q.float(), kc.float(), vc.float(), tables, lens)
    torch.testing.assert_close(out.float(), ref, atol=2e-2, rtol=2e-2)


def test_paged_decode_alibi():
    dev = torch.device("cuda")
    torch.manual_seed(2)
    kc, vc, tables = _mk_cache(3, 256, 16, 8, 128, torch.float16, dev)
    lens = torch.tensor([5, 100, 256], device=dev, dtype=torch.int32)
    q = torch.randn(3, 8, 128, device=dev, dtype=torch.float16)
    slopes = torch.tensor([2 ** (-(i + 1)) for i in range(8)], device=dev, dtype=torch.float32)
    out = iops.paged_decode_attention(q, kc, vc, tables, lens, alibi_slopes=slopes)
    ref = iops.paged_decode_attention_ref(q.float(), kc.float(), vc.float(), tables, lens, alibi_slopes=slopes)
    torch.testing.assert_close(out.float(), ref, atol=2e-2, rtol=2e-2)


# wider grid in the spirit of the reference's flash-decoding test
# (tests/test_infer/test_kernels/cuda/test_flash_decoding_attention.py:59-66: batch x block size x context x group size x
#  head dim x same / mixed context lengths, with and without ALiBi)
@pytest.mark.parametrize("bsz", [1, 7, 32])
@pytest.mark.parametrize("bs", [8, 16, 32])
@pytest.mark.parametrize("max_blocks", [1, 8, 67])
@pytest.mark.parametrize("group", [1, 4, 8])
@pytest.mark.parametrize("D", [64, 128, 256])
@pytest.mark.parametrize("same_len", [True, False])
def test_paged_decode_grid(bsz, bs, max_blocks, group, D, same_len):
    dev = torch.device("cuda")
    torch.manual_seed(bsz * 131 + bs * 17 + max_blocks + group + D)
    Hkv = 2
    Hq = Hkv * group
    max_len = bs * max_blocks
    kc, vc, tables = _mk_cache(bsz, max_len, bs, Hkv, D, torch.bfloat16, dev)
    lens = torch.full((bsz,), max_len, dtype=torch.int32) if same_len else torch.randint(1, max_len + 1, (bsz,)).int()
    lens = lens.to(dev)
    q = torch.randn(bsz, Hq, D, device=dev, dtype=torch.bfloat16)
    out = iops.paged_decode_attention(q, kc, vc, tables, lens)
    ref = iops.paged_decode_attention_ref(q.float(), kc.float(), vc.float(), tables, lens)
    torch.testing.assert_close(out.float(), ref, atol=2e-2, rtol=2e-2)


@pytest.mark.parametrize("D", [128, 256])          # tensor-core and CUDA-core kernels
@pytest.mark.parametrize("window", [1, 16, 100, 4096])
@pytest.mark.parametrize("alibi", [False, True])
def test_paged_decode_sliding_window(window, alibi, D):
    """`window_start` inside the split-KV kernel: only the last `window` cached tokens are visible."""
    dev = torch.device("cuda")
    torch.manual_seed(3)
    kc, vc, tables = _mk_cache(5, 3000, 16, 4, D, torch.bfloat16, dev)
    lens = torch.tensor([1, 15, 100, 1025, 3000], device=dev, dtype=torch.int32)
    q = torch.randn(5, 16, D, device=dev, dtype=torch.bfloat16)
    slopes = torch.tensor([2 ** (-(i + 1) / 2) for i in range(16)], device=dev, dtype=torch.float32) if alibi else None
    out = iops.paged_decode_attention(q, kc, vc, tables, lens, alibi_slopes=slopes, window=window)
    ref = iops.paged_decode_attention_ref(q.float(), kc.float(), vc.float(), tables, lens, alibi_slopes=slopes,
                                          window=window)
    torch.testing.assert_close(out.float(), ref, atol=2e-2, rtol=2e-2)


@pytest.mark.parametrize("tokens,Hkv,D", [(1, 8, 128), (33, 2, 64), (4096, 8, 128), (515, 4, 256)])
def test_kv_cache_write_vectorised_shapes(tokens, Hkv, D):
    """The 16-byte path of `cb_kv_cache_write` over prefill-sized token counts and strided (fused-QKV view) inputs."""
    dev = torch.device("cuda")
    torch.manual_seed(tokens)
    bs = 16
    n_seqs = max(1, tokens // 100)
    per = (tokens + n_seqs - 1) // n_seqs
    seq = (torch.arange(tokens, device=dev) // per).int()
    pos = (torch.arange(tokens, device=dev) % per).int()
    kc, vc, tables = _mk_cache(n_seqs, per, bs, Hkv, D, torch.bfloat16, dev)
    fused = torch.randn(tokens, 3 * Hkv * D, device=dev, dtype=torch.bfloat16)
    k = fused[:, Hkv * D: 2 * Hkv * D].view(tokens, Hkv, D)          # row stride 3 * Hkv * D
    v = fused[:, 2 * Hkv * D:].view(tokens, Hkv, D)
    kc.zero_(); vc.zero_()
    iops.kv_cache_write(k, v, kc, vc, tables, seq, pos)
    blk = tables[seq.long(), (pos // bs).long()].long()
    torch.testing.assert_close(kc[blk, (pos % bs).long()], k, atol=0, rtol=0)
    torch.testing.assert_close(vc[blk, (pos % bs).long()], v, atol=0, rtol=0)


@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16])
def test_kv_cache_write(dtype):
    dev = torch.device("cuda")
    torch.manual_seed(3)
    bs, Hkv, D = 16, 4, 128
    kc, vc, tables = _mk_cache(3, 64, bs, Hkv, D, dtype, dev)
    kc0, vc0 = kc.clone(), vc.clone()
    lens = [5, 33, 64]
    seq = torch.repeat_interleave(torch.arange(3), torch.tensor(lens)).to(dev, torch.int32)
    pos = torch.cat([torch.arange(l) for l in lens]).to(dev, torch.int32)
    T = sum(lens)
    kv = torch.randn(T, 2 * Hkv * D + 7, device=dev, dtype=dtype)   # strided views like a fused qkv output
    k = kv[:, : Hkv * D].view(T, Hkv, D)
    v = kv[:, Hkv * D: 2 * Hkv * D].view(T, Hkv, D)
    iops.kv_cache_write(k, v, kc, vc, tables, seq, pos)
    blk = tables[seq.long(), (pos // bs).long()].long()
    slot = (pos % bs).long()
    kc0[blk, slot] = k
    vc0[blk, slot] = v
    assert torch.equal(kc, kc0) and torch.equal(vc, vc0)


def test_convert_fp8_roundtrip():
    dev = torch.device("cuda")
    x = torch.randn(1000, 130, device=dev, dtype=torch.bfloat16)
    q = iops.convert_fp8(x, True)
    ref = x.to(torch.float8_e5m2)
    assert torch.equal(q, ref.view(torch.uint8))
    back = iops.convert_fp8(q, False, torch.bfloat16)
    assert torch.equal(back, ref.to(torch.bfloat16))


def test_engine_gpu_cuda_graph_matches_eager():
    from colossalai_b200.inference import InferenceConfig, InferenceEngine
    from colossalai_b200.inference.config import GenerationConfig
    from colossalai_b200.kernel import loader
    from colossalai_b200.models import build_model, get_config

    torch.manual_seed(0)
    # head_dim 64 so the decode step runs the native paged kernel (the torch reference path syncs and cannot be captured)
    model = build_model(get_config("llama-tiny", hidden_size=256, intermediate_size=512)).to(torch.bfloat16).cuda().eval()
    loader.launch_counter.reset()
    prompts = [[5, 9, 13, 200, 7], [11, 3], [400, 401, 402, 403, 404, 405, 406, 407, 408, 409]]
    outs = []
    for graph in (False, True):
        cfg = InferenceConfig(max_batch_size=4, max_input_len=32, max_output_len=12, block_size=16, dtype="bf16",
                              use_cuda_graph=graph)
        eng = InferenceEngine(model, None, cfg)
        _, ids = eng.generate(prompts_token_ids=prompts, return_token_ids=True,
                              generation_config=GenerationConfig(max_new_tokens=12))
        outs.append(ids)
    assert outs[0] == outs[1]
    assert loader.launch_counter.by_name.get("paged_decode_attention", 0) > 0
