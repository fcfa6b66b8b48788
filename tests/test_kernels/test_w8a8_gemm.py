"""SmoothQuant W8A8 on the GPU (`ops/w8a8.py`: the int8 mode of `cb_int8_quant_rows` in kernel/csrc/quant.cu and
`cb_gemm_w8a8` in kernel/csrc/gemm_wgmma.cu).

Integer sums are exact, so every check here is bitwise:
* the native quantiser equals `quantize_activation_per_token` (and the static-scale formula of `W8A8Linear`) in both
  the int8 values and the fp32 scales, including all-zero rows and values that land exactly half-way between integers;
* `w8a8_linear` equals the PyTorch epilogue of `W8A8Linear` applied to the exact int32 product (`torch._int_mm`, padded
  to its shape rules), across M from 1 to 4096, N / K on and off the 128 tile, bias, output dtype and static scales;
* both sides of the launcher's split-K choice run, the int32 bound holds at the largest accepted K, shapes outside the
  envelope run the old path, a bf16 cast keeps the scales, and an engine with CUDA-graph decode generates the same
  tokens as one whose W8A8 linears run the PyTorch reference.
"""
import ctypes

import pytest
import torch
import torch.nn as nn

pytestmark = pytest.mark.gpu

DTYPES = [torch.bfloat16, torch.float16, torch.float32]
DT_IDS = ["bf16", "fp16", "fp32"]


def _counts():
    from colossalai_b200.kernel import loader

    return dict(loader.launch_counter.by_name)


def _launched(before, name):
    return _counts().get(name, 0) - before.get(name, 0)


def _bits(t):
    return t.view(torch.int16) if t.element_size() == 2 else t.view(torch.int32) if t.element_size() == 4 else t


def _assert_bitwise(got, want):
    assert got.dtype == want.dtype and got.shape == want.shape, (got.dtype, want.dtype, got.shape, want.shape)
    diff = (_bits(got) != _bits(want))
    assert not diff.any(), f"{int(diff.sum())} of {diff.numel()} elements differ; first at {diff.nonzero()[0].tolist()}"


def _exact_int_mm(a, b):
    """int32 [M, N] = a [M, K] @ b [N, K]^T, exact: torch._int_mm with M padded to a multiple of 8 above 16 and N to a
    multiple of 8."""
    M, N = a.shape[0], b.shape[0]
    Mp, Np = max(24, (M + 7) // 8 * 8), (N + 7) // 8 * 8
    ap = torch.zeros(Mp, a.shape[1], dtype=torch.int8, device=a.device)
    bp = torch.zeros(Np, b.shape[1], dtype=torch.int8, device=b.device)
    ap[:M], bp[:N] = a, b
    return torch._int_mm(ap, bp.t().contiguous())[:M, :N]


def _ref_epilogue(acc, sx, w_scale, bias, dtype):
    y = acc.float() * sx * w_scale[None, :]
    if bias is not None:
        y = y + bias.float()
    return y.to(dtype)


def _ref_quant(x2, act_scale):
    from colossalai_b200.quantization.smoothquant import quantize_activation_per_token

    if act_scale is None:
        return quantize_activation_per_token(x2)
    return torch.clamp(torch.round(x2.float() / act_scale), -127, 127).to(torch.int8), act_scale


def _reference(x2, w_q, w_scale, bias, act_scale=None):
    xq, sx = _ref_quant(x2, act_scale)
    return _ref_epilogue(_exact_int_mm(xq, w_q), sx, w_scale, bias, x2.dtype)


def _weights(N, K, seed=0, bias_dtype=None):
    from colossalai_b200.quantization.smoothquant import quantize_weight_per_channel

    g = torch.Generator().manual_seed(seed)
    w_q, w_scale = quantize_weight_per_channel(torch.randn(N, K, generator=g) * 0.05)
    bias = None if bias_dtype is None else (torch.randn(N, generator=g) * 0.5).to(bias_dtype).cuda()
    return w_q.cuda(), w_scale.cuda(), bias


def _acts(M, K, dtype, seed=1):
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(M, K, generator=g)
    x[:, :: max(1, K // 7)] *= 20          # SmoothQuant-like outlier channels
    return x.to(dtype).cuda()


# ------------------------------------------------------------------------------------------------ quantiser
def _quant_rows(M, K, dtype):
    x = _acts(M, K, torch.float32, seed=K)
    x[0] = 0                                                    # all-zero row: the 1e-8 clamp
    half = torch.tensor([2.5, -2.5, 3.5, -3.5, 0.5, -0.5, 1.5, -1.5])
    x[1] = 0
    x[1, 0] = 127                                               # amax 127 -> scale exactly 1.0
    x[1, 1:1 + min(K - 1, 8)] = half[:min(K - 1, 8)]            # x / scale exactly k + 0.5
    x[2] = 0
    x[2, -1] = -254                                             # scale 2.0: 5 / 2, 7 / 2, ... are half-way
    x[2, : min(K - 1, 8)] = half[: min(K - 1, 8)] * 2
    x[3] *= 1e-6                                                # tiny scales
    return x.to(dtype).cuda()


@pytest.mark.parametrize("K", [16, 272, 4096, 14336])
@pytest.mark.parametrize("dtype", DTYPES, ids=DT_IDS)
def test_quantize_per_token_bitwise(dtype, K):
    from colossalai_b200.ops import w8a8
    from colossalai_b200.quantization.smoothquant import quantize_activation_per_token

    x = _quant_rows(37, K, dtype)
    c = _counts()
    xq, sx = w8a8.quantize_per_token(x)
    assert _launched(c, "w8a8_quant") == 1
    want_q, want_s = quantize_activation_per_token(x)
    _assert_bitwise(sx, want_s)
    _assert_bitwise(xq, want_q)
    if K >= 16:
        assert xq[1, 1:9].tolist()[: min(K - 1, 8)] == [2, -2, 4, -4, 0, 0, 2, -2][: min(K - 1, 8)]


@pytest.mark.parametrize("K", [16, 272, 4096, 14336])
@pytest.mark.parametrize("dtype", DTYPES, ids=DT_IDS)
def test_quantize_static_bitwise(dtype, K):
    from colossalai_b200.ops import w8a8

    x = _quant_rows(37, K, dtype)
    for s in (1.0, 0.5, 0.0371):                                # 1.0 / 0.5: exact half-way quotients
        act_scale = torch.tensor(s, device="cuda")
        _assert_bitwise(w8a8.quantize_static(x, act_scale), _ref_quant(x, act_scale)[0])


def test_quantize_strided_rows():
    from colossalai_b200.ops import w8a8
    from colossalai_b200.quantization.smoothquant import quantize_activation_per_token

    x = _acts(9, 512, torch.bfloat16)[:, 64:336]                # row stride 512, 272 columns
    xq, sx = w8a8.quantize_per_token(x)
    want_q, want_s = quantize_activation_per_token(x)
    _assert_bitwise(sx, want_s)
    _assert_bitwise(xq, want_q)


# ------------------------------------------------------------------------------------------------ GEMM
def _run_linear(M, N, K, dtype, bias_dtype, static, seed=0):
    from colossalai_b200.ops import w8a8

    w_q, w_scale, bias = _weights(N, K, seed, bias_dtype)
    x = _acts(M, K, dtype, seed + 1)
    act_scale = torch.tensor(float(x.float().abs().max()) / 127.0, device="cuda") if static else None
    assert w8a8.supported(x, w_q, w_scale, bias, act_scale)
    c = _counts()
    got = w8a8.w8a8_linear(x, w_q, w_scale, bias, act_scale)
    assert _launched(c, "w8a8_quant") == 1
    assert _launched(c, "gemm_w8a8") + _launched(c, "gemm_w8a8_splitk") == 1
    _assert_bitwise(got, _reference(x, w_q, w_scale, bias, act_scale))
    return c


@pytest.mark.parametrize("NK", [(264, 272), (4096, 4096), (6144, 14336)], ids=lambda s: f"N{s[0]}K{s[1]}")
@pytest.mark.parametrize("M", [1, 7, 16, 17, 64, 128, 200, 1000, 4096])
def test_w8a8_linear_shapes_bitwise(M, NK):
    _run_linear(M, NK[0], NK[1], torch.bfloat16, torch.float32, False)


@pytest.mark.parametrize("static", [False, True], ids=["per_token", "static"])
@pytest.mark.parametrize("bias_dtype", [None, torch.float32, torch.bfloat16, torch.float16],
                         ids=["nobias", "bias_fp32", "bias_bf16", "bias_fp16"])
@pytest.mark.parametrize("dtype", DTYPES, ids=DT_IDS)
@pytest.mark.parametrize("MNK", [(16, 4096, 4096), (1000, 2050, 1040)], ids=["splitk", "plain"])
def test_w8a8_linear_epilogue_bitwise(MNK, dtype, bias_dtype, static):
    _run_linear(*MNK, dtype, bias_dtype, static)


@pytest.mark.parametrize("MNK,branch", [((1, 4096, 4096), "gemm_w8a8_splitk"), ((64, 4096, 14336), "gemm_w8a8_splitk"),
                                        ((16, 6144, 4096), "gemm_w8a8_splitk"), ((16, 28672, 4096), "gemm_w8a8"),
                                        ((4096, 4096, 4096), "gemm_w8a8"), ((16, 4096, 272), "gemm_w8a8"),
                                        ((64, 4096, 4096), "gemm_w8a8")])
def test_split_k_selection(MNK, branch):
    """Decode shapes with few output tiles and K >= 128 M split K (int32 partials summed in a workspace,
    deterministic); shapes that fill the SMs, or whose K is short (next to M, or under 4 stages per split), do not.
    Either way the result is bitwise the reference."""
    c = _run_linear(*MNK, torch.bfloat16, torch.bfloat16, False)
    assert _launched(c, branch) == 1
    from colossalai_b200.ops import w8a8

    w_q, w_scale, bias = _weights(MNK[1], MNK[2], 3, torch.float32)
    x = _acts(MNK[0], MNK[2], torch.bfloat16, 4)
    first = w8a8.w8a8_linear(x, w_q, w_scale, bias)
    _assert_bitwise(w8a8.w8a8_linear(x, w_q, w_scale, bias), first)


def test_int32_range_at_largest_k():
    """All-+-127 operands at the largest K whose sum fits in int32: the product is exact."""
    from colossalai_b200.ops import w8a8

    K = w8a8.MAX_K // 16 * 16
    assert 127 * 127 * K < 2 ** 31 <= 127 * 127 * (K + 16)
    M, N = 16, 16
    x = torch.full((M, K), 127.0, device="cuda", dtype=torch.float32)
    x[1::2] = -127.0                                             # rows alternate +-127
    w_q = torch.full((N, K), 127, dtype=torch.int8, device="cuda")
    w_q[N // 2:] = -127
    w_scale = torch.ones(N, device="cuda")
    act_scale = torch.tensor(1.0, device="cuda")
    got = w8a8.w8a8_linear(x, w_q, w_scale, None, act_scale)
    exact = 127 * 127 * K
    sign = torch.tensor([1.0, -1.0], device="cuda").repeat(M // 2)[:, None] * torch.tensor(
        [1.0] * (N // 2) + [-1.0] * (N // 2), device="cuda")[None, :]
    _assert_bitwise(got, (sign * float(exact)).float())
    xq = torch.where(x > 0, 127, -127).to(torch.int8)
    _assert_bitwise(got, _ref_epilogue(_exact_int_mm(xq, w_q), act_scale, w_scale, None, torch.float32))


def test_k_above_bound_is_rejected_and_falls_back():
    from colossalai_b200.kernel import loader
    from colossalai_b200.ops import w8a8
    from colossalai_b200.quantization.smoothquant import W8A8Linear

    K = (w8a8.MAX_K // 16 + 1) * 16
    M, N = 16, 16
    a = torch.ones(M, K, dtype=torch.int8, device="cuda")
    b = torch.ones(N, K, dtype=torch.int8, device="cuda")
    y = torch.empty(M, N, device="cuda")
    ones = torch.ones(max(M, N), device="cuda")
    gemm, _ = w8a8._libs()
    rc = gemm.cb_gemm_w8a8(loader.ptr(a), loader.ptr(b), loader.ptr(y), M, N, K, K, K, N, loader.ptr(ones), 1,
                           loader.ptr(ones), None, 0, 0, None, ctypes.c_longlong(0), loader.stream_ptr())
    assert rc == 1                                               # cudaErrorInvalidValue
    lin = W8A8Linear(K, N, bias=False).cuda()
    lin.weight.fill_(1)
    x = torch.ones(M, K, device="cuda")
    assert not w8a8.supported(x, lin.weight, lin.weight_scale)
    c = _counts()
    with torch.no_grad():
        got = lin(x)
    assert _launched(c, "gemm_w8a8") + _launched(c, "gemm_w8a8_splitk") + _launched(c, "w8a8_quant") == 0
    torch.testing.assert_close(got, torch.full((M, N), float(K), device="cuda"), atol=0, rtol=1e-4)


@pytest.mark.parametrize("NK", [(64, 72), (63, 64)], ids=["K_not_16", "N_odd"])
def test_outside_envelope_runs_old_path(NK):
    from colossalai_b200.ops._dispatch import force_torch
    from colossalai_b200.quantization.smoothquant import W8A8Linear

    N, K = NK
    torch.manual_seed(0)
    lin = W8A8Linear.from_float(nn.Linear(K, N).cuda())
    x = torch.randn(2, 7, K, device="cuda")     # 14 rows: the old path's fp32 branch (cuBLASLt's int8 GEMM refuses K 72)
    c = _counts()
    with torch.no_grad():
        got = lin(x)
    assert sum(v for k, v in _counts().items()) == sum(c.values())      # nothing native launched
    with force_torch(), torch.no_grad():
        want = lin(x)
    _assert_bitwise(got, want)


def test_force_torch_selects_pytorch_path():
    from colossalai_b200.ops._dispatch import force_torch
    from colossalai_b200.quantization.smoothquant import W8A8Linear

    lin = W8A8Linear.from_float(nn.Linear(256, 128).cuda())
    c = _counts()
    with force_torch(), torch.no_grad():
        lin(torch.randn(24, 256, device="cuda"))
    assert _launched(c, "w8a8_quant") == 0


@pytest.mark.parametrize("act_quant", ["per_token", "static"])
def test_cast_keeps_scales_and_native_matches_torch(act_quant):
    from colossalai_b200.ops._dispatch import force_torch
    from colossalai_b200.quantization.smoothquant import W8A8Linear

    torch.manual_seed(0)
    lin = W8A8Linear.from_float(nn.Linear(1024, 512).cuda(), act_quant, act_absmax=40.0).to(torch.bfloat16)
    assert lin.weight_scale.dtype == torch.float32 and lin.act_scale.dtype == torch.float32
    assert lin.bias.dtype == torch.bfloat16 and lin.weight.dtype == torch.int8
    x = (torch.randn(2, 20, 1024, device="cuda") * 8).bfloat16()      # 40 rows: the old path's exact _int_mm branch
    c = _counts()
    with torch.no_grad():
        got = lin(x)
    assert _launched(c, "w8a8_quant") == 1 and _launched(c, "gemm_w8a8") + _launched(c, "gemm_w8a8_splitk") == 1
    with force_torch(), torch.no_grad():
        want = lin(x)
    _assert_bitwise(got, want)


def test_bias_needing_grad_stays_on_autograd_path():
    from colossalai_b200.quantization.smoothquant import W8A8Linear

    lin = W8A8Linear.from_float(nn.Linear(256, 128).cuda())
    x = torch.randn(24, 256, device="cuda")
    c = _counts()
    lin(x).sum().backward()
    assert _launched(c, "w8a8_quant") == 0
    torch.testing.assert_close(lin.bias.grad, torch.full((128,), 24.0, device="cuda"))


# ------------------------------------------------------------------------------------------------ engine
def test_engine_cuda_graph_decode_matches_reference(monkeypatch):
    """A SmoothQuant-quantised bf16 llama (head_dim 64: paged decode on the native kernel, CUDA-graph decode) with
    continuous batching generates exactly the tokens of the same engine whose W8A8 linears run the PyTorch reference."""
    from colossalai_b200.inference import InferenceConfig, InferenceEngine
    from colossalai_b200.inference.config import GenerationConfig
    from colossalai_b200.models import build_model, get_config
    from colossalai_b200.ops import w8a8
    from colossalai_b200.quantization.smoothquant import W8A8Linear, smooth_and_quantize_model

    torch.manual_seed(0)
    model = build_model(get_config("llama-tiny", hidden_size=256, intermediate_size=512)).to(torch.bfloat16).cuda().eval()
    batches = [dict(input_ids=torch.randint(0, 512, (2, 32), device="cuda")) for _ in range(2)]
    smooth_and_quantize_model(model, batches)
    assert sum(isinstance(m, W8A8Linear) for m in model.modules()) == 4 * 4
    prompts = [[5, 9, 13, 200, 7], [11, 3], [400, 401, 402, 403, 404, 405, 406, 407, 408, 409], [17] * 6, [99, 98, 97]]
    kw = dict(max_batch_size=3, max_input_len=32, max_output_len=12, block_size=16, dtype="bf16", ignore_eos=True,
              use_cuda_graph=True)

    def run():
        eng = InferenceEngine(model, None, InferenceConfig(**kw))
        _, ids = eng.generate(prompts_token_ids=prompts, return_token_ids=True,
                              generation_config=GenerationConfig(max_new_tokens=12))
        return eng, ids

    c = _counts()
    eng, got = run()
    assert eng.use_cuda_graph and eng.graph_runners
    assert _launched(c, "w8a8_quant") > 0 and _launched(c, "gemm_w8a8") + _launched(c, "gemm_w8a8_splitk") > 0
    assert _launched(c, "paged_decode_attention") > 0
    lin = next(m for m in model.modules() if isinstance(m, W8A8Linear))
    assert lin.weight_scale.dtype == torch.float32 and lin.act_scale.dtype == torch.float32

    def reference(x, w_q, w_scale, bias, act_scale=None):
        x2 = x.reshape(-1, x.shape[-1])
        return _reference(x2, w_q, w_scale, bias, act_scale).reshape(*x.shape[:-1], w_q.shape[0])

    monkeypatch.setattr(w8a8, "w8a8_linear", reference)
    c = _counts()
    _, want = run()
    assert _launched(c, "w8a8_quant") == 0
    assert got == want
    assert all(len(g) == len(p) + 12 for p, g in zip(prompts, got))
