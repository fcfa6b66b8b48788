"""Weight-only-quantised GEMMs (`kernel/csrc/wq_gemm_wgmma.cu`, `ops/wq_gemm.py`) on the GPU.

* `cb_wq_dequantize` is bitwise equal to the PyTorch `dequantize_reference()` for nf4, fp4, nf4 with double
  quantisation and int8, in bf16 and fp16.
* The NT (forward) and NN (input gradient) GEMMs - native decode into a scratch weight, then the dense wgmma GEMM -
  against a float64 GEMM on the dequantised weight.  The largest error may be at most twice that of torch's 16-bit
  matmul on the same dequantised weight, plus 1e-5 of the largest |reference|: a wrong nibble or absmax moves an
  output by a sizeable fraction of |ref|.
* Shapes outside the envelope take the dequantise-then-matmul reference and stay correct.
* A chain of 4-bit layers run with an input that needs a gradient keeps no 16-bit weight alive.
* QLoRA end to end through TorchDDPPlugin: the loss falls and the first step's adapter gradients match a model on the
  dequantised weights.
"""
import copy

import pytest
import torch
import torch.nn as nn

pytestmark = pytest.mark.gpu

FORMATS = ["nf4", "fp4", "nf4_dq", "int8"]
DTYPES = [torch.bfloat16, torch.float16]


def _layer(fmt, N, K, dtype, block=64, bias=False, seed=0):
    from colossalai_b200.quantization.bnb import Linear4bit, Linear8bit

    g = torch.Generator().manual_seed(seed)
    lin = nn.Linear(K, N, bias=bias)
    with torch.no_grad():
        lin.weight.copy_(torch.randn(N, K, generator=g) * 0.05)
    lin = lin.cuda()
    if fmt == "int8":
        return Linear8bit(lin, dtype)
    return Linear4bit(lin, dtype, "fp4" if fmt == "fp4" else "nf4", block, double_quant=(fmt == "nf4_dq"))


def _counts():
    from colossalai_b200.kernel import loader

    return dict(loader.launch_counter.by_name)


def _launched(before, name):
    return _counts().get(name, 0) - before.get(name, 0)


@pytest.mark.parametrize("dtype", DTYPES, ids=["bf16", "fp16"])
@pytest.mark.parametrize("fmt", FORMATS)
@pytest.mark.parametrize("shape", [(136, 256, 64), (384, 512, 128), (64, 192, 64), (1000, 1024, 256)])
def test_dequantize_bitwise(fmt, dtype, shape):
    from colossalai_b200.ops import wq_gemm

    N, K, block = shape
    layer = _layer(fmt, N, K, dtype, block)
    c = _counts()
    got = wq_gemm.dequantize(layer)
    assert _launched(c, "wq_dequantize") == 1
    want = layer.dequantize_reference()
    assert got.dtype == want.dtype == dtype and got.shape == want.shape == (N, K)
    assert torch.equal(got.view(torch.int16), want.view(torch.int16))
    assert torch.equal(layer.dequantize().view(torch.int16), want.view(torch.int16))


def _check(got, a, w, layout):
    """got vs a float64 GEMM of the operands; bound = 2 x torch's 16-bit matmul error + 1e-5 max|ref|."""
    ref = a.double() @ (w.double().t() if layout == "nt" else w.double())
    torch16 = (a @ (w.t() if layout == "nt" else w)).double()
    e_kernel = (got.double() - ref).abs().max().item()
    e_torch = (torch16 - ref).abs().max().item()
    bound = 2 * e_torch + 1e-5 * ref.abs().max().item()
    assert e_kernel <= bound, (e_kernel, e_torch, ref.abs().max().item())


SHAPES = [(256, 256), (200, 320), (1000, 768), (4096, 14336)]


def _run_both(fmt, dtype, M, N, K, block):
    from colossalai_b200.ops import wq_gemm

    layer = _layer(fmt, N, K, dtype, block, seed=M + N + K)
    assert wq_gemm.gemm_supported(layer)
    w = layer.dequantize_reference()
    g = torch.Generator(device="cuda").manual_seed(1)
    x = torch.randn(M, K, device="cuda", dtype=dtype, generator=g)
    dy = torch.randn(M, N, device="cuda", dtype=dtype, generator=g)
    c = _counts()
    y = wq_gemm.wq_linear(x, layer)
    dx = wq_gemm.wq_matmul_nn(dy, layer)
    assert _launched(c, "wq_dequantize") == 2 and _launched(c, "gemm_tcgen05") == 2
    assert y.shape == (M, N) and dx.shape == (M, K) and y.dtype == dx.dtype == dtype
    _check(y, x, w, "nt")
    _check(dx, dy, w, "nn")


@pytest.mark.parametrize("dtype", DTYPES, ids=["bf16", "fp16"])
@pytest.mark.parametrize("fmt", FORMATS)
@pytest.mark.parametrize("M", [1, 77, 128, 1000, 4096])
@pytest.mark.parametrize("shape", SHAPES, ids=lambda s: f"{s[0]}x{s[1]}")
def test_gemm_against_float64(fmt, dtype, M, shape):
    N, K = shape
    if N * K > 2**24 and M not in (1, 4096):
        pytest.skip("the largest weight runs at the smallest and largest M only")
    _run_both(fmt, dtype, M, N, K, 64)


@pytest.mark.parametrize("dtype", DTYPES, ids=["bf16", "fp16"])
@pytest.mark.parametrize("fmt", ["nf4", "fp4", "nf4_dq"])
@pytest.mark.parametrize("block", [64, 128, 256])
@pytest.mark.parametrize("M,N,K", [(77, 136, 768), (1000, 520, 1536), (4096, 1024, 512)])
def test_gemm_block_sizes(fmt, dtype, block, M, N, K):
    _run_both(fmt, dtype, M, N, K, block)


def test_gemm_k192_block64():
    _run_both("nf4", torch.bfloat16, 300, 192, 192, 64)
    _run_both("nf4", torch.bfloat16, 300, 64, 96, 64)      # K % block != 0: blocks straddle rows
    _run_both("int8", torch.bfloat16, 300, 192, 200, 64)   # int8: K a multiple of 8 only


@pytest.mark.parametrize("fmt,N,K,block", [("nf4", 64, 96, 36),      # block size not a multiple of 8
                                           ("int8", 64, 100, 64),    # K not a multiple of 8
                                           ("int8", 60, 128, 64),    # N not a multiple of 8
                                           ("nf4_dq", 100, 128, 64)])  # N not a multiple of 8
def test_fallback_outside_envelope(fmt, N, K, block):
    from colossalai_b200.ops import wq_gemm

    layer = _layer(fmt, N, K, torch.bfloat16, block)
    assert not wq_gemm.gemm_supported(layer)
    w = layer.dequantize_reference()
    x = torch.randn(33, K, device="cuda", dtype=torch.bfloat16)
    dy = torch.randn(33, N, device="cuda", dtype=torch.bfloat16)
    c = _counts()
    y = wq_gemm.wq_linear(x, layer)
    dx = wq_gemm.wq_matmul_nn(dy, layer)
    assert _launched(c, "gemm_tcgen05") == 0
    _check(y, x, w, "nt")
    _check(dx, dy, w, "nn")


@pytest.mark.parametrize("fmt", FORMATS)
def test_module_autograd_matches_reference(fmt):
    layer = _layer(fmt, 256, 512, torch.bfloat16, bias=True)
    w = layer.dequantize_reference()
    x = torch.randn(3, 50, 512, device="cuda", dtype=torch.bfloat16, requires_grad=True)
    y = layer(x)
    y.float().pow(2).sum().backward()
    xr = x.detach().double().requires_grad_(True)
    yr = xr @ w.double().t() + layer.bias.double()
    yr.pow(2).sum().backward()
    assert (y.double() - yr).abs().max() <= 2e-2 * yr.abs().max()
    assert (x.grad.double() - xr.grad).abs().max() <= 3e-2 * xr.grad.abs().max()


def test_forward_keeps_no_16bit_weight():
    from colossalai_b200.quantization.bnb import Linear4bit

    layers = []
    for i in range(8):
        lin = nn.Linear(4096, 4096, bias=False, device="cuda")
        layers.append(Linear4bit(lin, torch.bfloat16, "nf4", 64))
        del lin
    chain = nn.Sequential(*layers)
    M = 256
    x = torch.randn(M, 4096, device="cuda", dtype=torch.bfloat16, requires_grad=True)
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    base = torch.cuda.memory_allocated()
    y = chain(x)
    torch.cuda.synchronize()
    growth = torch.cuda.max_memory_allocated() - base
    activations = 9 * M * 4096 * 2
    assert growth < 32 * 2**20 + activations, growth
    y.float().sum().backward()
    assert x.grad is not None and torch.isfinite(x.grad.float()).all()


def test_qlora_end_to_end_ddp():
    import colossalai_b200
    from colossalai_b200.booster import Booster
    from colossalai_b200.booster.lora import LoraConfig, LoraLinear
    from colossalai_b200.booster.plugin import TorchDDPPlugin
    from colossalai_b200.models import build_model
    from colossalai_b200.quantization import BnbQuantizationConfig
    from colossalai_b200.quantization.bnb import Linear4bit
    from colossalai_b200.testing import free_port

    if not torch.distributed.is_initialized():
        colossalai_b200.launch(0, 1, "127.0.0.1", free_port(), verbose=False)
    torch.manual_seed(0)
    model = build_model("llama-tiny")
    booster = Booster(plugin=TorchDDPPlugin())
    model = booster.enable_lora(
        model, lora_config=LoraConfig(r=8, lora_alpha=16, target_modules=["qkv_proj", "o_proj", "gate_up_proj",
                                                                           "down_proj"]),
        bnb_quantization_config=BnbQuantizationConfig(load_in_4bit=True, bnb_4bit_quant_type="nf4",
                                                      bnb_4bit_compute_dtype="bf16"))
    model = model.cuda()
    opt = torch.optim.AdamW([p for p in model.parameters() if p.requires_grad], lr=1e-2)
    model, opt, *_ = booster.boost(model, opt)
    inner = model.unwrap()
    inner = inner.module if hasattr(inner, "module") and not hasattr(inner, "cfg") else inner

    # the reference: the same model with every quantised base as a bf16 nn.Linear on the dequantised weight
    ref = copy.deepcopy(inner)
    for m in ref.modules():
        if isinstance(m, LoraLinear) and isinstance(m.base_layer, Linear4bit):
            lin = nn.Linear(m.base_layer.in_features, m.base_layer.out_features, bias=False, device="cuda",
                            dtype=torch.bfloat16)
            lin.weight.data = m.base_layer.dequantize_reference()
            m.base_layer = lin.requires_grad_(False)

    torch.manual_seed(1)
    ids = torch.randint(0, 512, (4, 64), device="cuda")
    ref(input_ids=ids, labels=ids)["loss"].backward()
    losses = []
    for step in range(20):
        loss = model(input_ids=ids, labels=ids)["loss"]
        booster.backward(loss, opt)
        if step == 0:
            want = {n: p.grad for n, p in ref.named_parameters() if p.requires_grad}
            got = {n: p.grad for n, p in inner.named_parameters() if p.requires_grad}
            assert got.keys() == want.keys() and got
            for n, g in got.items():
                err = (g.double() - want[n].double()).abs().max().item()
                assert err <= 5e-2 * want[n].double().abs().max().item() + 1e-6, (n, err)
        opt.step()
        opt.zero_grad()
        losses.append(loss.item())
    assert losses[-1] < 0.95 * losses[0], losses
