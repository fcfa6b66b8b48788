"""fp8 (E4M3 / E5M2) wgmma GEMM (m64n128k32, fp32 promotion per 128-deep stage) against an fp32 PyTorch reference of the same
de-quantised operands."""
import os

import pytest
import torch

pytestmark = pytest.mark.gpu

SHAPES = [(4096, 4096, 4096), (2560, 4096, 1088), (8192, 6144, 4096), (4100, 2056, 512)]


def _quant(x, dtype):
    fmax = torch.finfo(dtype).max
    scale = x.abs().max().float() / fmax
    return (x.float() / scale).clamp(-fmax, fmax).to(dtype), scale.reshape(1)


@pytest.mark.parametrize("M,N,K", SHAPES)
@pytest.mark.parametrize("a_dtype", ["e4m3", "e5m2"])
@pytest.mark.parametrize("out_dtype", [torch.bfloat16, torch.float32])
def test_fp8_gemm_matches_fp32_reference(M, N, K, a_dtype, out_dtype):
    from colossalai_b200.ops import gemm_native

    if not gemm_native.available():
        pytest.skip("needs an H100")
    torch.manual_seed(0)
    adt = torch.float8_e4m3fn if a_dtype == "e4m3" else torch.float8_e5m2
    a, sa = _quant(torch.randn(M, K, device="cuda"), adt)
    b, sb = _quant(torch.randn(N, K, device="cuda") * 0.5, torch.float8_e4m3fn)
    assert gemm_native.supported_fp8_nt(a, b)
    c = gemm_native.gemm_fp8_nt(a, b, sa, sb, out_dtype)
    ref = (a.float() * sa) @ (b.float() * sb).t()
    torch.cuda.synchronize()
    err = (c.float() - ref).abs().max().item()
    tol = 2e-2 * ref.abs().max().item() if out_dtype == torch.bfloat16 else 1e-3 * ref.abs().max().item()
    assert err <= tol, (err, tol)


def test_linear_fp8_native_backend_matches_cublaslt():
    from colossalai_b200.ops import gemm_native
    from colossalai_b200.quantization.fp8 import linear_fp8

    if not gemm_native.available():
        pytest.skip("needs an H100")
    torch.manual_seed(0)
    x = torch.randn(4096, 4096, device="cuda", dtype=torch.bfloat16, requires_grad=True)
    w = (torch.randn(6144, 4096, device="cuda", dtype=torch.bfloat16) * 0.02).requires_grad_()
    outs = {}
    for be in ("cublaslt", "native"):
        gemm_native.set_fp8_backend(be)
        x.grad = w.grad = None
        y = linear_fp8(x, w)
        y.float().pow(2).mean().backward()
        outs[be] = (y.detach().float(), x.grad.float().clone(), w.grad.float().clone())
    gemm_native.set_fp8_backend(os.environ.get("CB200_FP8_GEMM", "native"))
    for a, b in zip(outs["cublaslt"], outs["native"]):
        assert (a - b).abs().max() <= 2e-2 * a.abs().max() + 1e-6
