"""wgmma grouped (per-expert) GEMM: forward / dgrad with variable rows per expert and wgrad with variable reduction
length, against fp32 per-expert matmuls.  Expert sizes include 0, 1, non-multiples of the tile and of the k-block."""
import pytest
import torch

pytestmark = pytest.mark.gpu


def _ref(x, w, counts):
    out = torch.empty(x.shape[0], w.shape[1], dtype=torch.float32, device=x.device)
    s = 0
    for e, n in enumerate(counts.tolist()):
        out[s:s + n] = x[s:s + n].float() @ w[e].float().t()
        s += n
    return out


CASES = [
    ([300, 0, 1, 255, 256, 257, 700, 131], 512, 768),          # ragged groups, an empty one
    ([2048] * 8, 4096, 2816),                                  # balanced, Mixtral-like aspect
    ([5, 9000, 17, 3], 1024, 1408),                            # one dominant expert, output width not a tile multiple
    ([128 * i for i in range(1, 17)], 2048, 2816),             # 16 experts, every size a k-block multiple
]


@pytest.mark.parametrize("counts,K,N", CASES)
@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16])
def test_grouped_forward(counts, K, N, dtype):
    from colossalai_b200.moe import grouped_gemm as gg

    torch.manual_seed(0)
    c = torch.tensor(counts, device="cuda")
    rows = int(sum(counts))
    x = (torch.randn(rows, K, device="cuda") * 0.5).to(dtype)
    w = (torch.randn(len(counts), N, K, device="cuda") * 0.05).to(dtype)
    assert gg.native_ok(x, w)
    y = gg.grouped_linear(x, w, c)
    ref = _ref(x, w, c)
    torch.testing.assert_close(y.float(), ref, atol=2e-2 + 2e-3 * K ** 0.5 * 0.05, rtol=1.6e-2)


@pytest.mark.parametrize("counts,K,N", CASES)
@pytest.mark.parametrize("aligned", [False, True])
def test_grouped_backward(counts, K, N, aligned):
    """dX (variable-M NN kernel) and dW (variable-K TN kernel; padded on the device when the layout is not aligned)."""
    from colossalai_b200.moe import grouped_gemm as gg

    if N % 128 != 0:
        pytest.skip("dgrad kernel needs the expert output width to be a multiple of 128")
    if aligned and any(n % 128 for n in counts):
        pytest.skip("layout is not aligned")
    torch.manual_seed(1)
    c = torch.tensor(counts, device="cuda")
    rows = int(sum(counts))
    x = (torch.randn(rows, K, device="cuda") * 0.5).bfloat16().requires_grad_(True)
    w = (torch.randn(len(counts), N, K, device="cuda") * 0.05).bfloat16().requires_grad_(True)
    dy = (torch.randn(rows, N, device="cuda") * 0.1).bfloat16()
    gg.grouped_linear(x, w, c, aligned=aligned).backward(dy)
    xf, wf = x.detach().float().requires_grad_(True), w.detach().float().requires_grad_(True)
    out = torch.empty(rows, N, device="cuda")
    s, parts = 0, []
    for e, n in enumerate(counts):
        parts.append(xf[s:s + n] @ wf[e].t())
        s += n
    torch.cat(parts, 0).backward(dy.float())
    dxe = (x.grad.float() - xf.grad).abs().max().item()
    assert dxe <= 1.6e-2 * xf.grad.abs().max().item() + 1e-3, dxe
    for e, n in enumerate(counts):
        ref = wf.grad[e]
        err = (w.grad[e].float() - ref).abs().max().item()
        assert err <= 1.6e-2 * ref.abs().max().item() + 2e-3 * max(n, 1) ** 0.5 * 0.05 + 1e-3, (e, n, err)


def test_grouped_gemm_counts_stay_on_device():
    """No host synchronisation: the group sizes are only ever read by the kernel."""
    from colossalai_b200.moe import grouped_gemm as gg

    c = torch.tensor([100, 200, 300, 424], device="cuda")
    x = torch.randn(1024, 512, device="cuda", dtype=torch.bfloat16)
    w = torch.randn(4, 256, 512, device="cuda", dtype=torch.bfloat16)
    torch.cuda.synchronize()
    with torch.cuda.stream(torch.cuda.Stream()):
        torch.cuda.set_sync_debug_mode("error")
        try:
            y = gg.grouped_linear(x, w, c)
        finally:
            torch.cuda.set_sync_debug_mode("default")
    torch.cuda.synchronize()
    torch.testing.assert_close(y.float(), _ref(x, w, c), atol=0.5, rtol=2e-2)
