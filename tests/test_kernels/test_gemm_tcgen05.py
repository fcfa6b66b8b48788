"""wgmma GEMM numerics vs fp32 torch.matmul for the three linear-layer GEMM flavours (NT / NN / TN), tails and
accumulate-into-C."""
import pytest
import torch

pytestmark = pytest.mark.gpu


def _mk(*shape, dtype=torch.bfloat16):
    return (torch.randn(*shape, device="cuda") * 0.5).to(dtype)


# (4096, 4096, 4096): 256 pair tiles -> 3 full waves + 34 tail tiles cut in 2 K ranges; (4096, 6144, 4096): 384 tiles,
# 14 tail tiles cut in 5; (2560, 2304, 1024): 90 tiles, 16 tail tiles cut in 2 (8 k-blocks); (8192, 6144, 4096): 768 / 28
SHAPES = [(128, 256, 64), (256, 512, 128), (1000, 768, 520), (4096, 4096, 4096), (336, 1024, 2048), (8192, 6144, 4096),
          (4096, 6144, 4096), (2560, 2304, 1024)]


def _set_tail(monkeypatch, tail):
    """Schedule of the CTA-pair kernel's partial last wave: whole tiles / 256 x 128 halves (default) / K ranges."""
    monkeypatch.setenv("CB200_GEMM_TAIL_HALF", "1" if tail == "half" else "0")
    monkeypatch.setenv("CB200_GEMM_TAIL_SPLIT", "3" if tail == "ksplit" else "0")


def _tol(K):
    """inputs ~ N(0, 0.25): |y| ~ 0.25 sqrt(K); fp32 accumulation, one rounding to the 16-bit output (<= 2^-9 rel.).
    Tight enough that a dropped 8-element k tail (error ~ 0.7) or a dropped k-block fails everywhere."""
    return dict(atol=0.002 * K ** 0.5 + 0.01, rtol=1.6e-2)


@pytest.mark.parametrize("M,N,K", SHAPES)
@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16])
def test_gemm_nt(M, N, K, dtype):
    from colossalai_b200.ops import gemm_native as g

    M = 333 if M == 336 else M     # odd M is fine for K-major A

    torch.manual_seed(0)
    x, w = _mk(M, K, dtype=dtype), _mk(N, K, dtype=dtype)
    y = g.gemm_nt(x, w)
    ref = x.float() @ w.float().t()
    torch.testing.assert_close(y.float(), ref, **_tol(K))


@pytest.mark.parametrize("M,N,K", SHAPES)
def test_gemm_nn(M, N, K):
    from colossalai_b200.ops import gemm_native as g

    torch.manual_seed(0)
    a, b = _mk(M, K), _mk(K, N)
    c = g.gemm_nn(a, b)
    ref = a.float() @ b.float()
    torch.testing.assert_close(c.float(), ref, **_tol(K))


@pytest.mark.parametrize("M,N,K", SHAPES)
def test_gemm_tn(M, N, K):
    from colossalai_b200.ops import gemm_native as g

    torch.manual_seed(0)
    a, b = _mk(K, M), _mk(K, N)      # contraction over dim 0
    c = g.gemm_tn(a, b)
    ref = a.float().t() @ b.float()
    torch.testing.assert_close(c.float(), ref, **_tol(K))


def test_gemm_block_n_and_tail_have_no_effect(monkeypatch):
    """`block_n` and `CB200_GEMM_TAIL_*` are accepted for interface stability and have no effect: every GEMM flavour
    returns the same bits with and without them."""
    from colossalai_b200.ops import gemm_native as g

    torch.manual_seed(0)
    M, N, K = 1000, 768, 520
    x, w, b, dy = _mk(M, K), _mk(N, K), _mk(K, N), _mk(M, N)
    base = (g.gemm_nt(x, w), g.gemm_nn(x, b), g.gemm_tn(x, dy))
    for tail in ("half", "ksplit"):
        _set_tail(monkeypatch, tail)
        for block_n in (128, 256, 512):
            got = (g.gemm_nt(x, w, block_n=block_n), g.gemm_nn(x, b, block_n=block_n),
                   g.gemm_tn(x, dy, block_n=block_n))
            for name, r, e in zip(("nt", "nn", "tn"), got, base):
                assert torch.equal(r.view(torch.int16), e.view(torch.int16)), \
                    f"gemm_{name} changed with block_n={block_n}, tail={tail}"


@pytest.mark.parametrize("out_dtype", [torch.float32, torch.bfloat16])
def test_gemm_tn_accumulate(out_dtype):
    from colossalai_b200.ops import gemm_native as g

    torch.manual_seed(0)
    a, b = _mk(2048, 512), _mk(2048, 768)
    acc = torch.randn(512, 768, device="cuda").to(out_dtype)
    ref = acc.float() + a.float().t() @ b.float()
    g.gemm_tn(a, b, out=acc, accumulate=True)
    torch.testing.assert_close(acc.float(), ref, atol=0.3, rtol=2e-2)


@pytest.mark.parametrize("M,N,K", [(4096, 4096, 4096), (6144, 4096, 4096)])
@pytest.mark.parametrize("out_dtype", [torch.float32, torch.bfloat16])
@pytest.mark.parametrize("tail", ["half", "ksplit"])
def test_gemm_tn_accumulate_with_tail_split(M, N, K, out_dtype, tail, monkeypatch):
    """wgrad shape of the N=1 Llama step: `main_grad += dY^T X` where the tail wave is split along K (the fix-up unit is
    the one that reads and updates C)."""
    from colossalai_b200.ops import gemm_native as g

    _set_tail(monkeypatch, tail)
    torch.manual_seed(0)
    a, b = _mk(K, M), _mk(K, N)
    acc = (torch.randn(M, N, device="cuda") * 4).to(out_dtype)
    ref = acc.float() + a.float().t() @ b.float()
    for _ in range(2):           # second launch reuses the re-armed workspace flags
        out = acc.clone()
        g.gemm_tn(a, b, out=out, accumulate=True, block_n=512)
        torch.testing.assert_close(out.float(), ref, **_tol(K))


def test_gemm_tail_split_off_matches_on(monkeypatch):
    """Same launch with and without the tail-wave split: both within tolerance of fp32 and of each other."""
    import os
    import subprocess
    import sys

    code = ("import torch; from colossalai_b200.ops import gemm_native as g; torch.manual_seed(0); "
            "x=(torch.randn(4096,4096,device='cuda')*0.5).bfloat16(); w=(torch.randn(4096,4096,device='cuda')*0.5).bfloat16(); "
            "y=g.gemm_nt(x,w,block_n=512); print('CHK', float(y.float().abs().sum()), float((y.float()-x.float()@w.float().t()).abs().max()))")
    outs = []
    for flag in ("0", "1"):
        env = dict(os.environ, CB200_GEMM_TAIL_HALF=flag, CB200_GEMM_TAIL_SPLIT="0")
        r = subprocess.run([sys.executable, "-c", code], capture_output=True, text=True, env=env, timeout=600,
                           cwd=os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__)))))
        line = [l for l in r.stdout.splitlines() if l.startswith("CHK")]
        assert line, r.stderr[-2000:]
        outs.append([float(v) for v in line[0].split()[1:]])
    assert outs[0][1] < 0.3 and outs[1][1] < 0.3, outs     # bf16 ulp at |y| ~ 64 is 0.25
    assert abs(outs[0][0] - outs[1][0]) <= 1e-3 * outs[0][0], outs


def test_linear_autograd_through_native_gemm():
    """The op-level entry points (`ops.linear_forward / matmul_nn / matmul_tn`) used by every parallel linear."""
    from colossalai_b200 import ops
    from colossalai_b200.kernel import loader
    from colossalai_b200.ops import gemm as gemm_ops
    from colossalai_b200.shardformer.layer._operation import linear_with_grad_accum

    torch.manual_seed(0)
    x = _mk(1024, 512).requires_grad_(True)
    w = _mk(768, 512).requires_grad_(True)
    old = gemm_ops.get_gemm_backend()
    gemm_ops.set_gemm_backend("native")
    before = loader.launch_counter.count
    try:
        y = linear_with_grad_accum(x, w)
        (y.float() * 0.01).sum().backward()
    finally:
        gemm_ops.set_gemm_backend(old)
    assert loader.launch_counter.count >= before + 3, "the tcgen05 GEMM must have run for fwd, dgrad and wgrad"
    xr, wr = x.detach().float().requires_grad_(True), w.detach().float().requires_grad_(True)
    ((xr @ wr.t()) * 0.01).sum().backward()
    torch.testing.assert_close(y.float(), xr @ wr.t(), atol=0.2, rtol=2e-2)
    torch.testing.assert_close(x.grad.float(), xr.grad, atol=2e-2, rtol=2e-2)
    torch.testing.assert_close(w.grad.float(), wr.grad, atol=5e-2, rtol=2e-2)
