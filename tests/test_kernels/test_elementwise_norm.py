"""Numerics of the sm_90a norm / activation / rope / CE kernels against plain PyTorch fp32 references."""
import pytest
import torch

from colossalai_b200 import ops
from colossalai_b200.ops import cross_entropy as ce

pytestmark = pytest.mark.gpu

DTYPES = [torch.bfloat16, torch.float16, torch.float32]


def _tol(dtype):
    return dict(atol=3e-2, rtol=3e-2) if dtype != torch.float32 else dict(atol=1e-4, rtol=1e-3)


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("shape", [(37, 1024), (512, 4096), (8, 8192), (5, 16384)])
@pytest.mark.parametrize("with_res", [False, True])
def test_rmsnorm_fwd_bwd(dtype, shape, with_res):
    torch.manual_seed(0)
    x = torch.randn(*shape, device="cuda", dtype=dtype, requires_grad=True)
    w = (1 + 0.1 * torch.randn(shape[1], device="cuda")).to(dtype).requires_grad_(True)
    res = torch.randn(*shape, device="cuda", dtype=dtype, requires_grad=True) if with_res else None
    xr, wr = x.detach().float().requires_grad_(True), w.detach().float().requires_grad_(True)
    rr = res.detach().float().requires_grad_(True) if with_res else None
    out = ops.rms_norm(x, w, 1e-5, res)
    ref = ops.rms_norm_ref(xr, wr, 1e-5, rr)
    if with_res:
        y, h = out
        yr, hr = ref
        g1, g2 = torch.randn_like(yr), torch.randn_like(hr)
        (y.float() * g1).sum().backward(retain_graph=True)
        (h.float() * g2).sum().backward()
        ((yr * g1).sum() + (hr * g2).sum()).backward()
        torch.testing.assert_close(h.float(), hr, **_tol(dtype))
        torch.testing.assert_close(res.grad.float(), rr.grad, **_tol(dtype))
    else:
        y, yr = out, ref
        g1 = torch.randn_like(yr)
        (y.float() * g1).sum().backward()
        (yr * g1).sum().backward()
    torch.testing.assert_close(y.float(), yr, **_tol(dtype))
    torch.testing.assert_close(x.grad.float(), xr.grad, **_tol(dtype))
    wt = dict(atol=0.5, rtol=5e-2) if dtype != torch.float32 else dict(atol=1e-3, rtol=1e-3)
    torch.testing.assert_close(w.grad.float(), wr.grad, **wt)


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("bias", [True, False])
def test_layernorm_fwd_bwd(dtype, bias):
    torch.manual_seed(0)
    x = torch.randn(300, 2048, device="cuda", dtype=dtype, requires_grad=True)
    w = (1 + 0.1 * torch.randn(2048, device="cuda")).to(dtype).requires_grad_(True)
    b = (0.1 * torch.randn(2048, device="cuda")).to(dtype).requires_grad_(True) if bias else None
    xr, wr = x.detach().float().requires_grad_(True), w.detach().float().requires_grad_(True)
    br = b.detach().float().requires_grad_(True) if bias else None
    y = ops.layer_norm(x, w, b, 1e-5)
    yr = torch.nn.functional.layer_norm(xr, (2048,), wr, br, 1e-5)
    g = torch.randn_like(yr)
    (y.float() * g).sum().backward()
    (yr * g).sum().backward()
    torch.testing.assert_close(y.float(), yr, **_tol(dtype))
    torch.testing.assert_close(x.grad.float(), xr.grad, **_tol(dtype))
    wt = dict(atol=0.5, rtol=5e-2) if dtype != torch.float32 else dict(atol=1e-3, rtol=1e-3)
    torch.testing.assert_close(w.grad.float(), wr.grad, **wt)
    if bias:
        torch.testing.assert_close(b.grad.float(), br.grad, **wt)


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("act", ["silu", "gelu_tanh", "gelu"])
def test_glu_fwd_bwd(dtype, act):
    torch.manual_seed(0)
    gu = torch.randn(333, 2 * 1792, device="cuda", dtype=dtype, requires_grad=True)
    gr = gu.detach().float().requires_grad_(True)
    y = ops.glu(gu, act)
    yr = ops.glu_ref(gr, act)
    g = torch.randn_like(yr)
    (y.float() * g).sum().backward()
    (yr * g).sum().backward()
    torch.testing.assert_close(y.float(), yr, **_tol(dtype))
    torch.testing.assert_close(gu.grad.float(), gr.grad, **_tol(dtype))


@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float32])
def test_bias_act(dtype):
    x = torch.randn(100, 512, device="cuda", dtype=dtype, requires_grad=True)
    b = torch.randn(512, device="cuda", dtype=dtype, requires_grad=True)
    xr, br = x.detach().float().requires_grad_(True), b.detach().float().requires_grad_(True)
    y = ops.bias_act(x, b, "gelu")
    yr = torch.nn.functional.gelu(xr + br)
    y.float().sum().backward()
    yr.sum().backward()
    torch.testing.assert_close(y.float(), yr, **_tol(dtype))
    torch.testing.assert_close(x.grad.float(), xr.grad, **_tol(dtype))


@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float32])
@pytest.mark.parametrize("interleaved,rot", [(False, 128), (False, 64), (True, 64)])
def test_rope_qkv(dtype, interleaved, rot):
    torch.manual_seed(0)
    T, hq, hkv, D = 200, 8, 2, 128
    qkv = torch.randn(T, (hq + 2 * hkv) * D, device="cuda", dtype=dtype, requires_grad=True)
    pos = torch.randint(0, 4096, (T,), device="cuda")
    cos, sin = ops.build_rope_cache(4096, rot, 10000.0, device="cuda")
    out = ops.rope_qkv(qkv, pos, cos, sin, hq, hkv, D, rot_dim=rot, interleaved=interleaved)
    qr = qkv.detach().float().requires_grad_(True)
    x = qr.view(T, hq + 2 * hkv, D)
    ref = torch.cat([ops.rope_ref(x[:, : hq + hkv], pos, cos, sin, rot, interleaved), x[:, hq + hkv:]], 1).reshape(T, -1)
    g = torch.randn_like(ref)
    (out.float() * g).sum().backward()
    (ref * g).sum().backward()
    torch.testing.assert_close(out.float(), ref, **_tol(dtype))
    torch.testing.assert_close(qkv.grad.float(), qr.grad, **_tol(dtype))


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("V,valid,start", [(32000, 32000, 0), (16064, 16000, 16064), (4096, 4096, 8192)])
def test_cross_entropy_blocks(dtype, V, valid, start):
    torch.manual_seed(0)
    T = 257
    logits = (3 * torch.randn(T, V, device="cuda")).to(dtype)
    target = torch.randint(start, start + valid, (T,), device="cuda")
    target[::7] = -100
    target[1::11] = 3   # owned by another rank (unless start == 0)
    with ops.force_torch():
        m_ref = ce.row_max(logits, valid)
        s_ref = ce.sumexp_and_target(logits, target, m_ref, start, -100, valid)
        scale = torch.rand(T, device="cuda")
        g_ref = ce.softmax_grad(logits, target, m_ref, s_ref[0], None, start, -100, row_scale=scale, valid_cols=valid)
    m = ce.row_max(logits, valid)
    s = ce.sumexp_and_target(logits, target, m, start, -100, valid)
    g = ce.softmax_grad(logits, target, m, s[0], None, start, -100, row_scale=scale, valid_cols=valid)
    torch.testing.assert_close(m, m_ref)
    torch.testing.assert_close(s, s_ref, atol=1e-3, rtol=1e-4)
    torch.testing.assert_close(g.float(), g_ref.float(), atol=2e-3 if dtype != torch.float32 else 1e-6, rtol=2e-2)


def test_dist_cross_entropy_matches_torch():
    from colossalai_b200.shardformer.layer.loss import cross_entropy_1d

    torch.manual_seed(0)
    logits = torch.randn(512, 32000, device="cuda", dtype=torch.bfloat16, requires_grad=True)
    tgt = torch.randint(0, 32000, (512,), device="cuda")
    tgt[:17] = -100
    lr = logits.detach().float().requires_grad_(True)
    loss = cross_entropy_1d(logits, tgt, process_group="local", vocab_size=32000)
    ref = torch.nn.functional.cross_entropy(lr, tgt, ignore_index=-100)
    loss.backward()
    ref.backward()
    torch.testing.assert_close(loss, ref, atol=2e-3, rtol=1e-3)
    torch.testing.assert_close(logits.grad.float(), lr.grad, atol=1e-5, rtol=5e-2)


def test_glu_row_limit():
    """`valid_rows`: rows past the device-side limit are neither read nor written, forward and backward."""
    import torch

    from colossalai_b200 import ops

    torch.manual_seed(0)
    x = torch.randn(512, 2 * 256, device="cuda", dtype=torch.bfloat16, requires_grad=True)
    n = torch.tensor(300, device="cuda")
    y = ops.glu(x, "silu", valid_rows=n)
    ref = ops.glu(x.detach()[:300], "silu")
    torch.testing.assert_close(y[:300], ref, atol=0, rtol=0)
    dy = torch.randn(512, 256, device="cuda", dtype=torch.bfloat16)
    (g,) = torch.autograd.grad(y, x, dy)
    xr = x.detach()[:300].clone().requires_grad_(True)
    (gr,) = torch.autograd.grad(ops.glu(xr, "silu"), xr, dy[:300])
    torch.testing.assert_close(g[:300], gr, atol=0, rtol=0)
