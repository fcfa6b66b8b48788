"""wgmma flash-attention forward against an fp32 PyTorch reference (out and log-sum-exp), plus gradients."""
import os

import pytest
import torch

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("B,S,Hq,Hkv,D", [(1, 128, 2, 2, 128), (2, 512, 8, 2, 128), (1, 1024, 4, 4, 64),
                                          (1, 4096, 32, 8, 128)])
@pytest.mark.parametrize("causal", [True, False])
@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16])
def test_flash_fwd_matches_reference(B, S, Hq, Hkv, D, causal, dtype):
    from colossalai_b200.ops import flash_attn_native as fa
    from colossalai_b200.ops.attention import attention_with_lse_ref

    torch.manual_seed(0)
    q = torch.randn(B * S, Hq, D, device="cuda", dtype=dtype)
    k = torch.randn(B * S, Hkv, D, device="cuda", dtype=dtype)
    v = torch.randn(B * S, Hkv, D, device="cuda", dtype=dtype)
    out, lse = fa.flash_fwd(q, k, v, B, causal, None)
    ref_o, ref_lse = attention_with_lse_ref(q.float(), k.float(), v.float(), batch=B, causal=causal)
    torch.cuda.synchronize()
    torch.testing.assert_close(lse, ref_lse, atol=2e-3, rtol=2e-3)
    torch.testing.assert_close(out.float(), ref_o, atol=2e-2, rtol=2e-2)


def test_flash_native_gradients_match_library():
    from colossalai_b200.ops import flash_attn_native as fa

    torch.manual_seed(0)
    B, S, Hq, Hkv, D = 2, 512, 8, 2, 128
    q, k, v = (torch.randn(B * S, h, D, device="cuda", dtype=torch.bfloat16, requires_grad=True) for h in (Hq, Hkv, Hkv))
    fa.enable(True)
    try:
        out = fa.flash_attention(q, k, v, batch=B, causal=True)
        out.float().pow(2).mean().backward()
        got = [t.grad.float().clone() for t in (q, k, v)]
    finally:
        fa.enable(os.environ.get("CB200_FLASH_NATIVE", "0") == "1")
    for t in (q, k, v):
        t.grad = None
    from colossalai_b200.ops.attention import attention_ref

    attention_ref(q, k, v, B, True, None).float().pow(2).mean().backward()
    for g, t in zip(got, (q, k, v)):
        assert (g - t.grad.float()).abs().max() <= 3e-2 * t.grad.float().abs().max() + 1e-6


@pytest.mark.parametrize("B,S,Hq,Hkv", [(1, 128, 2, 2), (1, 256, 4, 1), (2, 512, 8, 2), (1, 2048, 8, 8), (1, 4096, 32, 8)])
@pytest.mark.parametrize("causal", [True, False])
@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16])
def test_flash_bwd_matches_reference(B, S, Hq, Hkv, causal, dtype):
    """wgmma backward (dq, dk, dv) against autograd through the explicit fp32 softmax reference."""
    from colossalai_b200.ops import flash_attn_native as fa
    from colossalai_b200.ops.attention import attention_with_lse_ref

    D = 128
    torch.manual_seed(1)
    q = torch.randn(B * S, Hq, D, device="cuda", dtype=dtype)
    k = torch.randn(B * S, Hkv, D, device="cuda", dtype=dtype)
    v = torch.randn(B * S, Hkv, D, device="cuda", dtype=dtype)
    dout = torch.randn(B * S, Hq, D, device="cuda", dtype=dtype)
    out, lse = fa.flash_fwd(q, k, v, B, causal, None)
    dq, dk, dv = fa.flash_bwd(q, k, v, out, dout, lse, B, causal, None)
    qf, kf, vf = (t.float().requires_grad_(True) for t in (q, k, v))
    ref_o, _ = attention_with_lse_ref(qf, kf, vf, batch=B, causal=causal)
    ref_o.backward(dout.float())
    torch.cuda.synchronize()
    for name, got, ref in (("dq", dq, qf.grad), ("dk", dk, kf.grad), ("dv", dv, vf.grad)):
        err = (got.float() - ref).abs().max().item()
        scale = ref.abs().max().item()
        assert err <= 2e-2 * scale + 1e-3, f"{name}: max err {err:.4g} vs max |ref| {scale:.4g}"
        # no systematic bias: the mean signed error is tiny compared with the mean magnitude
        assert (got.float() - ref).mean().abs().item() <= 2e-3 * ref.abs().mean().item() + 1e-5, name


def _packed_reference(q, k, v, dout, lens, causal):
    """Per-sequence fp32 oracle for a packed batch: returns out, lse, dq, dk, dv."""
    from colossalai_b200.ops.attention import attention_with_lse_ref

    qf, kf, vf = (t.float().requires_grad_(True) for t in (q, k, v))
    outs, lses, s = [], [], 0
    for n in lens:
        o, l = attention_with_lse_ref(qf[s:s + n], kf[s:s + n], vf[s:s + n], batch=1, causal=causal)
        outs.append(o)
        lses.append(l)
        s += n
    out = torch.cat(outs, 0)
    out.backward(dout.float())
    return out.detach(), torch.cat(lses, 0).detach(), qf.grad, kf.grad, vf.grad


@pytest.mark.parametrize("lens", [[128, 256], [100, 128, 333, 1000], [1, 7, 64, 65, 129], [2048, 77]])
@pytest.mark.parametrize("causal", [True, False])
@pytest.mark.parametrize("Hq,Hkv", [(4, 4), (8, 2)])
def test_flash_varlen_fwd_bwd(lens, causal, Hq, Hkv):
    """Packed variable-length batch: cu_seqlens stays on the device, lengths are not multiples of the tile."""
    from colossalai_b200.ops import flash_attn_native as fa

    D, dtype = 128, torch.bfloat16
    T = sum(lens)
    torch.manual_seed(2)
    q = torch.randn(T, Hq, D, device="cuda", dtype=dtype)
    k = torch.randn(T, Hkv, D, device="cuda", dtype=dtype)
    v = torch.randn(T, Hkv, D, device="cuda", dtype=dtype)
    dout = torch.randn(T, Hq, D, device="cuda", dtype=dtype)
    cu = torch.tensor([0] + list(torch.tensor(lens).cumsum(0)), device="cuda", dtype=torch.int32)
    out, lse = fa.flash_fwd(q, k, v, 1, causal, None, cu_seqlens=cu)
    dq, dk, dv = fa.flash_bwd(q, k, v, out, dout, lse, 1, causal, None, cu_seqlens=cu)
    ref_o, ref_lse, rdq, rdk, rdv = _packed_reference(q, k, v, dout, lens, causal)
    torch.cuda.synchronize()
    torch.testing.assert_close(lse, ref_lse, atol=2e-3, rtol=2e-3)
    torch.testing.assert_close(out.float(), ref_o, atol=2e-2, rtol=2e-2)
    for name, got, ref in (("dq", dq, rdq), ("dk", dk, rdk), ("dv", dv, rdv)):
        err = (got.float() - ref).abs().max().item()
        assert err <= 2e-2 * ref.abs().max().item() + 1e-3, f"{name}: max err {err:.4g}"


@pytest.mark.parametrize("lens", [[300, 1000], [128, 640, 77], [2048]])
@pytest.mark.parametrize("window,alibi", [(0, True), (100, False), (256, False), (130, True), (4096, False)])
@pytest.mark.parametrize("Hq,Hkv,D", [(8, 2, 128), (4, 4, 64)])
def test_flash_prefill_window_and_alibi(lens, window, alibi, Hq, Hkv, D):
    """Inference prefill variant: sliding window and / or ALiBi inside the kernel vs an fp32 masked softmax."""
    from colossalai_b200.ops import flash_attn_native as fa

    dtype = torch.bfloat16
    T = sum(lens)
    torch.manual_seed(4)
    q = torch.randn(T, Hq, D, device="cuda", dtype=dtype)
    k = torch.randn(T, Hkv, D, device="cuda", dtype=dtype)
    v = torch.randn(T, Hkv, D, device="cuda", dtype=dtype)
    slopes = (2.0 ** -(torch.arange(1, Hq + 1, device="cuda").float() * 8.0 / Hq)) if alibi else None
    cu = torch.tensor([0] + list(torch.tensor(lens).cumsum(0)), device="cuda", dtype=torch.int32)
    out = fa.flash_prefill(q, k, v, cu, None, window=window, alibi_slopes=slopes)
    torch.cuda.synchronize()
    s0 = 0
    g = Hq // Hkv
    for n in lens:
        qs = q[s0:s0 + n].float().transpose(0, 1)                                  # [Hq, n, D]
        ks = k[s0:s0 + n].float().transpose(0, 1).repeat_interleave(g, 0)
        vs = v[s0:s0 + n].float().transpose(0, 1).repeat_interleave(g, 0)
        sc = qs @ ks.transpose(1, 2) / D ** 0.5
        pos = torch.arange(n, device="cuda")
        rel = pos[None, :] - pos[:, None]                                          # key - query
        if alibi:
            sc = sc + slopes[:, None, None] * rel[None].float()
        keep = rel <= 0
        if window > 0:
            keep = keep & (rel > -window)
        ref = (sc.masked_fill(~keep[None], float("-inf")).softmax(-1) @ vs).transpose(0, 1)
        torch.testing.assert_close(out[s0:s0 + n].float(), ref, atol=2e-2, rtol=2e-2)
        s0 += n


@pytest.mark.parametrize("B,S", [(2, 200), (3, 64), (1, 1000)])
def test_flash_ragged_uniform_lengths(B, S):
    """Equal-length batches whose length is not a multiple of 128."""
    from colossalai_b200.ops import flash_attn_native as fa
    from colossalai_b200.ops.attention import attention_with_lse_ref

    Hq, Hkv, D = 8, 2, 128
    torch.manual_seed(3)
    q = torch.randn(B * S, Hq, D, device="cuda", dtype=torch.bfloat16)
    k = torch.randn(B * S, Hkv, D, device="cuda", dtype=torch.bfloat16)
    v = torch.randn(B * S, Hkv, D, device="cuda", dtype=torch.bfloat16)
    dout = torch.randn_like(q)
    out, lse = fa.flash_fwd(q, k, v, B, True, None)
    dq, dk, dv = fa.flash_bwd(q, k, v, out, dout, lse, B, True, None)
    qf, kf, vf = (t.float().requires_grad_(True) for t in (q, k, v))
    ref_o, ref_lse = attention_with_lse_ref(qf, kf, vf, batch=B, causal=True)
    ref_o.backward(dout.float())
    torch.testing.assert_close(lse, ref_lse, atol=2e-3, rtol=2e-3)
    torch.testing.assert_close(out.float(), ref_o.detach(), atol=2e-2, rtol=2e-2)
    for name, got, ref in (("dq", dq, qf.grad), ("dk", dk, kf.grad), ("dv", dv, vf.grad)):
        assert (got.float() - ref).abs().max().item() <= 2e-2 * ref.abs().max().item() + 1e-3, name


def test_attention_frontend_packed_uses_native_kernels():
    """`ops.attention` with cu_seqlens: one native launch for the whole packed batch, autograd included."""
    from colossalai_b200.kernel import loader
    from colossalai_b200.ops.attention import attention

    lens = [300, 212, 512]
    T, Hq, Hkv, D = sum(lens), 8, 2, 128
    torch.manual_seed(4)
    q, k, v = (torch.randn(T, h, D, device="cuda", dtype=torch.bfloat16, requires_grad=True) for h in (Hq, Hkv, Hkv))
    cu = torch.tensor([0, 300, 512, 1024], device="cuda", dtype=torch.int32)
    before = dict(loader.launch_counter.by_name)
    out = attention(q, k, v, causal=True, cu_seqlens_q=cu, cu_seqlens_k=cu)
    out.float().pow(2).mean().backward()
    after = loader.launch_counter.by_name
    assert after.get("flash_attn_varlen_fwd", 0) == before.get("flash_attn_varlen_fwd", 0) + 1
    assert after.get("flash_attn_bwd", 0) == before.get("flash_attn_bwd", 0) + 1
    dout = (2.0 / out.numel()) * out.detach().float()
    _, _, rdq, rdk, rdv = _packed_reference(q.detach(), k.detach(), v.detach(), dout, lens, True)
    for got, ref in ((q.grad, rdq), (k.grad, rdk), (v.grad, rdv)):
        assert (got.float() - ref).abs().max().item() <= 3e-2 * ref.abs().max().item() + 1e-6


@pytest.mark.parametrize("D", [64, 128])
@pytest.mark.parametrize("rows,Hq,Hkv", [(256, 8, 2), (512, 4, 4), (1024, 8, 8)])
@pytest.mark.parametrize("big_second", [False, True])
def test_flash_block_mode_state_carry(rows, Hq, Hkv, big_second, D):
    """Block mode (ring attention building block): the keys are visited as two blocks by two launches; the second
    launch resumes from the fp32 (output, LSE) state of the first.  `big_second` scales the second block's keys so that
    its scores dominate (the carried accumulator has to be rescaled inside the kernel).  Both head dims the block
    forward accepts."""
    import math

    from colossalai_b200.ops import flash_attn_native as fa

    dtype = torch.bfloat16
    torch.manual_seed(7)
    q = torch.randn(rows, Hq, D, device="cuda", dtype=dtype)
    k = torch.randn(2 * rows, Hkv, D, device="cuda", dtype=dtype)
    v = torch.randn(2 * rows, Hkv, D, device="cuda", dtype=dtype)
    if big_second:
        k[rows:] *= 4.0
    o_state = torch.empty(rows, Hq, D, device="cuda", dtype=torch.float32)
    lse = torch.empty(rows, Hq, device="cuda", dtype=torch.float32)
    scale = 1.0 / math.sqrt(D)
    for blk, (causal, has_prev) in enumerate([(0, 0), (1, 1)]):
        fa.flash_block_fwd(q.data_ptr(), k[blk * rows:].data_ptr(), v[blk * rows:].data_ptr(), o_state.data_ptr(),
                           lse.data_ptr(), rows, Hq, Hkv, D, causal, has_prev, scale, dtype)
    torch.cuda.synchronize()
    # oracle: queries are the LAST `rows` positions of a 2*rows sequence (first block fully visible, second causal)
    g = Hq // Hkv
    qs = q.float().transpose(0, 1)
    ks = k.float().transpose(0, 1).repeat_interleave(g, 0)
    vs = v.float().transpose(0, 1).repeat_interleave(g, 0)
    sc = qs @ ks.transpose(1, 2) * scale
    qpos = torch.arange(rows, device="cuda") + rows
    keep = torch.arange(2 * rows, device="cuda")[None, :] <= qpos[:, None]
    sc = sc.masked_fill(~keep[None], float("-inf"))
    ref = (sc.softmax(-1) @ vs).transpose(0, 1)
    ref_lse = torch.logsumexp(sc, -1).transpose(0, 1)
    torch.testing.assert_close(lse, ref_lse, atol=3e-3, rtol=3e-3)
    torch.testing.assert_close(o_state, ref, atol=2e-2, rtol=2e-2)


@pytest.mark.parametrize("rows,Hq,Hkv", [(256, 8, 2), (512, 4, 4), (200, 8, 2)])
@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16])
def test_flash_block_mode_backward(rows, Hq, Hkv, dtype):
    """Block-mode backward (ring attention building block) on one GPU: the queries are the last `rows` positions of a
    2*rows sequence, the keys two blocks (the first fully visible, the second causal).  Each block's backward adds into
    the same fp32 dQ / dK / dV accumulators, with the merged forward's LSE and delta."""
    from colossalai_b200.ops import flash_attn_native as fa
    from colossalai_b200.ops.attention import attention_with_lse_ref

    D = 128
    scale = D ** -0.5
    torch.manual_seed(8)
    q = torch.randn(rows, Hq, D, device="cuda", dtype=dtype)
    k = torch.randn(2 * rows, Hkv, D, device="cuda", dtype=dtype)
    v = torch.randn(2 * rows, Hkv, D, device="cuda", dtype=dtype)
    dout = torch.randn(rows, Hq, D, device="cuda", dtype=dtype)
    o_state = torch.empty(rows, Hq, D, device="cuda", dtype=torch.float32)
    lse = torch.empty(rows, Hq, device="cuda", dtype=torch.float32)
    blocks = [(0, False), (1, True)]                      # (key block, causal)
    for blk, causal in blocks:
        fa.flash_block_fwd(q.data_ptr(), k[blk * rows:].data_ptr(), v[blk * rows:].data_ptr(), o_state.data_ptr(),
                           lse.data_ptr(), rows, Hq, Hkv, D, causal, blk > 0, scale, dtype)
    delta = fa.flash_delta(o_state.to(dtype), dout)
    dq_acc = torch.zeros(rows, Hq, D, device="cuda", dtype=torch.float32)
    dk_acc = torch.zeros(2 * rows, Hkv, D, device="cuda", dtype=torch.float32)
    dv_acc = torch.zeros_like(dk_acc)
    for blk, causal in blocks:
        fa.flash_block_bwd(q.data_ptr(), k[blk * rows:].data_ptr(), v[blk * rows:].data_ptr(), dout.data_ptr(),
                           lse.data_ptr(), delta.data_ptr(), dq_acc.data_ptr(), dk_acc[blk * rows:].data_ptr(),
                           dv_acc[blk * rows:].data_ptr(), rows, Hq, Hkv, D, causal, scale, dtype)
    qf, kf, vf = (t.float().requires_grad_(True) for t in (q, k, v))
    ref_o, _ = attention_with_lse_ref(qf, kf, vf, batch=1, causal=True, scale=scale)     # bottom-right causal
    ref_o.backward(dout.float())
    torch.cuda.synchronize()
    for name, got, ref in (("dq", dq_acc, qf.grad), ("dk", dk_acc, kf.grad), ("dv", dv_acc, vf.grad)):
        err = (got - ref).abs().max().item()
        scale_ = ref.abs().max().item()
        assert err <= 2e-2 * scale_ + 1e-3, f"{name}: max err {err:.4g} vs max |ref| {scale_:.4g}"
        assert (got - ref).mean().abs().item() <= 2e-3 * ref.abs().mean().item() + 1e-5, name


def test_flash_fwd_launcher_rejects_out_of_envelope():
    """The forward launcher validates before anything else, empty problems included: every call outside its envelope
    fails with cudaErrorInvalidValue (1) and writes nothing."""
    from colossalai_b200.ops import flash_attn_native as fa

    T, Hq, Hkv, D, dtype = 256, 4, 2, 128, torch.bfloat16
    torch.manual_seed(9)
    q = torch.randn(T, Hq, D, device="cuda", dtype=dtype)
    k = torch.randn(T, Hkv, D, device="cuda", dtype=dtype)
    v = torch.randn(T, Hkv, D, device="cuda", dtype=dtype)
    out = torch.full_like(q, float("nan"))
    lse = torch.full((T, Hq), float("nan"), device="cuda")
    o_state = torch.full((T, Hq, D), float("nan"), device="cuda")
    cu = torch.tensor([0, 100, T], device="cuda", dtype=torch.int32)
    slopes = torch.ones(Hq, device="cuda")
    uniform = dict(q=q.data_ptr(), k=k.data_ptr(), v=v.data_ptr(), out=out.data_ptr(), lse=lse.data_ptr(), batch=1,
                   seqlen_q=T, seqlen_k=T, hq=Hq, hkv=Hkv, d=D, causal=True, scale=D ** -0.5, dtype=dtype)
    packed = dict(uniform, batch=2, seqlen_q=0, seqlen_k=0, cu_seqlens=cu.data_ptr(), total_tokens=T)
    block = dict(uniform, out=0, o_state=o_state.data_ptr())
    rejected = {
        "fp32": dict(uniform, dtype=torch.float32),
        "head_dim 96": dict(uniform, d=96),
        "hq % hkv != 0": dict(uniform, hq=3),
        "hkv 0": dict(uniform, hkv=0),
        "causal, seqlen_q != seqlen_k": dict(uniform, seqlen_k=T // 2),
        "window without cu_seqlens": dict(uniform, window=64),
        "alibi without cu_seqlens": dict(uniform, alibi=slopes.data_ptr()),
        "negative window": dict(packed, window=-1),
        "window, not causal": dict(packed, causal=False, window=64),
        "alibi, not causal": dict(packed, causal=False, alibi=slopes.data_ptr()),
        "block mode, null lse": dict(block, lse=0),
        "block mode with cu_seqlens": dict(block, cu_seqlens=cu.data_ptr(), total_tokens=T),
        "has_prev without o_state": dict(uniform, has_prev=True),
        "empty, head_dim 96": dict(uniform, batch=0, d=96),
        "empty packed, fp32": dict(packed, total_tokens=0, dtype=torch.float32),
    }
    for name, args in rejected.items():
        with pytest.raises(RuntimeError, match=r"CUDA error 1$"):
            fa._fwd(name, **args)
    torch.cuda.synchronize()
    for t in (out, lse, o_state):
        assert torch.isnan(t).all(), "a rejected call wrote its output"
    # the same buffers are written by calls inside the envelope
    fa._fwd("uniform", **uniform)
    fa._fwd("block", **block)
    torch.cuda.synchronize()
    for t in (out, lse, o_state):
        assert torch.isfinite(t).all()
