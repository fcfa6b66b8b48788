"""The memory-bound training kernels against float64 references, at tolerances that can fail.

Every reference here is plain PyTorch in float64, computed from the exact 16-bit (or fp32) values the kernel read.
Each element is checked against

    |got - ref| <= k * ulp_out(|ref|) + floor

where `ulp_out` is the output dtype's spacing at that magnitude (2^-8 relative for bf16, 2^-11 for fp16, 2^-22 for
fp32 to leave room for `__expf`; never below the dtype's subnormal step), `k` is 2 or 3, and `floor` is the
rounding bound of the fp32 arithmetic the kernel performs: `depth * 2^-24 * sum|terms|` for a sum whose longest
chain of sequential fp32 adds is `depth` (a per-thread loop followed by a shuffle / shared-memory tree), plus the
argument error of the fast exponential where the kernel uses one.  `check` refuses a floor above 1% of the median
|ref|, so a loosened floor fails loudly instead of making a comparison vacuous.  Elements whose reference is
exactly zero (masked keys, padded vocabulary columns, ignored rows, an all-zero row's output) must be exactly zero.

Backward references take what the kernel saved as their input, because that is the operation the kernel defines:
the forward output `y` for softmax, the residual stream `h` for RMSNorm (statistics recomputed in float64).

Shapes are chosen per launch branch; the arithmetic is next to each case.  On an H100 (132 SMs):
  * `ew_grid` caps the elementwise kernels at 16 * 132 = 2112 CTAs of 256 threads = 540,672 work items per trip;
  * `grid_for` caps the fp8 kernels at 8 * 132 = 1056 CTAs;
  * `cb_norm_bwd_grid(rows)` = min(rows, 2 * 132 = 264) persistent backward CTAs.
"""
import math

import pytest
import torch

from colossalai_b200.ops._align import aligned, is_aligned, rows_aligned

U = 2.0 ** -24                                                     # fp32 unit roundoff
_REL = {torch.bfloat16: 2.0 ** -8, torch.float16: 2.0 ** -11, torch.float32: 2.0 ** -22}
_SUB = {torch.bfloat16: 2.0 ** -133, torch.float16: 2.0 ** -24, torch.float32: 2.0 ** -149}
DTYPES = [torch.bfloat16, torch.float16, torch.float32]
_WORST = {}                                                        # kernel -> largest |err| / tol seen


def ulp_out(ref: torch.Tensor, dtype: torch.dtype) -> torch.Tensor:
    return (ref.abs() * _REL[dtype]).clamp_min(_SUB[dtype])


def check(what, got, ref, dtype, k=2, floor=0.0):
    """Assert |got - ref| <= k * ulp_out(|ref|) + floor elementwise (see the module docstring)."""
    got, ref = got.double(), ref.double()
    assert got.shape == ref.shape, (what, got.shape, ref.shape)
    assert torch.isfinite(ref).all(), f"{what}: non-finite reference"
    zero = ref == 0
    nz_zero = int((got[zero] != 0).sum())
    assert nz_zero == 0, f"{what}: {nz_zero} elements whose reference is exactly 0 are not 0"
    nz = ~zero
    if not nz.any():
        return
    floor = torch.as_tensor(floor, dtype=torch.float64, device=ref.device).expand_as(ref)
    med = ref[nz].abs().median()
    assert floor[nz].median() <= 0.01 * med, f"{what}: floor {floor[nz].median():.3g} > 1% of median |ref| {med:.3g}"
    tol = k * ulp_out(ref, dtype) + floor
    err = (got - ref).abs()
    bad = nz & ~(err <= tol)                    # NaN in `got` counts as bad
    if bad.any():
        i = int(bad.flatten().nonzero()[0])
        raise AssertionError(f"{what}: {int(bad.sum())} of {int(nz.sum())} elements out of tolerance; first at flat "
                             f"index {i}: got {got.flatten()[i].item():.9g} ref {ref.flatten()[i].item():.9g} "
                             f"tol {tol.flatten()[i].item():.3g}")
    ratio = float((err[nz] / tol[nz]).max())
    name = what.split(" ")[0]
    _WORST[name] = max(_WORST.get(name, 0.0), ratio)


@pytest.fixture(scope="module", autouse=True)
def _report_worst():
    yield
    if _WORST:
        print("\nlargest error-to-tolerance ratio per kernel:")
        for k, v in sorted(_WORST.items()):
            print(f"  {k:<24} {v:.3f}")
        if torch.cuda.is_available():
            print(f"peak CUDA memory allocated: {torch.cuda.max_memory_allocated() / 2**30:.2f} GiB")


def _f32(x: float) -> float:
    return float(torch.tensor(x, dtype=torch.float32))


# ============================================================================================ comparator (CPU)
@pytest.mark.parametrize("dtype", DTYPES)
def test_comparator_rejects_corruptions(dtype):
    """Each corruption a broken kernel could produce is rejected; the reference rounded to `dtype` is accepted."""
    g = torch.Generator().manual_seed(0)
    x = torch.randn(64, 512, generator=g, dtype=torch.float64)
    ref = torch.softmax(0.5 * x, -1)
    floor = ref * (512 / 32 + 5) * U                                   # a warp-row sum of 512 terms
    check("selftest exact", ref.to(dtype), ref, dtype, floor=floor)

    def rejected(bad):
        with pytest.raises(AssertionError):
            check("selftest corrupt", bad.to(dtype), ref, dtype, floor=floor)

    z = ref.clone(); z[5] = 0; rejected(z)                              # one zeroed row
    z = ref.clone(); z[:, 128:256] = 0; rejected(z)                     # one zeroed 128-column block
    rejected(torch.roll(ref, 1, dims=1))                                # output shifted by one column
    rejected(ref * (1 + 2.0 ** -6))                                     # every element 1.6% too large

    # a column reduction over rows (a norm's dw) missing one row's contribution
    dy, xhat = torch.randn(512, 256, generator=g, dtype=torch.float64), torch.randn(512, 256, generator=g,
                                                                                   dtype=torch.float64)
    dw = (dy * xhat).sum(0)
    dw_floor = (2 + 264) * U * (dy * xhat).abs().sum(0)
    check("selftest dw", dw.to(dtype), dw, dtype, floor=dw_floor)
    with pytest.raises(AssertionError):
        check("selftest dw", (dw - dy[-1] * xhat[-1]).to(dtype), dw, dtype, floor=dw_floor)
    # a floor that has grown to swamp the values is refused outright
    with pytest.raises(AssertionError, match="floor"):
        check("selftest floor", ref.to(dtype), ref, dtype, floor=ref.abs().median() * 0.02)


# ============================================================================================ alignment (CPU)
def test_alignment_predicate_on_offset_views():
    buf = torch.zeros(4096, dtype=torch.bfloat16)
    assert is_aligned(buf) and is_aligned(None)
    for k in range(32):
        view = buf[k:k + 1024]
        assert view.is_contiguous()
        assert is_aligned(view) == (view.data_ptr() % 16 == 0) == (k % 8 == 0), k
    raw = torch.zeros(64, dtype=torch.uint8)
    for k in range(8):
        assert is_aligned(raw[k:], 4) == (k % 4 == 0)
    assert rows_aligned(buf.view(64, 64))
    assert not rows_aligned(buf[:63 * 9].view(63, 9))                   # 18-byte rows
    assert not rows_aligned(buf[8:8 + 63 * 64].view(63, 64)[:, 1:])     # rows start 2 bytes in
    off = buf[3:3 + 512]
    off.copy_(torch.arange(512, dtype=torch.bfloat16))
    c = aligned(off)
    assert c is not off and is_aligned(c) and torch.equal(c, off)
    assert aligned(buf) is buf


# ============================================================================================ GPU helpers
def _cuda():
    if not torch.cuda.is_available():
        pytest.skip("needs a GPU")
    return torch.device("cuda")


def _sm_count():
    return torch.cuda.get_device_properties(0).multi_processor_count


def _rand(shape, dtype, scale=1.0, seed=0):
    g = torch.Generator(device="cuda").manual_seed(seed)
    return (torch.randn(shape, device="cuda", generator=g, dtype=torch.float32) * scale).to(dtype)


# ============================================================================================ softmax
# Warp kernel: one warp per row, PER = 1, 2, 4, 8, 16, 32 elements per lane for sk <= 32, 64, 128, 256, 512, 1024.
# CTA kernel (256 threads) above 1024.  The sizes sit on both sides of every boundary:
#   1, 31 -> PER 1;  33, 64 -> PER 2;  65 -> PER 4;  200, 256 -> PER 8;  257, 512 -> PER 16;  513, 1024 -> PER 32;
#   1025, 4096, 4097, 8193 -> CTA per row (5, 16, 17, 33 columns per thread).
SOFTMAX_SK = [1, 31, 33, 64, 65, 200, 256, 257, 512, 513, 1024, 1025, 4096, 4097, 8193]


def _softmax_depth(sk):
    """Longest fp32 add chain of the row sums: per-lane loop + 5 shuffles (warp kernel), or per-thread loop +
    5 shuffles + 5 more over the 8 warp partials (CTA kernel)."""
    if sk <= 1024:
        return 2 ** math.ceil(math.log2(max(1, math.ceil(sk / 32)))) + 5
    return math.ceil(sk / 256) + 10


def _softmax_case(kind, sk):
    if kind == "mask":
        return 2, 2, 8
    if kind == "mask_b1":
        return 2, 2, 5
    if kind == "causal_short":                   # sq < sk (sq == sk when sk == 1)
        return 2, 1, max(1, min(sk - 1, 24))
    return 1, 1, sk + (7 if sk <= 64 else 3)     # causal_tall: sq > sk, the first sq - sk rows see no key


@pytest.mark.gpu
@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("sk", SOFTMAX_SK)
@pytest.mark.parametrize("kind", ["mask", "mask_b1", "causal_short", "causal_tall"])
def test_softmax_envelope(dtype, sk, kind):
    _cuda()
    from colossalai_b200.ops.softmax import scaled_causal_softmax, scaled_masked_softmax

    if kind == "causal_tall" and sk > 1025:
        pytest.skip("sq > sk is covered on both kernels up to sk = 1025; larger squares only cost memory")
    b, h, sq = _softmax_case(kind, sk)
    scale = 0.6
    s32 = _f32(scale)
    x = _rand((b, h, sq, sk), dtype, seed=sk).requires_grad_(True)
    x64 = x.detach().double()
    t = x64 * s32
    if kind.startswith("mask"):
        mb = 1 if kind == "mask_b1" else b
        g = torch.Generator(device="cuda").manual_seed(1)
        mask = torch.rand((mb, 1, sq, sk), device="cuda", generator=g) < 0.25
        mask[:, :, 1] = True                                    # a fully masked row: uniform 1/sk
        y = scaled_masked_softmax(x, mask, scale)
        unm = (~mask).expand(b, h, sq, sk)
        t = t.masked_fill(~unm, -10000.0)
    else:
        y = scaled_causal_softmax(x, scale)
        keep = torch.ones(sq, sk, dtype=torch.bool, device="cuda").tril(diagonal=sk - sq)
        unm = keep.expand(b, h, sq, sk)
        t = t.masked_fill(~unm, float("-inf"))
    # float64 softmax; rows without a visible key give 0 (what the kernel writes)
    empty = ~torch.isfinite(t).any(-1, keepdim=True)
    ref = torch.softmax(t.masked_fill(empty, 0.0), -1).masked_fill(empty, 0.0)
    depth = _softmax_depth(sk)
    m = t.amax(-1, keepdim=True)
    # each term: fp32 rounding of x*scale (unmasked only) and of the row max, then t - m and the exp2 argument
    term = 2.0 ** -22 + U * (unm * t.abs().nan_to_num(0, 0, 0) + m.abs().nan_to_num(0, 0, 0) * unm.any(-1, True)
                             + 3 * (t - m).abs().nan_to_num(0, 0, 0))
    term = term * (ref > 0)                                    # masked keys add exactly 0 to the sum
    floor = ref * (depth * U + term.amax(-1, keepdim=True) + term)
    check(f"softmax_fwd {kind} sk={sk}", y, ref, dtype, floor=floor)

    dy = _rand(y.shape, dtype, seed=sk + 1)
    (dx,) = torch.autograd.grad(y, x, dy)
    y64, dy64 = y.detach().double(), dy.double()
    dot = (dy64 * y64).sum(-1, keepdim=True)
    ref_dx = s32 * y64 * (dy64 - dot)
    floor_dx = s32 * y64.abs() * (depth + 1) * U * (dy64 * y64).abs().sum(-1, keepdim=True)
    check(f"softmax_bwd {kind} sk={sk}", dx, ref_dx, dtype, floor=floor_dx)


@pytest.mark.gpu
def test_causal_softmax_reference_agrees_on_rows_without_keys():
    _cuda()
    from colossalai_b200.ops.softmax import scaled_causal_softmax, scaled_causal_softmax_ref

    x = _rand((3, 40, 16), torch.float32)
    y = scaled_causal_softmax(x, 0.5)
    r = scaled_causal_softmax_ref(x, 0.5)
    assert torch.isfinite(r).all() and (y[:, :24] == 0).all() and (r[:, :24] == 0).all()
    torch.testing.assert_close(y, r, rtol=1e-5, atol=1e-7)


# ============================================================================================ cross entropy
# One CTA of 512 threads per row, 16-byte loads: a thread's chain is ceil(Vv / (512 * VEC)) * VEC adds, then
# 5 shuffles + 5 over the 16 warp partials.  V = 8 is less than one vector per thread in the first warp;
# 151936 bf16 = 37.1 vectors of 4096 per row, so the last trip is partial.
CE_V = [8, 4096, 32000, 128256, 151936]


def _ce_depth(Vv, dtype):
    vec = 4 if dtype == torch.float32 else 8
    return math.ceil(max(Vv, 1) / (512 * vec)) * vec + 10


@pytest.mark.gpu
@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("V", CE_V)
@pytest.mark.parametrize("case", ["full", "padded", "offset", "large"])
def test_cross_entropy_blocks_envelope(dtype, V, case):
    _cuda()
    from colossalai_b200.ops import cross_entropy as ce

    T, ignore = 48, -100
    Vv = V if case in ("full", "large") else V - 3                     # padded: last 3 columns hold no vocabulary
    start = 5 * V if case == "offset" else 0
    if case == "offset":
        Vv = V
    base = 1000.0 if case == "large" else 0.0                         # exp(1000) overflows without the max shift
    logits = (base + _rand((T, V), torch.float32, 3.0, seed=V)).to(dtype)
    g = torch.Generator(device="cuda").manual_seed(2)
    target = torch.randint(start, start + Vv, (T,), device="cuda", generator=g)
    target[::7] = ignore
    target[3::11] = start + Vv + 17 if case != "full" else start - 1  # owned by another rank
    target[0] = start + Vv - 1                                        # last valid column
    x64 = logits.double()[:, :Vv]

    m = ce.row_max(logits, Vv)
    assert torch.equal(m, logits[:, :Vv].float().amax(-1)), "row_max"
    st = ce.sumexp_and_target(logits, target, m, start, ignore, Vv)
    m64 = m.double()[:, None]
    e = torch.exp(x64 - m64)
    d = (x64 - m64).abs()
    term = 2.0 ** -22 + 3 * U * d
    s_ref = e.sum(-1)
    s_floor = _ce_depth(Vv, dtype) * U * s_ref + (e * term).sum(-1)
    check(f"ce_sumexp V={V} {case}", st[0], s_ref, torch.float32, k=3, floor=s_floor)
    local = target - start
    own = (target != ignore) & (local >= 0) & (local < Vv)
    tl = torch.where(own, logits.float().gather(1, local.clamp(0, V - 1)[:, None])[:, 0], torch.zeros_like(m))
    assert torch.equal(st[1], tl), "target logit"

    rs = torch.rand(T, device="cuda", generator=g) + 0.5
    grad = ce.softmax_grad(logits, target, m, st[0], None, start, ignore, row_scale=rs, valid_cols=Vv)
    p = e / st[0].double()[:, None]                                   # the kernel's saved sum-exp is an input
    onehot = torch.zeros_like(p)
    onehot[own.nonzero()[:, 0], local[own]] = 1.0
    rs64 = rs.double()[:, None]
    ref = rs64 * (p - onehot)
    floor = rs64 * p * (2.0 ** -21 + (3 * d + 4) * U)                 # fp32 divide, exp argument, two products
    live = (target != ignore)[:, None]
    ref, floor = ref * live, floor * live
    ref = torch.cat([ref, ref.new_zeros(T, V - Vv)], 1)
    floor = torch.cat([floor, floor.new_zeros(T, V - Vv)], 1)
    check(f"ce_softmax_grad V={V} {case}", grad, ref, dtype, floor=floor)


@pytest.mark.gpu
@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float32])
def test_cross_entropy_1d_gradient_envelope(dtype):
    """The whole vocab-parallel loss (one rank) against a float64 cross entropy, loss and every gradient element."""
    _cuda()
    from colossalai_b200.shardformer.layer.loss import cross_entropy_1d

    T, V = 512, 32000
    logits = _rand((T, V), dtype, 2.0).requires_grad_(True)
    tgt = torch.randint(0, V, (T,), device="cuda", generator=torch.Generator(device="cuda").manual_seed(3))
    tgt[:17] = -100
    loss = cross_entropy_1d(logits, tgt, process_group="local", vocab_size=V)
    (grad,) = torch.autograd.grad(loss, logits)
    x64 = logits.detach().double()
    valid = tgt != -100
    n = int(valid.sum())
    lse = torch.logsumexp(x64, -1)
    tok = lse - x64.gather(1, tgt.clamp_min(0)[:, None])[:, 0]
    ref_loss = (tok * valid).sum() / n
    depth = _ce_depth(V, dtype)
    m = x64.amax(-1)
    tok_err = (depth + 4) * U + 2.0 ** -22 + 3 * U * (x64 - m[:, None]).abs().amax(-1) + 2 * U * (lse.abs() + m.abs())
    loss_floor = ((tok_err * valid).sum() + (T + 2) * U * (tok * valid).abs().sum()) / n
    check("ce_1d_loss", loss.reshape(1), ref_loss.reshape(1), torch.float32, k=3, floor=loss_floor)
    p = torch.exp(x64 - lse[:, None])
    onehot = torch.zeros_like(p)
    onehot[valid.nonzero()[:, 0], tgt[valid]] = 1.0
    ref = (p - onehot) * valid[:, None] / n
    floor = p / n * ((depth + 4) * U + 2.0 ** -21 + 3 * U * (x64 - m[:, None]).abs()) * valid[:, None]
    check("ce_1d_grad", grad, ref, dtype, floor=floor)


# ============================================================================================ RMSNorm / LayerNorm
# block = 32 * ceil(H / VEC / 32) threads, capped at 1024; iters = ceil(H / VEC / block) -> MAX_ITERS 1, 2 or 4.
#   16-bit (VEC 8):  H 256 -> 32 threads;  768 -> 96;  5120 -> 640;  12288 = 1536 vectors -> 1024 x 2 iterations,
#                    the second half full (partial last iteration);  20480 = 2560 vectors -> 3 iterations, run by
#                    MAX_ITERS = 4;  32768 = 4096 vectors -> 4 full iterations, the gate's maximum.
#   fp32 (VEC 4):    H 128 -> 32;  384 -> 96;  2560 -> 640;  6144 -> 1024 x 2 partial;  10240 -> 3;  16384 -> 4.
# Rows: 1;  263 = one fewer than the 264 backward CTAs (each CTA one row);  264;  4099 = 15.5 rows per CTA
# (4099 only at the narrow widths, to keep the float64 references small).
def _norm_cases():
    cases = []
    for H16, H32, rows in [(256, 128, (1, 263, 264, 4099)), (768, 384, (1, 263, 264, 4099)),
                           (5120, 2560, (1, 263, 264)), (12288, 6144, (263, 264)),
                           (20480, 10240, (1, 264)), (32768, 16384, (1, 263))]:
        for r in rows:
            cases.append((H16, H32, r))
    return cases


def _norm_inputs(rows, H, dtype, seed):
    x = _rand((rows, H), torch.float32, 1.0, seed)
    if rows > 2:
        x[1] = 0.0                                     # all-zero row: y = b, rstd = 1/sqrt(eps)
        x[2] *= 3e-3                                   # mean(x^2) ~ 9e-6, comparable to eps = 1e-5
    return x.to(dtype)


def _stat_depth(H, dtype):
    vec = 4 if dtype == torch.float32 else 8
    block = min(1024, max(32, 32 * math.ceil(H / vec / 32)))
    return math.ceil(H / vec / block) * vec + 10


@pytest.mark.gpu
@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("H16,H32,rows", _norm_cases())
@pytest.mark.parametrize("with_res", [False, True])
def test_rmsnorm_envelope(dtype, H16, H32, rows, with_res):
    _cuda()
    from colossalai_b200 import ops

    H = H32 if dtype == torch.float32 else H16
    eps = 1e-5
    x = _norm_inputs(rows, H, dtype, 0).requires_grad_(True)
    w = (1 + 0.2 * _rand((H,), torch.float32, seed=1)).to(dtype).requires_grad_(True)
    res = (0.5 * _rand((rows, H), torch.float32, seed=2)).to(dtype) if with_res else None
    if with_res and rows > 2:
        res[1] = 0.0
        res[2] *= 3e-3
    if with_res:
        res.requires_grad_(True)
        y, h = ops.rms_norm(x, w, eps, res)
        check(f"rmsnorm_fwd_h H={H} rows={rows}", h, x.detach().double() + res.detach().double(), dtype)
    else:
        y, h = ops.rms_norm(x, w, eps), x
    h64, w64 = h.detach().double(), w.detach().double()
    depth = _stat_depth(H, dtype)
    ms = h64.square().mean(-1, keepdim=True)
    rs = (ms + eps).rsqrt()
    d_rs = depth * U + 2.0 ** -21                          # sum of squares, divide, rsqrtf
    xhat = h64 * rs
    check(f"rmsnorm_fwd H={H} rows={rows}", y, xhat * w64, dtype, floor=(xhat * w64).abs() * d_rs)

    dy = _rand((rows, H), dtype, seed=3)
    outs, gouts = (y,), (dy,)
    if with_res:
        dh = _rand((rows, H), dtype, seed=4)
        outs, gouts = (y, h), (dy, dh)
    inputs = (x, w) + ((res,) if with_res else ())
    grads = torch.autograd.grad(outs, inputs, gouts)
    dy64 = dy.double()
    gw = dy64 * w64
    c1 = (gw * xhat).mean(-1, keepdim=True)
    dx_ref = rs * (gw - xhat * c1) + (dh.double() if with_res else 0)
    c1_err = depth * U * (gw * xhat).abs().mean(-1, keepdim=True) + (gw * xhat).abs().mean(-1, keepdim=True) * d_rs
    dx_floor = rs * ((gw.abs() + 2 * (xhat * c1).abs()) * (d_rs + 2 * U) + xhat.abs() * c1_err)
    check(f"rmsnorm_bwd_dx H={H} rows={rows}", grads[0], dx_ref, dtype, floor=dx_floor)
    if with_res:
        assert torch.equal(grads[2], grads[0])
    grid = min(rows, 2 * _sm_count())
    dw_depth = math.ceil(rows / grid) + grid + 2
    t = dy64 * xhat
    check(f"rmsnorm_bwd_dw H={H} rows={rows}", grads[1], t.sum(0), dtype,
          floor=dw_depth * U * t.abs().sum(0) + t.abs().sum(0) * d_rs)


@pytest.mark.gpu
@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("H16,H32,rows", _norm_cases())
@pytest.mark.parametrize("with_bias", [False, True])
def test_layernorm_envelope(dtype, H16, H32, rows, with_bias):
    _cuda()
    from colossalai_b200 import ops

    H = H32 if dtype == torch.float32 else H16
    eps = 1e-5
    x = (_norm_inputs(rows, H, torch.float32, 5) + 0.5).to(dtype)       # a non-zero mean
    if rows > 2:
        x[1] = 0
    x.requires_grad_(True)
    w = (1 + 0.2 * _rand((H,), torch.float32, seed=6)).to(dtype).requires_grad_(True)
    b = (0.1 * _rand((H,), torch.float32, seed=7)).to(dtype).requires_grad_(True) if with_bias else None
    y = ops.layer_norm(x, w, b, eps)
    x64, w64 = x.detach().double(), w.detach().double()
    b64 = b.detach().double() if with_bias else 0.0
    depth = _stat_depth(H, dtype)
    mu = x64.mean(-1, keepdim=True)
    xc = x64 - mu
    rs = (xc.square().mean(-1, keepdim=True) + eps).rsqrt()
    d_mu = depth * U * x64.abs().mean(-1, keepdim=True) + U * mu.abs()
    d_rs = depth * U + 2.0 ** -21 + (rs * d_mu).square()             # a mean error moves the variance to 2nd order
    xhat = xc * rs
    dxhat = rs * d_mu + xhat.abs() * (d_rs + U)                         # error of the kernel's xhat
    y_ref = xhat * w64 + b64
    check(f"layernorm_fwd H={H} rows={rows}", y, y_ref, dtype, floor=w64.abs() * dxhat + U * y_ref.abs())

    dy = _rand((rows, H), dtype, seed=8)
    grads = torch.autograd.grad(y, (x, w) + ((b,) if with_bias else ()), dy)
    dy64 = dy.double()
    gw = dy64 * w64
    c0, c1 = gw.mean(-1, keepdim=True), (gw * xhat).mean(-1, keepdim=True)
    dx_ref = rs * (gw - c0 - xhat * c1)
    c0_err = depth * U * gw.abs().mean(-1, keepdim=True)
    c1_err = depth * U * (gw * xhat).abs().mean(-1, keepdim=True) + (gw.abs() * dxhat).mean(-1, keepdim=True)
    dx_floor = rs * ((gw.abs() + c0.abs() + (xhat * c1).abs()) * (d_rs + 3 * U) + c0_err
                     + dxhat * c1.abs() + xhat.abs() * c1_err)
    check(f"layernorm_bwd_dx H={H} rows={rows}", grads[0], dx_ref, dtype, floor=dx_floor)
    grid = min(rows, 2 * _sm_count())
    dw_depth = math.ceil(rows / grid) + grid + 2
    t = dy64 * xhat
    check(f"layernorm_bwd_dw H={H} rows={rows}", grads[1], t.sum(0), dtype,
          floor=dw_depth * U * t.abs().sum(0) + (dy64.abs() * dxhat).sum(0))
    if with_bias:
        check(f"layernorm_bwd_db H={H} rows={rows}", grads[2], dy64.sum(0), dtype,
              floor=dw_depth * U * dy64.abs().sum(0))


# ============================================================================================ GLU / bias-act
def _act64(x, act):
    if act == "silu":
        return x * torch.sigmoid(x)
    if act == "gelu_tanh":   # 0.5 x (1 + tanh u) == x sigmoid(2u), without the cancellation for x << 0
        return x * torch.sigmoid(2 * math.sqrt(2 / math.pi) * (x + 0.044715 * x ** 3))
    return 0.5 * x * (1 + torch.erf(x / math.sqrt(2)))


def _act_grad64(x, act):
    xx = x.detach().clone().requires_grad_(True)
    (g,) = torch.autograd.grad(_act64(xx, act).sum(), xx)
    return g


def _act_err(x):
    """Bound on the fp32 error of act(x) and act'(x) as the kernels evaluate them (__expf, erff, fast divide)."""
    return 8 * U * (2 + x.abs()) ** 3


def _check_glu(what, gu, y, dy, dgu, act, dtype):
    """GLU forward and backward against float64, 256 rows at a time to keep the references small."""
    for r in range(0, y.shape[0], 256):
        g64, u64 = gu[r:r + 256].double().chunk(2, -1)
        a, err, d64 = _act64(g64, act), _act_err(g64), dy[r:r + 256].double()
        check(f"glu_fwd_{act} {what}", y[r:r + 256], a * u64, dtype, floor=u64.abs() * err)
        check(f"glu_bwd_{act} {what}", dgu[r:r + 256],
              torch.cat([d64 * u64 * _act_grad64(g64, act), d64 * a], -1), dtype,
              floor=torch.cat([(d64 * u64).abs() * err, d64.abs() * err], -1))


# GLU: items = rows * I / VEC.  16-bit 1024 x 14336 / 8 = 1.84M items = 3.4 trips of the 540,672-item grid;
# fp32 1024 x 7168 / 4 = 1.84M items, 3.4 trips.  333 x 1792 / 8 = 74.6k items is one partial trip.
@pytest.mark.gpu
@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("act", ["silu", "gelu_tanh", "gelu"])
@pytest.mark.parametrize("big", [False, True])
def test_glu_envelope(dtype, act, big):
    _cuda()
    from colossalai_b200 import ops

    rows, I = ((1024, 14336) if dtype != torch.float32 else (1024, 7168)) if big else (333, 1792)
    gu = _rand((rows, 2 * I), dtype, 1.5, seed=9).requires_grad_(True)
    y = ops.glu(gu, act)
    dy = _rand((rows, I), dtype, seed=10)
    (dgu,) = torch.autograd.grad(y, gu, dy)
    _check_glu(f"rows={rows}", gu.detach(), y, dy, dgu, act, dtype)


@pytest.mark.gpu
@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16])
@pytest.mark.parametrize("act", ["silu", "gelu"])
def test_glu_valid_rows_envelope(dtype, act):
    """`valid_rows` at 0, mid-way and `rows`: the computed rows match float64; the input is never written."""
    _cuda()
    from colossalai_b200 import ops

    rows, I = 777, 1024
    gu = _rand((rows, 2 * I), dtype, seed=11)
    keep = gu.clone()
    dy = _rand((rows, I), dtype, seed=12)
    for lim in (0, 389, rows):
        x = gu.clone().requires_grad_(True)
        y = ops.glu(x, act, valid_rows=torch.tensor(lim, device="cuda"))
        (dgu,) = torch.autograd.grad(y, x, dy)
        assert torch.equal(x.detach(), keep)
        _check_glu(f"limit={lim}", keep[:lim], y[:lim], dy[:lim], dgu[:lim], act, dtype)


# bias-act: items = rows * H / VEC.  2048 x 8192 bf16 = 2.10M items = 3.9 trips; fp32 = 4.19M items = 7.8 trips.
@pytest.mark.gpu
@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("act", ["silu", "gelu_tanh", "gelu"])
@pytest.mark.parametrize("with_bias", [False, True])
def test_bias_act_envelope(dtype, act, with_bias):
    _cuda()
    from colossalai_b200 import ops

    rows, H = 2048, 8192
    x = _rand((rows, H), dtype, 1.5, seed=13).requires_grad_(True)
    b = _rand((H,), dtype, 0.5, seed=14).requires_grad_(True) if with_bias else None
    y = ops.bias_act(x, b, act)
    dy = _rand((rows, H), dtype, seed=15)
    grads = torch.autograd.grad(y, (x, b) if with_bias else (x,), dy)
    for r in range(0, rows, 256):
        h64 = x[r:r + 256].detach().double() + (b.detach().double() if with_bias else 0.0)
        # the kernel adds the bias in fp32: one rounding of h, carried through act
        err = _act_err(h64) + (U * h64.abs() * _act_grad64(h64, act).abs() if with_bias else 0)
        check(f"bias_act_fwd_{act}", y[r:r + 256], _act64(h64, act), dtype, floor=err)
        dy64 = dy[r:r + 256].double()
        check(f"bias_act_bwd_{act}", grads[0][r:r + 256], dy64 * _act_grad64(h64, act), dtype,
              floor=dy64.abs() * _act_err(h64) * 2)
    if with_bias:
        # db = dx.sum(0) of the kernel's (rounded) dx
        dx_got = grads[0].double()
        check(f"bias_act_db_{act}", grads[1], dx_got.sum(0), dtype, floor=(rows + 2) * U * dx_got.abs().sum(0))


# ============================================================================================ RoPE
# items = tokens * (n_q + n_kv) * (rot_dim / 2 / VEC).  20480 tokens x 10 heads x 8 (bf16, rot 128) = 1.64M items,
# 3.0 trips of the 540,672-item grid; fp32 (VEC 4) 3.28M items, 6.1 trips.
@pytest.mark.gpu
@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("interleaved", [False, True])
@pytest.mark.parametrize("D,rot,T", [(64, 64, 300), (128, 128, 300), (256, 256, 300), (128, 64, 300),
                                     (128, 128, 20480)])
def test_rope_envelope(dtype, interleaved, D, rot, T):
    _cuda()
    from colossalai_b200 import ops

    hq, hkv, max_pos = 8, 2, 4096
    qkv = _rand((T, (hq + 2 * hkv) * D), dtype, seed=16).requires_grad_(True)
    pos = torch.randint(0, max_pos, (T,), device="cuda", generator=torch.Generator(device="cuda").manual_seed(17))
    pos[0], pos[1] = 0, max_pos - 1
    cos, sin = ops.build_rope_cache(max_pos, rot, 10000.0, device="cuda")
    out = ops.rope_qkv(qkv, pos, cos, sin, hq, hkv, D, rot_dim=rot, interleaved=interleaved)

    def rotate(t64, p, sign):
        x = t64.view(len(p), hq + 2 * hkv, D)
        c = cos.double()[p][:, None]
        s = sin.double()[p][:, None] * sign
        qk = x[:, : hq + hkv, :rot]
        if interleaved:
            x1, x2 = qk[..., 0::2], qk[..., 1::2]
            r = torch.stack([x1 * c - x2 * s, x2 * c + x1 * s], -1).flatten(-2)
            mag = torch.stack([x1.abs() * c.abs() + x2.abs() * s.abs()] * 2, -1).flatten(-2)
        else:
            x1, x2 = qk[..., : rot // 2], qk[..., rot // 2:]
            r = torch.cat([x1 * c - x2 * s, x2 * c + x1 * s], -1)
            a = x1.abs() * c.abs() + x2.abs() * s.abs()
            mag = torch.cat([a, x2.abs() * c.abs() + x1.abs() * s.abs()], -1)
        o = x.clone()
        o[:, : hq + hkv, :rot] = r
        fl = torch.zeros_like(x)
        fl[:, : hq + hkv, :rot] = 3 * U * mag                          # two products and a sum in fp32
        return o.view(len(p), -1), fl.view(len(p), -1)

    dy = _rand(out.shape, dtype, seed=18)
    (dq,) = torch.autograd.grad(out, qkv, dy)
    for r in range(0, T, 2048):
        sl = slice(r, r + 2048)
        ref, fl = rotate(qkv[sl].detach().double(), pos[sl], 1.0)
        check(f"rope_fwd D={D} rot={rot} T={T}", out[sl], ref, dtype, floor=fl)
        ref, fl = rotate(dy[sl].double(), pos[sl], -1.0)              # the backward is the inverse rotation
        check(f"rope_bwd D={D} rot={rot} T={T}", dq[sl], ref, dtype, floor=fl)


# ============================================================================================ fp8 cast
# Per-tensor kernels: 512 threads, VEC elements per thread per trip (8 for 16-bit, 4 for fp32); grid_for caps at
# 1056 CTAs = 4.33M (16-bit) / 2.16M (fp32) elements per trip.  257 x 1001 = 257,257 elements leaves a scalar tail
# of 1 (mod 8 and mod 4); 2049 x 4097 = 8,394,753 elements takes 2 (16-bit) / 4 (fp32) trips and also has a tail
# of 1.  Dequant: 4 bytes per thread, 1056 x 2048 = 2.16M bytes per trip (4 trips at 8.39M); per-row scales with
# cols = 1001 or 4097 (cols % 4 = 1) take the scalar path, with cols = 1000 or 72 the 4-byte path.
_FP8 = {"e4m3": (torch.float8_e4m3fn, 448.0, 2.0 ** -3, 2.0 ** -9), "e5m2": (torch.float8_e5m2, 57344.0, 2.0 ** -2,
                                                                                2.0 ** -16)}


@pytest.mark.gpu
@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("fmt", ["e4m3", "e5m2"])
@pytest.mark.parametrize("per_row", [False, True])
@pytest.mark.parametrize("shape,zero", [((257, 1001), None), ((2049, 4097), None), ((64, 1000), "row"),
                                        ((33, 72), "all")])
def test_fp8_cast_envelope(dtype, fmt, per_row, shape, zero):
    _cuda()
    from colossalai_b200.quantization import cast_from_fp8, cast_to_fp8

    f8, fmax, spacing, sub = _FP8[fmt]
    x = _rand(shape, dtype, 4.0, seed=19)
    if zero == "row":
        x[5] = 0
    elif zero == "all":
        x.zero_()
    q, sinv = cast_to_fp8(x, fmt, per_channel_scale=per_row)
    x32 = x.float()
    amax = (x32.abs().amax(-1) if per_row else x32.abs().amax().reshape(1))
    amax = torch.where(amax > 0, amax, torch.ones_like(amax))
    s_ref = amax / fmax                                                # fp32, correctly rounded
    got_s = sinv.reshape(-1)
    # the kernels divide with --use_fast_math's approximate division: at most 2 ulp from the rounded quotient
    ulps = (got_s.view(torch.int32) - s_ref.view(torch.int32)).abs().max().item()
    assert ulps <= 2, f"scale_inv is {ulps} ulp from amax / fp8_max"
    scale = fmax / amax
    q_ref = ((scale[:, None] if per_row else scale) * x32).clamp(-fmax, fmax).to(f8)
    mism = (q.view(torch.uint8) != q_ref.view(torch.uint8)).float().mean().item()
    assert mism < 2e-3, mism
    if zero == "all":
        assert (q.view(torch.uint8) == 0).all()
    # dequant: exactly q * scale_inv, rounded once to `dtype`
    back = cast_from_fp8(q, sinv, dtype, per_channel_scale=per_row)
    s64 = got_s.double()
    q64 = q.double() * (s64[:, None] if per_row else s64)
    check(f"fp8_dequant_{fmt}", back, q64, dtype)
    # round trip: within one fp8 step of x (relative spacing, or the subnormal step, in scaled units)
    step = (x.double().abs() * spacing).clamp_min(sub * (s64[:, None] if per_row else s64))
    assert ((back.double() - x.double()).abs() <= step + ulp_out(x.double(), dtype) * 2).all()


# ============================================================================================ misaligned inputs
def _offset_view(shape, dtype, seed, elems=1):
    """A contiguous tensor that starts `elems` elements into a fresh buffer (2 bytes in for 16-bit dtypes)."""
    n = math.prod(shape)
    buf = torch.empty(n + elems, dtype=dtype, device="cuda")
    v = buf[elems:].view(shape)
    v.copy_(_rand(shape, dtype, seed=seed))
    assert v.is_contiguous() and not is_aligned(v), "the view must be misaligned before any op sees it"
    return v


@pytest.mark.gpu
@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16])
def test_misaligned_views_stay_native_and_exact(dtype):
    """Contiguous views 2 bytes into a buffer go through every native gate: the ops run natively on an aligned copy
    and give bitwise the result of the same op on an aligned tensor."""
    _cuda()
    from colossalai_b200 import ops
    from colossalai_b200.kernel import launch_counter
    from colossalai_b200.ops import cross_entropy as ce

    def same(fn, *views):
        launch_counter.reset()
        a = fn(*views)
        native = launch_counter.count
        b = fn(*[v.clone() for v in views])
        assert native > 0, "a misaligned input left the native path"
        for u, v in zip(a if isinstance(a, tuple) else (a,), b if isinstance(b, tuple) else (b,)):
            assert torch.equal(u, v)

    rows, H = 37, 1024

    def norm_fn(x, w, r, dy):
        x, w, r = (t.detach().requires_grad_(True) for t in (x, w, r))
        y, h = ops.rms_norm(x, w, 1e-5, r)
        return (y, h) + torch.autograd.grad((y, h), (x, w), (dy, dy))

    same(norm_fn, _offset_view((rows, H), dtype, 1), _offset_view((H,), dtype, 2), _offset_view((rows, H), dtype, 3),
         _offset_view((rows, H), dtype, 4))

    def ln_fn(x, w, b, dy):
        x, w, b = (t.detach().requires_grad_(True) for t in (x, w, b))
        y = ops.layer_norm(x, w, b, 1e-5)
        return (y,) + torch.autograd.grad(y, (x, w, b), dy)

    same(ln_fn, _offset_view((rows, H), dtype, 5), _offset_view((H,), dtype, 6), _offset_view((H,), dtype, 7),
         _offset_view((rows, H), dtype, 8))

    def glu_fn(gu, dy):
        gu = gu.detach().requires_grad_(True)
        y = ops.glu(gu, "silu")
        return (y,) + torch.autograd.grad(y, gu, dy)

    same(glu_fn, _offset_view((rows, 2 * H), dtype, 9), _offset_view((rows, H), dtype, 10))

    def bias_fn(x, b, dy):
        x, b = x.detach().requires_grad_(True), b.detach().requires_grad_(True)
        y = ops.bias_act(x, b, "gelu")
        return (y,) + torch.autograd.grad(y, (x, b), dy)

    same(bias_fn, _offset_view((rows, H), dtype, 11), _offset_view((H,), dtype, 12), _offset_view((rows, H), dtype, 13))

    cos, sin = ops.build_rope_cache(512, 128, device="cuda")
    pos = torch.arange(rows, device="cuda")

    def rope_fn(qkv, dy):
        qkv = qkv.detach().requires_grad_(True)
        y = ops.rope_qkv(qkv, pos, cos, sin, 4, 2, 128)
        return (y,) + torch.autograd.grad(y, qkv, dy)

    same(rope_fn, _offset_view((rows, 8 * 128), dtype, 14), _offset_view((rows, 8 * 128), dtype, 15))

    tgt = torch.randint(0, 4000, (rows,), device="cuda")

    def ce_fn(logits):
        m = ce.row_max(logits, 4000)
        s = ce.sumexp_and_target(logits, tgt, m, 0, -100, 4000)
        g = ce.softmax_grad(logits, tgt, m, s[0], None, 0, -100, row_scale=torch.ones(rows, device="cuda"),
                            valid_cols=4000)
        return m, s, g

    same(ce_fn, _offset_view((rows, 4096), dtype, 16))


@pytest.mark.gpu
@pytest.mark.parametrize("dtype", DTYPES)
def test_misaligned_fp8_buffers_stay_native_and_exact(dtype):
    """fp8 casts on offset views: the input, the `out` buffer, and byte slices of a received fp8 buffer."""
    _cuda()
    from colossalai_b200.kernel import launch_counter
    from colossalai_b200.quantization import cast_from_fp8, cast_to_fp8

    n = 4099
    x = _offset_view((n,), dtype, 20)
    q_ref, s_ref = cast_to_fp8(x.clone(), "e4m3")
    launch_counter.reset()
    q, s = cast_to_fp8(x, "e4m3")
    assert launch_counter.by_name.get("fp8_quant_tensor")
    assert torch.equal(q.view(torch.uint8), q_ref.view(torch.uint8)) and torch.equal(s, s_ref)
    out_buf = torch.empty(n + 3, dtype=torch.uint8, device="cuda")
    out = out_buf[3:].view(torch.float8_e4m3fn)
    assert not is_aligned(out, 8)
    q2, _ = cast_to_fp8(x, "e4m3", out=out)
    assert q2.data_ptr() == out.data_ptr() and torch.equal(out.view(torch.uint8), q_ref.view(torch.uint8))
    # a rank's slice of a flat fp8 receive buffer (as the fp8 all-reduce / all-to-all take) starts at any byte
    recv = torch.cat([torch.zeros(1, dtype=torch.uint8, device="cuda"), q_ref.view(torch.uint8)])
    assert is_aligned(recv)
    for off in (1, 2, 3):
        piece = recv[off:].view(torch.float8_e4m3fn)
        assert not is_aligned(piece, 4)
        launch_counter.reset()
        got = cast_from_fp8(piece, s_ref, dtype)
        assert launch_counter.by_name.get("fp8_dequant")
        assert torch.equal(got, cast_from_fp8(piece.clone(), s_ref, dtype))
