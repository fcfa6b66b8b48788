"""The multi-tensor optimizer kernels (`multi_tensor_optim.cu`, `cpu_adam.cpp`) against float64 references.

Every reference is plain float64 arithmetic from the update formulas (`multi_tensor_{adam,sgd,lamb,l2norm,scale}`
and torch's `clip_grad_norm_`), evaluated on the exact values the kernel read.  The scalar hyper-parameters enter
as the fp32 numbers the kernel receives (`f32(lr)`, `f32(1 - beta1 ** step)`, ...), because those are its inputs.
Each step's reference starts from the state the kernel stored on the previous step, so errors do not compound, and
the parameter's reference takes the moments the kernel stored in the same step (they are checked on their own), so
a cancellation in `m` cannot widen the parameter's bound.

Each element is checked against

    |got - ref| <= k * ulp(|ref|) + floor

where `ulp` is the output dtype's spacing at |ref| (never below its subnormal step) and `floor` bounds the fp32
rounding of the arithmetic in front of the final store.  `check` refuses a floor above 1% of the median |ref|, and
elements whose reference is exactly zero with every term zero (floor 0) must be exactly zero.

Bounds (U = 2^-24, the fp32 unit roundoff):
  * m, v: k = 2 plus 4U (6U for v) times the sum of the magnitudes of the terms, which covers cancellation.
  * p: k = 1 plus C * 2^-22 * |lr| * (|m_hat / (sqrt(v_hat) + eps)| + |wd * p|), C = 5.  The kernels are built
    with `--use_fast_math`, so `/` is `div.full.f32` (2 ulp = 2^-22 relative) and `sqrtf` is the approximate
    square root (budgeted at 3 ulp = 1.5 * 2^-22).  In units of 2^-22: m / bc1 (1) + v / bc2 halved by the sqrt
    (0.5) + sqrt (1.5) + the eps add (0.25) + the final division (1) + the weight-decay add (0.25) + lr * upd
    (0.25) = 4.75 <= C.  The fp32 store of p adds at most half an ulp of p, inside k = 1.
  * bf16/fp16 params (the generic path): one output ulp plus the same floor.
  * a low-precision copy next to an fp32 master must be bitwise `p_stored.to(lp.dtype)`.
"""
import math

import numpy as np
import pytest
import torch

U = 2.0 ** -24
C_DIV = 5.0                                                        # see the module docstring
CHUNK = 2048 * 16                                                  # elements per CTA work item
F32, BF16, F16 = torch.float32, torch.bfloat16, torch.float16
_MANT = {BF16: 8, F16: 11, F32: 24}
_MIN_STEP = {BF16: 2.0 ** -133, F16: 2.0 ** -24, F32: 2.0 ** -149}
_WORST = {}                                                        # kernel -> largest |err| / tol seen


def ulp(ref: torch.Tensor, dtype: torch.dtype) -> torch.Tensor:
    """Spacing of `dtype` at |ref|: |ref| = f * 2^e with f in [0.5, 1) has spacing 2^(e - mantissa bits)."""
    a = ref.abs().double()
    _, e = torch.frexp(a)
    return torch.ldexp(torch.ones_like(a), e - _MANT[dtype]).clamp_min(_MIN_STEP[dtype])


def check(what, got, ref, dtype, k=1.0, floor=0.0):
    """Assert |got - ref| <= k * ulp(|ref|) + floor elementwise (see the module docstring)."""
    got, ref = got.double().flatten(), ref.double().flatten()
    assert got.shape == ref.shape, (what, got.shape, ref.shape)
    assert torch.isfinite(ref).all(), f"{what}: non-finite reference"
    floor = torch.as_tensor(floor, dtype=torch.float64, device=ref.device).flatten().expand_as(ref)
    # a zero whose terms are all zero (floor 0) must stay exactly zero; a zero reached by cancelling non-zero
    # terms is bounded by the floor like any other value
    zero = (ref == 0) & (floor == 0)
    nz_zero = int((got[zero] != 0).sum())
    assert nz_zero == 0, f"{what}: {nz_zero} elements whose reference is exactly 0 are not 0"
    nz = ~zero
    if not nz.any():
        return
    med = ref[nz].abs().median()
    assert floor[nz].median() <= 0.01 * med, f"{what}: floor {floor[nz].median():.3g} > 1% of median |ref| {med:.3g}"
    tol = k * ulp(ref, dtype) + floor
    err = (got - ref).abs()
    bad = nz & ~(err <= tol)                    # NaN in `got` counts as bad
    if bad.any():
        i = int(bad.nonzero()[0])
        raise AssertionError(f"{what}: {int(bad.sum())} of {int(nz.sum())} elements out of tolerance; first at flat "
                             f"index {i}: got {got[i].item():.9g} ref {ref[i].item():.9g} tol {tol[i].item():.3g}")
    ratio = float((err[nz] / tol[nz]).max())
    name = what.split(" ")[0]
    _WORST[name] = max(_WORST.get(name, 0.0), ratio)


def check_bitwise(what, got, want):
    assert got.dtype == want.dtype and got.shape == want.shape, what
    iv = {F32: torch.int32, BF16: torch.int16, F16: torch.int16}[got.dtype]
    diff = got.reshape(-1).view(iv) != want.reshape(-1).view(iv)
    assert not diff.any(), f"{what}: {int(diff.sum())} of {diff.numel()} elements differ bitwise, first at " \
                           f"{int(diff.nonzero()[0])}"


@pytest.fixture(scope="module", autouse=True)
def _report_worst():
    yield
    if _WORST:
        print("\nlargest error-to-tolerance ratio per kernel:")
        for k, v in sorted(_WORST.items()):
            print(f"  {k:<24} {v:.3f}")
        if torch.cuda.is_available():
            print(f"peak CUDA memory allocated: {torch.cuda.max_memory_allocated() / 2**30:.2f} GiB")


def f32(x: float) -> float:
    return float(np.float32(x))


def _cuda():
    if not torch.cuda.is_available():
        pytest.skip("needs a GPU")
    return torch.device("cuda")


def _flat(ts):
    return torch.cat([t.detach().reshape(-1).double() for t in ts]) if ts else torch.zeros(0, dtype=torch.float64)


# ============================================================================================ Adam reference
class AdamScalars:
    """The fp32 scalars an Adam kernel computes with.  `cpu=True` mirrors `cpu_adam.cpp`, which forms the bias
    corrections in float from the fp32 betas (`1 - powf(beta, step)`, as the reference CPU Adam does)."""

    def __init__(self, lr, beta1, beta2, eps, wd, step, adamw, bias_correction=True, s=1.0, cpu=False):
        self.lr, self.eps, self.wd, self.adamw, self.s = f32(lr), f32(eps), f32(wd), adamw, s
        self.b1, self.b2 = f32(beta1), f32(beta2)
        self.ob1, self.ob2 = 1.0 - self.b1, 1.0 - self.b2          # exact in fp32 (Sterbenz)
        if not bias_correction:
            self.bc1 = self.bc2 = 1.0
        elif cpu:
            one, st = np.float32(1), np.float32(step)
            self.bc1 = float(one - np.power(np.float32(beta1), st))
            self.bc2 = float(one - np.power(np.float32(beta2), st))
        else:
            self.bc1, self.bc2 = f32(1.0 - beta1 ** step), f32(1.0 - beta2 ** step)


def adam_moments(p, g, m, v, S):
    """float64 m', v' and their floors from the values the kernel read."""
    gs = g * S.s
    gg = gs if S.adamw else gs + S.wd * p
    gmag = gs.abs() if S.adamw else gs.abs() + (S.wd * p).abs()
    m1 = S.b1 * m + S.ob1 * gg
    v1 = S.b2 * v + S.ob2 * gg * gg
    return m1, v1, 4 * U * (S.b1 * m.abs() + S.ob1 * gmag), 6 * U * (S.b2 * v + S.ob2 * gmag * gmag)


def adam_param(p, m1, v1, S, eps_inside=False):
    """float64 p' from the stored m', v' and its floor."""
    den = (v1 / S.bc2 + S.eps).sqrt() if eps_inside else (v1 / S.bc2).sqrt() + S.eps
    a = (m1 / S.bc1) / den
    wdp = S.wd * p
    upd = a + wdp if S.adamw else a
    mag = S.lr * (a.abs() + (wdp.abs() if S.adamw else 0.0))
    return p - S.lr * upd, C_DIV * 2.0 ** -22 * mag


def check_adam(name, before, p1, m1g, v1g, S, lp=None):
    """before = (p, g, m, v) as read by the kernel; p1/m1g/v1g/lp = what it stored (lists or tensors)."""
    p0, g0, m0, v0 = (_flat(x) if isinstance(x, (list, tuple)) else x.double().flatten() for x in before)
    pl = p1 if isinstance(p1, (list, tuple)) else [p1]
    p_dtype = pl[0].dtype
    mg = _flat(m1g) if isinstance(m1g, (list, tuple)) else m1g.double().flatten()
    vg = _flat(v1g) if isinstance(v1g, (list, tuple)) else v1g.double().flatten()
    m1, v1, fm, fv = adam_moments(p0, g0, m0, v0, S)
    check(f"{name}.m", mg, m1, F32, k=2, floor=fm)
    check(f"{name}.v", vg, v1, F32, k=2, floor=fv)
    pref, fp = adam_param(p0, mg, vg, S)
    check(f"{name}.p", _flat(pl), pref, p_dtype, k=1, floor=fp)
    if lp is not None:
        lps = lp if isinstance(lp, (list, tuple)) else [lp]
        for i, (pi, li) in enumerate(zip(pl, lps)):
            if li is None:
                continue
            if pi.dtype == F32:
                check_bitwise(f"{name}.lp[{i}]", li, pi.to(li.dtype))
        lp_idx = [i for i, li in enumerate(lps) if li is not None and pl[i].dtype != F32]
        if lp_idx:                                                  # low-precision copy of a low-precision param
            offs = np.cumsum([0] + [t.numel() for t in pl])
            sel = torch.cat([torch.arange(int(offs[i]), int(offs[i + 1])) for i in lp_idx]).to(pref.device)
            check(f"{name}.lp", _flat([lps[i] for i in lp_idx]), pref[sel], lps[lp_idx[0]].dtype, k=1,
                  floor=fp[sel])


# ============================================================================================ comparator (CPU)
def _emulate_adam(p, g, m, v, S, *, lr_scale=1.0, no_bc=False, eps_inside=False, swap_wd=False):
    """A float64 Adam kernel rounded once to fp32, with one optional mistake."""
    class _S:
        pass
    T = _S()
    T.__dict__.update(S.__dict__)
    T.lr = S.lr * lr_scale
    if no_bc:
        T.bc1 = T.bc2 = 1.0
    if swap_wd:
        T.adamw = not S.adamw
    m1, v1, _, _ = adam_moments(p, g, m, v, T)
    m1, v1 = m1.float(), v1.float()
    p1, _ = adam_param(p, m1.double(), v1.double(), T, eps_inside=eps_inside)
    return p1.float(), m1, v1


def test_comparator_rejects_adam_corruptions():
    """Each mistake a broken Adam kernel could make is rejected; the float64 reference rounded once is accepted."""
    gen = torch.Generator().manual_seed(0)
    n = 3 * CHUNK + 5
    p = (torch.randn(n, generator=gen) * 0.5).float().double()
    p[:64] = 0.0                                                    # a zero parameter stretch
    g = torch.randn(n, generator=gen, dtype=torch.float64) * 64
    m = (torch.randn(n, generator=gen) * 0.05).float().double()
    v = (m * m + torch.rand(n, generator=gen, dtype=torch.float64) * 0.01).float().double()
    tiny = torch.arange(0, n, 7)                                    # gradients and moments near eps
    g[tiny] = torch.randn(len(tiny), generator=gen, dtype=torch.float64) * 64e-8
    m[tiny] = (torch.randn(len(tiny), generator=gen) * 1e-9).float().double()
    v[tiny] = ((torch.randn(len(tiny), generator=gen) * 1e-8) ** 2).float().double()
    g = g.float().double()
    div_scale, clip = 64.0, f32(0.37)
    s = f32(f32(1.0 / div_scale) * clip)
    S = AdamScalars(0.05, 0.9, 0.999, 1e-8, 0.1, 3, True, s=s)
    lp0 = p.float().to(BF16)

    def run(p1, m1, v1, lp):
        check_adam("selftest", (p, g, m, v), p1, m1, v1, S, lp=[lp])

    p1, m1, v1 = _emulate_adam(p, g, m, v, S)
    run(p1, m1, v1, p1.to(BF16))

    def rejected(p1, m1, v1, lp=None):
        with pytest.raises(AssertionError):
            run(p1, m1, v1, p1.to(BF16) if lp is None else lp)

    rejected(*_emulate_adam(p, g, m, v, S, lr_scale=1.001))                        # lr off by 0.1%
    rejected(*_emulate_adam(p, g, m, v, S, no_bc=True))                            # bias correction dropped
    rejected(*_emulate_adam(p, g, m, v, S, eps_inside=True))                       # sqrt(v_hat + eps)
    rejected(*_emulate_adam(p, g, m, v, S, swap_wd=True))                          # coupled <-> decoupled decay
    rejected(*_emulate_adam(p, g * div_scale, m, v, S))                            # inv_scale ignored
    rejected(*_emulate_adam(p, g * clip, m, v, S))                                 # clip coefficient applied twice
    q1, qm, qv = (t.clone() for t in (p1, m1, v1))                                 # one chunk left unstepped
    q1[CHUNK:2 * CHUNK], qm[CHUNK:2 * CHUNK], qv[CHUNK:2 * CHUNK] = (t[CHUNK:2 * CHUNK].float()
                                                                      for t in (p, m, v))
    rejected(q1, qm, qv)
    lp = p1.to(BF16)                                                               # the lp tail left unwritten
    lp[-3:] = lp0[-3:]
    rejected(p1, m1, v1, lp)
    z = torch.tensor([0.0, 1.0, 2.0], dtype=torch.float64)                        # an all-zero-term element
    with pytest.raises(AssertionError, match="exactly 0"):
        check("selftest zero", z + torch.tensor([2.0 ** -149, 0, 0], dtype=torch.float64), z, F32)
    with pytest.raises(AssertionError, match="floor"):                            # a swamping floor is refused
        check("selftest floor", p1, p, F32, floor=p.abs().median() * 0.02)


def test_ulp_is_the_dtype_spacing():
    x = torch.tensor([1.0, 1.5, 2.0, 3.0, 0.75, 1e-30], dtype=torch.float64)
    assert ulp(x, F32).tolist()[:5] == [2.0 ** -23, 2.0 ** -23, 2.0 ** -22, 2.0 ** -22, 2.0 ** -24]
    assert ulp(x, BF16).tolist()[:3] == [2.0 ** -7, 2.0 ** -7, 2.0 ** -6]
    assert ulp(x, F16)[-1].item() == 2.0 ** -24                      # clamped at the subnormal step
    a = torch.tensor([1.0, 1.7, 100.0, 0.3, 3e-39])                  # adjacent fp32 numbers (last: subnormal)
    b = torch.nextafter(a, torch.full_like(a, 1e9))
    assert torch.equal(b.double() - a.double(), ulp(a.double(), F32))


# ============================================================================================ CPU Adam (CPU)
CPU_SIZES = [1, 3, 4, 8191, 8192, 8193, 3 * 8192 + 6]               # 8192-element OpenMP blocks, tails 1, 2, 3


@pytest.mark.parametrize("adamw", [True, False])
@pytest.mark.parametrize("p_dtype,g_dtype,lp_dtype", [(F32, F32, None), (F32, BF16, BF16), (F32, F32, F16),
                                                      (F32, F16, None), (BF16, BF16, None), (F16, F16, None),
                                                      (F16, F32, BF16), (BF16, F32, F16)])
def test_cpu_adam_envelope(adamw, p_dtype, g_dtype, lp_dtype):
    from colossalai_b200.nn.optimizer.cpu_adam import cpu_adam_step

    gen = torch.Generator().manual_seed(1)
    div_scale = 8.0
    for n in CPU_SIZES:
        p = (torch.randn(n, generator=gen) * 0.5).to(p_dtype)
        if n == 8193:
            p.zero_()
        m, v = torch.zeros(n), torch.zeros(n)
        lp = torch.zeros(n, dtype=lp_dtype) if lp_dtype is not None else None
        for step in range(1, 4):
            g = torch.randn(n, generator=gen) * div_scale
            g[::5] *= 1e-8                                          # gradients near eps
            g = g.to(g_dtype)
            before = (p.double(), g.double(), m.double(), v.double())
            S = AdamScalars(0.05, 0.9, 0.999, 1e-8, 0.1, step, adamw, s=f32(1 / div_scale), cpu=True)
            cpu_adam_step(p, g, m, v, 0.05, 0.9, 0.999, 1e-8, 0.1, step, True, adamw, 1 / div_scale, lp=lp)
            check_adam(f"cpu_adam n={n} step={step}", before, p, m, v, S, lp=[lp] if lp is not None else None)


# ============================================================================================ fallbacks (CPU)
def _lamb_moments(p, g, m, v, S, b3):
    """float64 LAMB stage-1 moments and their floors (beta3 = 1 - beta1 with grad averaging, else 1)."""
    gs = g * S.s
    gg = gs if S.adamw else gs + S.wd * p
    gmag = gs.abs() if S.adamw else gs.abs() + (S.wd * p).abs()
    m1 = S.b1 * m + b3 * gg
    v1 = S.b2 * v + S.ob2 * gg * gg
    return m1, v1, 4 * U * (S.b1 * m.abs() + b3 * gmag), 6 * U * (S.b2 * v + S.ob2 * gmag * gmag)


def _lamb_update(p, m1, v1, S):
    a = (m1 / S.bc1) / ((v1 / S.bc2).sqrt() + S.eps)
    wdp = S.wd * p
    u = a + wdp if S.adamw else a
    return u, C_DIV * 2.0 ** -22 * (a.abs() + (wdp.abs() if S.adamw else 0.0))


def _run_lamb_case(device, dtype, adam_w_mode=True, grad_averaging=True, bias_correction=True, wd=0.01,
                   use_nvlamb=False, max_norm=1.0, steps=2):
    from colossalai_b200.nn.optimizer import FusedLAMB
    from colossalai_b200.ops import multi_tensor as mt
    from colossalai_b200.ops._dispatch import use_native

    gen = torch.Generator().manual_seed(3)
    sizes = [CHUNK + 1, 100, 4097, 64]                 # [1] is an all-zero parameter, [3] gets all-zero grads
    ps = []
    for i, n in enumerate(sizes):
        t = (torch.randn(n, generator=gen) * 0.5).to(dtype)
        if i == 1:
            t.zero_()
        ps.append(torch.nn.Parameter(t.to(device)))
    lr, b1, b2, eps = 0.05, 0.9, 0.999, 1e-6
    opt = FusedLAMB(ps, lr=lr, betas=(b1, b2), eps=eps, weight_decay=wd, adam_w_mode=adam_w_mode,
                    grad_averaging=grad_averaging, bias_correction=bias_correction, max_grad_norm=max_norm,
                    use_nvlamb=use_nvlamb)
    native = use_native(ps[0])
    tag = f"lamb{'' if native else '_fallback'}"
    for step in range(1, steps + 1):
        for i, p in enumerate(ps):
            g = torch.randn(p.numel(), generator=gen) * (0.0 if i == 3 else 1.0)
            p.grad = g.to(dtype).to(device)
        grads = [p.grad for p in ps]
        g0 = [g.detach().double().clone() for g in grads]
        p0 = [p.detach().double().clone() for p in ps]
        m0 = [opt.state[p]["exp_avg"].double().clone() if p in opt.state else torch.zeros_like(q)
              for p, q in zip(ps, p0)]
        v0 = [opt.state[p]["exp_avg_sq"].double().clone() if p in opt.state else torch.zeros_like(q)
              for p, q in zip(ps, p0)]
        # global grad-norm clip: the kernel's norm, checked against float64, then the clip exactly as FusedLAMB
        # forms it (torch: clip_grad_norm_ divides by the clip factor max(1, ||g|| / max_norm))
        n64 = math.sqrt(sum(float((g * g).sum()) for g in g0))
        if native:
            gn = mt.norm_sq(mt.TensorTable(grads, grads), "grad")[0].sqrt()
            depth = 40 + math.ceil(sum(math.ceil(n / CHUNK) for n in sizes) / 1024)
            assert abs(gn.item() - n64) <= (depth * U + 2 * U) * n64, (gn.item(), n64)
        else:
            gn = torch.stack([g.float().pow(2).sum() for g in grads]).sum().sqrt()
        clip = (gn / max_norm).clamp(min=1.0)
        binds = n64 / max_norm > 1.0
        assert bool(clip.item() > 1.0) == binds
        s = f32(1.0 / clip.item())
        opt.step()
        S = AdamScalars(lr, b1, b2, eps, wd, step, adam_w_mode, bias_correction, s=s)
        if not native:
            S.ob2 = f32(1.0 - b2)                 # torch's addcmul_ takes 1 - beta2 formed in double
        b3 = f32(1.0 - b1) if grad_averaging else 1.0
        trust = use_nvlamb or wd != 0
        p0f, g0f, m0f, v0f = (_flat(x) for x in (p0, g0, m0, v0))
        m1, v1, fm, fv = _lamb_moments(p0f, g0f, m0f, v0f, S, b3)
        mg = _flat([opt.state[p]["exp_avg"] for p in ps])
        vg = _flat([opt.state[p]["exp_avg_sq"] for p in ps])
        case = f"step={step}"
        check(f"{tag}.m {case}", mg, m1, F32, k=2, floor=fm)
        check(f"{tag}.v {case}", vg, v1, F32, k=2, floor=fv)
        u_ref, fu = _lamb_update(p0f, mg, vg, S)
        if native:                        # stage 1 wrote u, rounded to the grad dtype, into the grad slot
            u_used = _flat(grads)
            check(f"{tag}.u {case}", u_used, u_ref, dtype, k=1, floor=fu)
        else:
            u_used = u_ref
        offs = np.cumsum([0] + sizes)
        want, floor = [], []
        for i in range(len(sizes)):
            sl = slice(int(offs[i]), int(offs[i + 1]))
            ratio, er = 1.0, 0.0
            if trust:
                pn, un = float(p0f[sl].norm()), float(u_used[sl].norm())
                if pn > 0 and un > 0:
                    ratio = pn / un
                    # per-tensor fp32 sums (depth 40 + one chunk per finalize thread), two sqrt, one division
                    er = (2 * 40 + 2) * U / 2 + 4 * 2.0 ** -22 + (0 if native else 64 * U)
            step_i = S.lr * ratio * u_used[sl]
            want.append(p0f[sl] - step_i)
            extra = 0.0 if native else S.lr * ratio * fu[sl]          # the fallback never rounds u
            floor.append((er + 2 * U) * step_i.abs() + extra)
        check(f"{tag}.p {case} trust={trust}", _flat(ps), torch.cat(want), dtype, k=1, floor=torch.cat(floor))


@pytest.mark.parametrize("wd,use_nvlamb", [(0.0, False), (0.0, True), (0.01, False)])
def test_fused_lamb_fallback_trust_ratio(wd, use_nvlamb):
    """The trust ratio applies only with `use_nvlamb` or a non-zero weight decay (CPU tier)."""
    _run_lamb_case("cpu", F32, wd=wd, use_nvlamb=use_nvlamb)


def _noncontiguous_adam(device):
    from colossalai_b200.nn.optimizer import FusedAdam

    gen = torch.Generator().manual_seed(4)
    w = torch.nn.Parameter((torch.randn(64, 32, generator=gen) * 0.5).to(device).t())
    b = torch.nn.Parameter((torch.randn(40, generator=gen) * 0.5).to(device))
    assert not w.is_contiguous()
    opt = FusedAdam([w, b], lr=0.05, weight_decay=0.1)
    for step in range(1, 4):
        w.grad = (torch.randn(32, 64, generator=gen) * 4).to(device)
        b.grad = (torch.randn(40, generator=gen) * 4).to(device)
        before = [t.detach().double().clone() for t in (w, b)]
        opt.step(div_scale=4.0)
        S = AdamScalars(0.05, 0.9, 0.999, 1e-8, 0.1, step, True)
        for name, p, p0 in (("w", w, before[0]), ("b", b, before[1])):
            st = opt.state[p]
            # the moments are contiguous; the parameter keeps its own (transposed) layout
            mg, vg = st["exp_avg"].double(), st["exp_avg_sq"].double()
            want, fp = adam_param(p0, mg, vg, S)
            check(f"fused_adam.p {name} step={step}", p.detach(), want, F32, k=1, floor=fp)
        opt.zero_grad()


def test_fused_adam_steps_noncontiguous_param_cpu():
    _noncontiguous_adam("cpu")


@pytest.mark.gpu
def test_fused_adam_steps_noncontiguous_param_gpu():
    _noncontiguous_adam(_cuda())


def test_cpu_adam_lp_rounds_ties_to_even():
    """With lr = 0 the parameter is unchanged, so the fp16/bf16 copy is the plain conversion of p: exact halfway
    cases (normal and subnormal fp16) must round to even, as `Tensor.to` does."""
    from colossalai_b200.nn.optimizer.cpu_adam import cpu_adam_step

    base = torch.tensor([1.0, 1.0 + 2.0 ** -10, 2.0 ** -14, 2.0 ** -20, 3.0 * 2.0 ** -24, 1000.0, 65504.0])
    half_ulp = torch.tensor([2.0 ** -11, 2.0 ** -11, 2.0 ** -25, 2.0 ** -25, 2.0 ** -25, 2.0 ** -2, 16.0])
    ties = torch.cat([base + half_ulp, -(base + half_ulp), base + 0.999 * half_ulp])   # last: just below a tie
    for lp_dtype in (F16, BF16):
        p = ties.clone()
        lp = torch.zeros_like(p, dtype=lp_dtype)
        cpu_adam_step(p, torch.ones_like(p), torch.zeros_like(p), torch.zeros_like(p), 0.0, 0.9, 0.999, 1e-8, 0.0,
                      1, True, True, lp=lp)
        assert torch.equal(p, ties)
        check_bitwise(f"cpu_adam lp ties {lp_dtype}", lp, ties.to(lp_dtype))


# ============================================================================================ Adam (GPU)
ADAM_SIZES = [1, 3, 4, 0, 32767, 32768, 32769, 32770, 5 * CHUNK + 7, 6, 4097]    # chunk tails = 1, 2, 3 (mod 4)
ZERO_P = 10                                                          # this tensor starts at p = 0


def _adam_problem(dev, sizes, p_dtype, g_dtype, lp_dtype, seed, offset=0):
    """Params, moments and lp copies.  offset > 0 places p, m and v `offset` elements into flat arenas, so they are
    4-12 bytes off a 16-byte boundary (the generic path)."""
    gen = torch.Generator(device=dev).manual_seed(seed)
    tot = sum(sizes) + 8 * len(sizes) + 8

    def arena(dtype):
        return torch.zeros(tot, dtype=dtype, device=dev)

    ap, am, av = arena(p_dtype), arena(F32), arena(F32)
    ps, ms, vs, lps = [], [], [], []
    o = offset
    for i, n in enumerate(sizes):
        p, m, v = ap[o:o + n], am[o:o + n], av[o:o + n]
        o += n + 4 + (-n) % 4                                         # keeps o = offset (mod 4)
        p.copy_((torch.randn(n, device=dev, generator=gen) * 0.5).to(p_dtype))
        if i == ZERO_P:
            p.zero_()
        ps.append(p)
        ms.append(m)
        vs.append(v)
        lps.append(p.to(lp_dtype) if lp_dtype is not None else None)
    if offset == 0:                                                   # separate, 16-byte aligned allocations
        ps = [p.clone() for p in ps]
        ms = [torch.zeros_like(m) for m in ms]
        vs = [torch.zeros_like(v) for v in vs]
    return ps, ms, vs, lps, gen


def _adam_grads(ps, g_dtype, gen, scale):
    gs = []
    for p in ps:
        g = torch.randn(p.numel(), device=p.device, generator=gen) * scale
        g[::5] *= 1e-8                                               # gradients near eps
        gs.append(g.to(g_dtype))
    return gs


def _run_adam(name, sizes, p_dtype, g_dtype, lp_dtype, adamw, offset=0, steps=3, seed=0):
    from colossalai_b200.ops import multi_tensor as mt

    dev = _cuda()
    ps, ms, vs, lps, gen = _adam_problem(dev, sizes, p_dtype, g_dtype, lp_dtype, seed, offset)
    div_scale = 8.0
    for step in range(1, steps + 1):
        gs = _adam_grads(ps, g_dtype, gen, div_scale)
        before = [_flat(x) for x in (ps, gs, ms, vs)]
        mt.adam(mt.TensorTable(ps, gs, ms, vs, lps), 0.05, 0.9, 0.999, 1e-8, 0.1, step, adamw,
                inv_scale=1.0 / div_scale)
        S = AdamScalars(0.05, 0.9, 0.999, 1e-8, 0.1, step, adamw, s=f32(1.0 / div_scale))
        check_adam(f"{name} step={step}", before, ps, ms, vs, S, lp=lps if lp_dtype is not None else None)


@pytest.mark.gpu
@pytest.mark.parametrize("adamw", [True, False])
@pytest.mark.parametrize("lp_dtype", [None, BF16, F16], ids=["nolp", "lpbf16", "lpfp16"])
@pytest.mark.parametrize("g_dtype", [F32, BF16, F16], ids=["gf32", "gbf16", "gfp16"])
def test_adam_dispatch_branches(g_dtype, lp_dtype, adamw):
    """fp32 params at 16-byte aligned addresses: every (grad, lp) pair of `multi_tensor_adam_kernel`, vectorised
    where a template instance exists (bf16->bf16, f32->bf16/f16, f16->f16, no lp) and generic otherwise."""
    _run_adam("adam", ADAM_SIZES, F32, g_dtype, lp_dtype, adamw)


@pytest.mark.gpu
@pytest.mark.parametrize("p_dtype,g_dtype,lp_dtype", [(BF16, BF16, None), (F16, F16, None), (BF16, F32, F16),
                                                      (F16, F32, BF16), (BF16, BF16, BF16)])
def test_adam_low_precision_params(p_dtype, g_dtype, lp_dtype):
    _run_adam("adam_generic", ADAM_SIZES, p_dtype, g_dtype, lp_dtype, True)


@pytest.mark.gpu
@pytest.mark.parametrize("offset", [1, 2, 3])
@pytest.mark.parametrize("g_dtype,lp_dtype", [(BF16, BF16), (F32, None)])
def test_adam_misaligned_views(offset, g_dtype, lp_dtype):
    """p, m, v are views 1-3 elements into flat arenas: the alignment test sends them to the generic path."""
    _run_adam("adam_generic", ADAM_SIZES, F32, g_dtype, lp_dtype, False, offset=offset)


@pytest.mark.gpu
def test_adam_three_thousand_tensors():
    """One launch over ~3000 tensors: every CTA binary-searches its tensor in the chunk prefix."""
    gen = torch.Generator().manual_seed(5)
    sizes = [int(x) for x in torch.randint(0, 300, (3000,), generator=gen)]
    for i in range(0, 3000, 97):
        sizes[i] = CHUNK + int(torch.randint(1, 9, (1,), generator=gen))
    _run_adam("adam", sizes, F32, BF16, BF16, True, steps=2, seed=5)


@pytest.mark.gpu
def test_adam_noop_flag_leaves_everything_bitwise():
    from colossalai_b200.ops import multi_tensor as mt

    dev = _cuda()
    ps, ms, vs, lps, gen = _adam_problem(dev, ADAM_SIZES, F32, BF16, BF16, 6)
    for m, v in zip(ms, vs):
        m.normal_(generator=gen)
        v.uniform_(generator=gen)
    gs = _adam_grads(ps, BF16, gen, 1.0)
    snap = [[t.clone() for t in lst] for lst in (ps, ms, vs, lps)]
    flag = torch.ones(1, dtype=torch.int32, device=dev)
    mt.adam(mt.TensorTable(ps, gs, ms, vs, lps), 0.05, 0.9, 0.999, 1e-8, 0.1, 1, True, noop_flag=flag)
    for lst, old in zip((ps, ms, vs, lps), snap):
        for t, o in zip(lst, old):
            check_bitwise("adam noop", t, o)
    flag.zero_()                                                     # and with the flag clear it does step
    mt.adam(mt.TensorTable(ps, gs, ms, vs, lps), 0.05, 0.9, 0.999, 1e-8, 0.1, 1, True, noop_flag=flag)
    assert not torch.equal(ps[-1], snap[0][-1])


@pytest.mark.gpu
def test_adam_device_scale_times_div_scale():
    """`inv_scale_dev` multiplies the host inv_scale in fp32: s = f32(f32(1 / div_scale) * coef)."""
    from colossalai_b200.ops import multi_tensor as mt

    dev = _cuda()
    ps, ms, vs, lps, gen = _adam_problem(dev, ADAM_SIZES, F32, F32, BF16, 7)
    div_scale, coef = 3.0, f32(0.37)
    for step in range(1, 3):
        gs = _adam_grads(ps, F32, gen, div_scale / coef)
        before = [_flat(x) for x in (ps, gs, ms, vs)]
        mt.adam(mt.TensorTable(ps, gs, ms, vs, lps), 0.05, 0.9, 0.999, 1e-8, 0.1, step, False,
                inv_scale=1.0 / div_scale, inv_scale_dev=torch.tensor([coef], device=dev))
        S = AdamScalars(0.05, 0.9, 0.999, 1e-8, 0.1, step, False, s=f32(f32(1.0 / div_scale) * coef))
        check_adam(f"adam_scaled step={step}", before, ps, ms, vs, S, lp=lps)


def _clip_coef(norm_dev, max_norm):
    """The device clip coefficient exactly as the optimizers form it, from their own fp32 norm."""
    return (max_norm / (norm_dev + 1e-6)).clamp(max=1.0).float().reshape(1)


@pytest.mark.gpu
@pytest.mark.parametrize("max_norm", [0.05, 1e4], ids=["binds", "free"])
def test_mixed_precision_step_envelope(max_norm):
    from colossalai_b200.amp import MixedPrecisionOptimizer
    from colossalai_b200.nn.optimizer import FusedAdam

    dev = _cuda()
    torch.manual_seed(8)
    model = torch.nn.Sequential(torch.nn.Linear(96, 200), torch.nn.GELU(), torch.nn.Linear(200, 33)).to(dev).bfloat16()
    opt = MixedPrecisionOptimizer(FusedAdam(model.parameters(), lr=0.02, weight_decay=0.1), model, precision="bf16",
                                  max_norm=max_norm)
    work = list(model.parameters())
    masters = [opt.working_to_master_map[p] for p in work]
    for step in range(1, 4):
        x = torch.randn(64, 96, device=dev).bfloat16()
        model(x).float().pow(2).mean().backward()
        grads = [p.grad.detach().clone() for p in work]
        st = opt.optim.state
        before = [_flat(masters), _flat(grads),
                  _flat([st[m]["exp_avg"] if m in st else torch.zeros_like(m) for m in masters]),
                  _flat([st[m]["exp_avg_sq"] if m in st else torch.zeros_like(m) for m in masters])]
        opt.step()
        n64 = float(before[1].norm())
        norm_dev = opt._grad_norm_dev
        assert abs(norm_dev.item() - n64) <= 64 * U * n64, (norm_dev.item(), n64)
        coef = _clip_coef(norm_dev, max_norm).item()
        assert (coef < 1.0) == (max_norm / (n64 + 1e-6) < 1.0)
        S = AdamScalars(0.02, 0.9, 0.999, 1e-8, 0.1, step, True, s=f32(1.0 * coef))
        check_adam(f"mixed_precision step={step}", before, masters, [st[m]["exp_avg"] for m in masters],
                   [st[m]["exp_avg_sq"] for m in masters], S, lp=[p.data for p in work])
        opt.zero_grad()


@pytest.mark.gpu
@pytest.mark.parametrize("max_norm", [0.05, 1e4], ids=["binds", "free"])
def test_low_level_zero_step_envelope(max_norm):
    import colossalai_b200
    from colossalai_b200.nn.optimizer import FusedAdam
    from colossalai_b200.testing import free_port
    from colossalai_b200.zero.low_level.low_level_optim import LowLevelZeroOptimizer

    dev = _cuda()
    if not torch.distributed.is_initialized():
        colossalai_b200.launch(0, 1, "127.0.0.1", free_port(), verbose=False)
    torch.manual_seed(9)
    model = torch.nn.Sequential(torch.nn.Linear(96, 200), torch.nn.GELU(), torch.nn.Linear(200, 33)).to(dev).bfloat16()
    opt = LowLevelZeroOptimizer(FusedAdam(model.parameters(), lr=0.02, weight_decay=0.1), clip_grad_norm=max_norm,
                                reduce_bucket_size=8192)
    assert len(opt.buckets) >= 2
    for step in range(1, 4):
        x = torch.randn(64, 96, device=dev).bfloat16()
        opt.backward(model(x).float().pow(2).mean())
        bs = [b for b in opt.buckets if b.grad_shard is not None]
        st = opt.optim.state
        masters = [b.master for b in bs]
        before = [_flat(masters), _flat([b.grad_shard for b in bs]),
                  _flat([st[m]["exp_avg"] if "exp_avg" in st[m] else torch.zeros_like(m) for m in masters]),
                  _flat([st[m]["exp_avg_sq"] if "exp_avg_sq" in st[m] else torch.zeros_like(m) for m in masters])]
        opt.step()
        n64 = float(before[1].norm())
        norm_dev = opt._grad_norm_dev
        assert abs(norm_dev.item() - n64) <= 64 * U * n64, (norm_dev.item(), n64)
        coef = _clip_coef(norm_dev, max_norm).item()
        assert (coef < 1.0) == (max_norm / (n64 + 1e-6) < 1.0)
        S = AdamScalars(0.02, 0.9, 0.999, 1e-8, 0.1, step, True, s=f32(1.0 * coef))
        check_adam(f"zero step={step}", before, [m.data for m in masters], [st[m]["exp_avg"] for m in masters],
                   [st[m]["exp_avg_sq"] for m in masters], S, lp=[b.working_shard() for b in bs])
        opt.zero_grad()


# ============================================================================================ SGD (GPU)
SGD_CASES = [dict(momentum=0.0), dict(momentum=0.9), dict(momentum=0.9, dampening=0.1),
             dict(momentum=0.9, nesterov=True), dict(momentum=0.9, weight_decay=0.05),
             dict(momentum=0.9, weight_decay=0.05, wd_after_momentum=True), dict(momentum=0.0, weight_decay=0.05)]


@pytest.mark.gpu
@pytest.mark.parametrize("p_dtype", [F32, BF16, F16])
@pytest.mark.parametrize("case", range(len(SGD_CASES)))
def test_fused_sgd_envelope(case, p_dtype):
    """FusedSGD over mt.sgd.  `first_run` is group-wide, as in the reference: it is true on the step where any
    param of the group creates its momentum buffer, and then every buffer of the group is overwritten with d."""
    from colossalai_b200.nn.optimizer import FusedSGD

    dev = _cuda()
    kw = dict(SGD_CASES[case])
    wd_after = kw.pop("wd_after_momentum", False)
    mu, damp, wd, nesterov = kw.get("momentum", 0.0), kw.get("dampening", 0.0), kw.get("weight_decay", 0.0), \
        kw.get("nesterov", False)
    gen = torch.Generator(device=dev).manual_seed(10 + case)
    sizes = [3, CHUNK + 5, 1000]
    ps = [torch.nn.Parameter((torch.randn(n, device=dev, generator=gen) * 0.5).to(p_dtype)) for n in sizes]
    lr = 0.05
    opt = FusedSGD(ps, lr=lr, wd_after_momentum=wd_after, **kw)
    L, M, D, W = f32(lr), f32(mu), f32(damp), f32(wd)
    omd = f32(1.0 - D)                                              # the kernel forms 1 - dampening in fp32
    for step in range(1, 4):
        for p in ps:
            p.grad = torch.randn(p.numel(), device=dev, generator=gen).to(p_dtype)
        p0, g0 = _flat(ps), _flat([p.grad for p in ps])
        b0 = _flat([opt.state[p]["momentum_buffer"] for p in ps]) if step > 1 else torch.zeros_like(p0)
        opt.step()
        d = g0 + W * p0 if (wd and not wd_after) else g0
        dmag = g0.abs() + ((W * p0).abs() if (wd and not wd_after) else 0.0)
        if mu:
            b = d if step == 1 else M * b0 + omd * d
            bg = _flat([opt.state[p]["momentum_buffer"] for p in ps])
            fb = 4 * U * (dmag if step == 1 else M * b0.abs() + omd * dmag)
            check(f"sgd.momentum step={step}", bg, b, F32, k=2, floor=fb)
            dmag = dmag + M * bg.abs() if nesterov else bg.abs()
            d = d + M * bg if nesterov else bg
        if wd and wd_after:
            d = d + W * p0
            dmag = dmag + (W * p0).abs()
        check(f"sgd.p step={step}", _flat(ps), p0 - L * d, p_dtype, k=1, floor=5 * U * L * dmag)


@pytest.mark.gpu
def test_mt_sgd_scaled_with_lp_copy():
    from colossalai_b200.ops import multi_tensor as mt

    dev = _cuda()
    gen = torch.Generator(device=dev).manual_seed(11)
    ps = [torch.randn(n, device=dev, generator=gen) * 0.5 for n in (7, CHUNK + 3)]
    ms = [torch.zeros_like(p) for p in ps]
    lps = [torch.zeros_like(p, dtype=BF16) for p in ps]
    for step in range(1, 3):
        gs = [(torch.randn(p.numel(), device=dev, generator=gen) * 4).to(BF16) for p in ps]
        p0, g0, b0 = _flat(ps), _flat(gs), _flat(ms)
        mt.sgd(mt.TensorTable(ps, gs, ms, None, lps), 0.05, 0.9, 0.0, 0.0, False, step == 1, inv_scale=0.25)
        d = g0 * 0.25
        b = d if step == 1 else f32(0.9) * b0 + d
        check(f"sgd.momentum scaled step={step}", _flat(ms), b, F32, k=2, floor=4 * U * (0.9 * b0.abs() + d.abs()))
        check(f"sgd.p scaled step={step}", _flat(ps), p0 - f32(0.05) * _flat(ms), F32, k=1,
              floor=3 * U * f32(0.05) * _flat(ms).abs())
        for p, lp in zip(ps, lps):
            check_bitwise("sgd.lp", lp, p.to(BF16))


# ============================================================================================ LAMB (GPU)
LAMB_CASES = [dict(), dict(adam_w_mode=False), dict(grad_averaging=False), dict(bias_correction=False),
              dict(wd=0.0), dict(wd=0.0, use_nvlamb=True), dict(use_nvlamb=True), dict(max_norm=1e9),
              dict(dtype=BF16), dict(dtype=BF16, wd=0.0)]


@pytest.mark.gpu
@pytest.mark.parametrize("case", range(len(LAMB_CASES)), ids=[",".join(f"{k}={v}" for k, v in c.items()) or "base"
                                                              for c in LAMB_CASES])
def test_fused_lamb_envelope(case):
    """FusedLAMB over mt.lamb.  bf16 params have bf16 gradients: stage 1 writes u into the gradient, so the
    reference rounds u to bf16 (it reads the stored u) before the trust ratio and stage 2."""
    kw = dict(LAMB_CASES[case])
    dtype = kw.pop("dtype", F32)
    _run_lamb_case(_cuda(), dtype, **kw)


# ============================================================================================ norms and scale (GPU)
def _arena_views(dev, dtype, sizes, base, gen):
    """Views into one arena starting `base` elements in (`base` = 1..7 lands off a 16-byte boundary: the scalar
    prologue), each next view at an odd offset."""
    tot = base + sum(s + 1 for s in sizes)
    a = (torch.randn(tot, device=dev, generator=gen) * 2).to(dtype)
    out, o = [], base
    for s in sizes:
        out.append(a[o:o + s])
        o += s + 1
    return out


@pytest.mark.gpu
@pytest.mark.parametrize("use_max", [False, True], ids=["l2", "max"])
@pytest.mark.parametrize("which,dtype", [("param", F32), ("param", BF16), ("param", F16), ("grad", F32),
                                         ("grad", BF16), ("grad", F16), ("m", F32)])
def test_norm_envelope(which, dtype, use_max):
    from colossalai_b200.ops import multi_tensor as mt

    dev = _cuda()
    gen = torch.Generator(device=dev).manual_seed(12)
    sizes = [int(x) for x in torch.randint(1, 40, (1100,), generator=torch.Generator().manual_seed(12))]
    sizes[5] = 0
    sizes[500] = 2 * CHUNK + 5
    sizes[1090] = CHUNK + 3                                         # past 1024 tensors: the finalize grid stride
    for base in (1, 3, 7):
        ts = _arena_views(dev, dtype, sizes, base, gen)
        tbl = {"param": lambda: mt.TensorTable(ts), "grad": lambda: mt.TensorTable(ts, ts),
               "m": lambda: mt.TensorTable(ts, None, ts)}[which]()
        tot, per = mt.norm_sq(tbl, which, per_tensor=True, use_max=use_max)
        x = [t.double() for t in ts]
        if use_max:                                                  # exact
            want = torch.stack([t.abs().max() if t.numel() else torch.zeros((), dtype=torch.float64, device=dev)
                                for t in x])
            assert torch.equal(per.double(), want), f"max {which} {dtype} base={base}"
            assert tot.item() == want.max().item()
        else:
            want = torch.stack([(t * t).sum() for t in x])
            nch = sum(math.ceil(s / CHUNK) for s in sizes)
            # per-thread loop (<= 16 adds) + block tree (10) + finalize loop (ceil(nch / 1024)) + its tree (10)
            depth = 16 + 10 + math.ceil(nch / 1024) + 10
            check(f"norm_l2.per {which} {dtype} base={base}", per, want, F32, k=1, floor=depth * U * want)
            check(f"norm_l2.total {which} {dtype} base={base}", tot, want.sum().reshape(1), F32, k=1,
                  floor=depth * U * want.sum())


@pytest.mark.gpu
@pytest.mark.parametrize("bad", [float("inf"), float("nan")], ids=["inf", "nan"])
@pytest.mark.parametrize("dtype", [F32, BF16])
def test_norm_propagates_inf_and_nan(bad, dtype):
    """inf gives inf and NaN gives NaN, for the L2 (sum of squares) and the max norm alike (torch's
    `vector_norm(ord=inf)` propagates NaN)."""
    from colossalai_b200.ops import multi_tensor as mt

    dev = _cuda()
    gen = torch.Generator(device=dev).manual_seed(13)
    ts = _arena_views(dev, dtype, [100, CHUNK + 9, 5], 3, gen)
    ts[1][CHUNK + 4] = bad
    for use_max in (False, True):
        tot, per = mt.norm_sq(mt.TensorTable(ts, ts), "grad", per_tensor=True, use_max=use_max)
        want = torch.linalg.vector_norm(ts[1].float(), ord=math.inf if use_max else 2)
        got = per[1]
        assert (got.isnan().item() and want.isnan().item()) or (got.item() == want.item() == math.inf), \
            (use_max, got.item(), want.item())
        assert tot.isnan().item() == bool(want.isnan().item()) and per[0].isfinite().item()


@pytest.mark.gpu
@pytest.mark.parametrize("src,dst", [(F32, F32), (BF16, F32), (F32, BF16), (F16, F16), (F32, F16)])
def test_scale_envelope(src, dst):
    from colossalai_b200.ops import multi_tensor as mt

    dev = _cuda()
    gen = torch.Generator(device=dev).manual_seed(14)
    sizes = [1, 3, 0, CHUNK, 3 * CHUNK + 5]
    xs = _arena_views(dev, src, sizes, 1, gen)
    ys = [torch.zeros(n, dtype=dst, device=dev) for n in sizes]
    s = 0.37
    flag = torch.zeros(1, dtype=torch.int32, device=dev)
    mt.scale(mt.TensorTable(xs, ys), s, flag)
    for x, y in zip(xs, ys):
        check_bitwise("scale", y, (x.float() * f32(s)).to(dst))
    assert flag.item() == 0
    for bad in (float("inf"), -float("inf"), float("nan")):
        for where in ("first", "last"):
            x2 = [x.clone() for x in xs]
            if where == "first":
                x2[0][0] = bad                                       # first element of the first chunk
            else:
                x2[-1][-1] = bad                                     # last element of the last chunk's tail
            flag.zero_()
            mt.scale(mt.TensorTable(x2, ys), s, flag)
            assert flag.item() == 1, (bad, where)
    flag.fill_(1)                                                    # finite data never clears the flag
    mt.scale(mt.TensorTable(xs, ys), s, flag)
    assert flag.item() == 1


# ============================================================================================ retention (GPU)
@pytest.mark.gpu
@pytest.mark.parametrize("opt_name", ["FusedAdam", "HybridAdam"])
def test_cached_tables_do_not_pin_gradients(opt_name):
    """20 steps with fresh gradients and zero_grad(): allocated memory returns to its level after step 1, within
    the size of the descriptor tables, instead of keeping earlier steps' gradients alive."""
    from colossalai_b200.nn import optimizer as optim

    dev = _cuda()
    ps = [torch.nn.Parameter(torch.randn(n, device=dev)) for n in (1 << 20, 3 << 18, 1000)]
    opt = getattr(optim, opt_name)(ps, lr=1e-3)
    grad_bytes = sum(p.numel() * 4 for p in ps)
    level = None
    for step in range(20):
        for p in ps:
            p.grad = torch.randn_like(p)
        opt.step()
        opt.zero_grad(set_to_none=True)
        torch.cuda.synchronize()
        if step == 0:
            level = torch.cuda.memory_allocated()
    tables = 17 * 2 * (len(ps) * 8 * 8 + 512)                        # at most 17 cached tables (+ allocator rounding)
    grown = torch.cuda.memory_allocated() - level
    assert grown <= tables, f"{opt_name}: {grown} bytes more after 20 steps ({grown / grad_bytes:.1f} gradient sets)"
