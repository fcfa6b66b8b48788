"""The flash-attention kernels (`flash_attn_wgmma.cu`) and the split-KV paged decode / verification kernels
(`inference.cu`) against float64 references, at tolerances that can fail.

Every reference is float64 on the GPU, computed from the exact 16-bit values the kernel read, chunked over heads and
query rows so that one score matrix stays under about 1 GB.  Elementwise checks use the comparator of the GEMM and
memory-bound envelopes:  |got - ref| <= k * ulp_out(|ref|) + floor, with a floor that is refused when its median
exceeds 1% of the median |ref|.  The worst err / tol per (kernel, dtype) is printed at module teardown.

Tier A - counting (q = 0, no ALiBi).  Every visible score is exactly 0, so every P entry is ex2(0) = 1, every masked
one is 0, and the fp32 row sum l equals the number n of visible keys exactly.  V holds integers in [-4, 4] (exact in
bf16, fp16 and e5m2; their fp32 sums are exact).  Then
  * lse == ln(n): the kernel forms (m + log2f(l)) * ln2 with m = 0; `lg2.approx` is budgeted at 2^-22 relative plus
    2^-22 absolute, the multiply at 2^-24, so |err| <= 2^-21 |ln n| + 2^-22;
  * O == mean of the visible V: o = sum V is exact, 1 / l is `rcp.approx` under fast math (budgeted 2^-22), the
    multiply adds 2^-24, and the output rounding half an ulp: |err| <= ulp_out / 2 + 5 * 2^-24 |O|;
  * block mode: o_state (fp32) == the mean over every key seen so far, to 5 * 2^-24 |O| after the first launch.  A
    resumed launch starts from m = lse * log2(e), so its keys weigh ex2(-m) ~ 1 / count instead of 1: that weight
    carries ex2.approx's error and, in the P V MMA only, the rounding to the input dtype (u_P times the new keys'
    share of the mean).  The lse stays exact to 2^-21 |lse| + 2^-22 + 2^-20 per resumed launch;
  * decode / verify: ml_part holds m = 0 and l == the count of keys in
    [max(s * part_len, window_start_j), min(len_j, (s + 1) * part_len)) for every (row, head, split); an empty split
    holds m = -inf and l = 0.  The reduced output obeys the O bound above (its merge weights are __expf(0) = 1).
This tier is exact about which keys each row sees: one dropped or extra key moves l by 1 and the lse by ~1 / n,
e.g. 6e-5 at n = 16384, 200 fp32 ulps.

Tier B - random operands, derived bound.  For the forward output, per element, with p the normalised softmax row:
    floor = u_P * P|V|                            P is rounded to the input dtype for the P V MMA (u_P = 2^-8 bf16,
                                                  2^-11 fp16), while l sums the unrounded P
          + (P eta) |V| + |O| * sum(P eta)        eta_j bounds the relative error of p_j from its exponent argument:
                                                  scale * (D / 16) * G16 * (|q| |k_j|) for Q K^T in k16 wgmma steps
                                                  (G16 = 2^-22 per step, the GEMM envelope's constant),
                                                  ln2 * 2^-24 * (4 |x_j| + |x_j - m|) for the fp32 scale multiply,
                                                  the ALiBi fmaf and the subtraction of the max (x in log2 units),
                                                  and 2^-22 for ex2.approx.ftz.  P eta (|V| + |O|) bounds
                                                  sum p eta |V - O|, the first-order effect of those errors on O
          + (8 * tiles * G16 + tiles * 2^-24) P|V|  the fp32 accumulator over key tiles (8 k16 steps per tile) and its
                                                  alpha rescale, once per tile
          + (tiles + 40) * 2^-24 * |O|            l: 32 adds per tile and thread, one per tile, the 4-lane shuffle sum,
                                                  plus 1 / l and the normalising multiply
          + fp16 only: 2^-25 * sum_visible |V| / l  P below 2^-14 rounds in fp16's subnormal range (absolute 2^-25)
and k = 1 ulp of the output dtype for its one rounding.  The LSE floor is sum(P delta) + (tiles + 40) * 2^-24 +
2^-22 (1 + |log2 l|) + 2^-23 |lse|, with delta = eta - 2^-22 plus 2^-22 for ex2: the error of ln sum exp(x) is the
P-weighted mean error of x, l's relative error, lg2.approx and the final roundings.  V is uniform in [0.5, 1.5]
(positive mean) so the floor stays under 1% of the median |O| even at S = 16384.  A large-scale case (scores up to
about +-150, where exp without the running max overflows fp32) exercises the alpha rescale.  A signed-mean check
requires |mean(got - ref)| <= (4 * mean(floor) + mean(ulp)) / sqrt(N), N the number of (row, head) outputs (the D
elements of one output row share its rounded P, so they are not independent samples): a P rounded toward zero shifts
every element the same way and fails it even where each element stays within its floor.  The limit adds one
one-signed budget, DRIFT16 = 2^-21 of P|V| per k16 step of the P V MMA: on an H100 the accumulator drifts toward zero
over long rows (measured at S = 16384, one head: mean error -3.4e-4 with bf16 and -5.3e-5 with fp16 for O ~ 1, that
is 2^-21.6 per step for bf16).  P rounded toward zero drifts by about u_P / 2 instead, over 100 times more.

Backward (`cb_flash_attn_bwd`, `cb_flash_attn_block_bwd`, the delta kernel): the references take what the forward
saved, the 16-bit `out` and fp32 `lse`: P = exp(scale q k^T - lse), delta = rowsum(dO o out), dS = P o (dP - delta).
  * P carries eta as above (lse enters the argument, its fp32 scaling adds 2^-23 |lse2|); P and dS are rounded to the
    input dtype before the MMAs (u_P, u_dS = u_P), with an absolute 2^-25 for fp16's subnormal range;
  * dP = dO V^T carries (D / 16) * G16 * |dO||V|; delta carries (D / 8 + 5) * 2^-24 * |dO||out| (8 products per lane,
    then a 5-level warp sum); flash_delta itself is checked against that floor;
  * dV = P^T dO and dK = scale dS^T Q accumulate over every query tile of every head of the GQA group in k16 steps
    (G16 per step); dQ = scale dS K takes 8 k16 steps per key tile and one fp32 atomic add (2^-24) per key tile.
To keep the floors under 1% of the median, the backward operands make dS keep its sign per key and dS K keep its
sign per query: V_k = c_k + noise and K_k = (c_k - 1) * (+1, -1, +1, ...) + noise with c_k uniform in [0.5, 1.5], and
Q, dO uniform in [0.5, 1.5] (so scores do not favour large c_k, and dQ = scale * Cov_P(dP, K) does not cancel).

Repeatability: every Tier B case runs twice and these must be bitwise identical: forward out, lse and o_state;
dK and dV of cb_flash_attn_bwd (accumulated in registers in a fixed order, stored once); decode and verify outputs.
dQ and the block-mode backward accumulators are excluded: they are sums of fp32 atomicAdds from different CTAs, whose
order the hardware does not fix.

Locality: the forward's out / lse rows of one sequence must not depend on another sequence's q / k / v rows, even
NaN / Inf ones (packed and uniform batches, and the paged variant's unwritten tail slots).  The backward does not keep
that promise (documented at `cb_flash_attn_bwd`); its test is a strict xfail.

`test_comparators_reject_simulated_faults` runs without a GPU: it simulates in float64 ten kernel faults at the GPU
tests' shapes and shows that the checks used here reject each.
"""
import ctypes
import itertools
import math

import pytest
import torch

U = 2.0 ** -24
G16 = 2.0 ** -22                      # per k16 wgmma step, of the running sum of |a * b| (test_gemm_envelope.py)
EX2 = 2.0 ** -22                      # ex2.approx.ftz relative error
DRIFT16 = 2.0 ** -21                  # one-signed drift of the P V accumulator per k16 step (measured, see docstring)
LN2 = math.log(2.0)
LOG2E = 1.0 / LN2
BF16, F16 = torch.bfloat16, torch.float16
DTYPES = [BF16, F16]
U_P = {BF16: 2.0 ** -8, F16: 2.0 ** -11}
SUB_P = {BF16: 0.0, F16: 2.0 ** -25}  # absolute rounding error of P / dS in fp16's subnormal range
_MANT = {BF16: 8, F16: 11, torch.float32: 24}
_MIN_STEP = {BF16: 2.0 ** -133, F16: 2.0 ** -24, torch.float32: 2.0 ** -149}
_NAME = {BF16: "bf16", F16: "f16", torch.float32: "f32"}
_WORST = {}                           # "kernel.dtype" -> largest |err| / tol seen
CHUNK = 2 ** 27                       # float64 elements per score chunk (1 GiB)


# ============================================================================================ comparators
def ulp(ref, dtype):
    """Spacing of `dtype` at |ref| (never below its subnormal step)."""
    _, e = torch.frexp(ref.abs().double())
    return torch.ldexp(torch.ones_like(ref, dtype=torch.float64), e - _MANT[dtype]).clamp_min(_MIN_STEP[dtype])


def _record(what, ratio):
    _WORST[what] = max(_WORST.get(what, 0.0), ratio)


def check(what, got, ref, dtype, k=1.0, floor=0.0, signed_mean=0, drift=0.0):
    """|got - ref| <= k * ulp(|ref|) + floor elementwise; a floor above 1% of the median |ref| is refused.  Where
    the reference is identically 0 (dK / dQ of a one-token sequence) the floor alone bounds |got|.
    `signed_mean` = g > 0 also bounds the mean signed error, counting groups of g elements (one output row of one
    head: its D elements share the same rounded P) as the independent samples, plus the mean of the one-signed
    `drift` budget."""
    got, ref = got.double().flatten(), ref.double().flatten()
    assert got.shape == ref.shape, (what, got.shape, ref.shape)
    assert torch.isfinite(ref).all(), f"{what}: non-finite reference"
    floor = torch.as_tensor(floor, dtype=torch.float64, device=ref.device).flatten().expand_as(ref)
    zero = (ref == 0) & (floor == 0)
    nz_zero = int((got[zero] != 0).sum())
    assert nz_zero == 0, f"{what}: {nz_zero} elements whose reference is exactly 0 are not 0"
    nz = ~zero
    if not nz.any():
        return
    med = ref[nz].abs().median()
    if med == 0:
        check_exact_tol(what, got, ref, floor)
        return
    assert floor[nz].median() <= 0.01 * med, f"{what}: floor {floor[nz].median():.3g} > 1% of median |ref| {med:.3g}"
    tol = k * ulp(ref, dtype) + floor
    err = (got - ref).abs()
    bad = nz & ~(err <= tol)                    # NaN in `got` counts as bad
    if bad.any():
        i = int(bad.nonzero()[0])
        raise AssertionError(f"{what}: {int(bad.sum())} of {int(nz.sum())} elements out of tolerance; first at flat "
                             f"index {i}: got {got[i].item():.9g} ref {ref[i].item():.9g} tol {tol[i].item():.3g}")
    if signed_mean:
        drift = torch.as_tensor(drift, dtype=torch.float64, device=ref.device).flatten().expand_as(ref)
        n = max(1, int(nz.sum()) // signed_mean)
        mean_err = float((got - ref)[nz].mean())
        lim = (4 * float(floor[nz].mean()) + float(ulp(ref[nz], dtype).mean())) / math.sqrt(n) + float(drift[nz].mean())
        assert abs(mean_err) <= lim, f"{what}: signed mean error {mean_err:.3g} beyond {lim:.3g}  over {n} rows"
    _record(what.split(" ")[0], float((err[nz] / tol[nz]).max()))


def check_exact_f32(what, got, ref, rel, abs_=0.0):
    """Tier A: |got - ref| <= rel * |ref| + abs_, with -inf only where ref is -inf."""
    got, ref = got.double().flatten(), ref.double().flatten()
    assert got.shape == ref.shape, (what, got.shape, ref.shape)
    inf = torch.isinf(ref)
    assert torch.equal(got[inf], ref[inf]), f"{what}: rows without keys must hold -inf, got {got[inf][:4].tolist()}"
    g, r = got[~inf], ref[~inf]
    tol = rel * r.abs() + abs_
    err = (g - r).abs()
    bad = ~(err <= tol)
    if bad.any():
        i = int(bad.nonzero()[0])
        raise AssertionError(f"{what}: {int(bad.sum())} of {r.numel()} out of tolerance; first: got "
                             f"{g[i].item():.9g} ref {r[i].item():.9g} tol {tol[i].item():.3g}")
    if r.numel():
        _record(what.split(" ")[0], float((err / tol.clamp_min(1e-300)).max()))


def check_count_out(what, got, ref, dtype):
    """Tier A output: half an ulp of `dtype` (fp32: none) plus 5 * 2^-24 |O| (rcp.approx and the multiply)."""
    half = 0.5 * ulp(ref, dtype) if dtype != torch.float32 else 0.0
    check_exact_tol(what, got, ref, half + 5 * U * ref.double().abs())


def check_exact_tol(what, got, ref, tol):
    got, ref = got.double().flatten(), ref.double().flatten()
    tol = torch.as_tensor(tol, dtype=torch.float64, device=ref.device).flatten().expand_as(ref)
    err = (got - ref).abs()
    bad = ~(err <= tol)
    if bad.any():
        i = int(bad.nonzero()[0])
        raise AssertionError(f"{what}: {int(bad.sum())} of {ref.numel()} out of tolerance; first at {i}: got "
                             f"{got[i].item():.9g} ref {ref[i].item():.9g} tol {tol[i].item():.3g}")
    pos = tol > 0
    if pos.any():
        _record(what.split(" ")[0], float((err[pos] / tol[pos]).max()))


def _bits(t):
    return t.contiguous().view({4: torch.int32, 2: torch.int16, 1: torch.int8}[t.element_size()])


def check_bitwise(what, got, want):
    assert got.dtype == want.dtype and got.shape == want.shape, (what, got.dtype, want.dtype, got.shape, want.shape)
    diff = (_bits(got) != _bits(want)).flatten()
    if diff.any():
        i = int(diff.nonzero()[0])
        raise AssertionError(f"{what}: {int(diff.sum())} of {diff.numel()} elements differ bitwise; first at flat "
                             f"index {i}: got {got.flatten()[i].item()!r} want {want.flatten()[i].item()!r}")


@pytest.fixture(scope="module", autouse=True)
def _report_worst():
    yield
    if _WORST:
        print("\nlargest error-to-tolerance ratio per kernel and dtype:")
        for k, v in sorted(_WORST.items()):
            print(f"  {k:<32} {v:.3f}")


# ============================================================================================ float64 references
def visible(qpos, kpos, causal, window=0):
    """[Sq, Sk] bool: key kpos visible from query qpos (absolute positions)."""
    rel = kpos[None, :] - qpos[:, None]
    keep = torch.ones_like(rel, dtype=torch.bool)
    if causal:
        keep &= rel <= 0
    if window:
        keep &= rel > -window
    return keep


def attn64(q, k, v, scale, keep, slopes=None, qpos=None, kpos=None, bounds=True, dtype=BF16):
    """float64 attention of one sequence: q [Sq, Hq, D], k / v [Sk, Hkv, D], keep [Sq, Sk].  Returns out [Sq, Hq, D],
    lse [Sq, Hq] and (with `bounds`) the Tier B floors of out and lse (module docstring)."""
    q, k, v = q.double(), k.double(), v.double()
    Sq, Hq, D = q.shape
    Sk, Hkv = k.shape[0], k.shape[1]
    G = Hq // Hkv
    tiles = max(1, -(-Sk // 128))
    out = torch.zeros(Sq, Hq, D, dtype=torch.float64, device=q.device)
    lse = torch.full((Sq, Hq), float("-inf"), dtype=torch.float64, device=q.device)
    f_out = torch.zeros_like(out)
    f_lse = torch.zeros_like(lse)
    rows = max(1, min(Sq, CHUNK // max(1, Sk * 4)))
    for h in range(Hq):
        kh, vh = k[:, h // G], v[:, h // G]
        for r0 in range(0, Sq, rows):
            r1 = min(Sq, r0 + rows)
            qh = q[r0:r1, h]
            x = (qh @ kh.t()) * (scale * LOG2E)                              # log2 units
            if slopes is not None:
                x = x + float(slopes[h]) * LOG2E * (kpos[None, :] - qpos[r0:r1, None]).double()
            x = x.masked_fill(~keep[r0:r1], float("-inf"))
            m = x.amax(-1, keepdim=True)
            live = torch.isfinite(m)
            ms = torch.where(live, m, torch.zeros_like(m))
            e = torch.exp2(x - ms)
            l = e.sum(-1, keepdim=True)
            p = e / l.clamp_min(1e-300)
            o = p @ vh
            out[r0:r1, h] = o
            lse[r0:r1, h] = torch.where(live[:, 0], (ms[:, 0] + torch.log2(l[:, 0])) * LN2,
                                        torch.full_like(l[:, 0], float("-inf")))
            if not bounds:
                continue
            a = (qh.abs() @ kh.abs().t()) * scale
            xf = torch.where(keep[r0:r1], x, torch.zeros_like(x))
            delta = a * (D / 16) * G16 + LN2 * U * (4 * xf.abs() + (xf - ms).abs())
            eta = delta + EX2
            vabs = vh.abs()
            pv = p @ vabs
            pe = p * eta
            fo = U_P[dtype] * pv + pe @ vabs + o.abs() * pe.sum(-1, keepdim=True)
            fo += (8 * tiles * G16 + tiles * U) * pv + (tiles + 40) * U * o.abs()
            if SUB_P[dtype]:
                fo += SUB_P[dtype] * (keep[r0:r1].double() @ vabs) / l.clamp_min(1e-300)
            f_out[r0:r1, h] = fo
            f_lse[r0:r1, h] = (p * delta).sum(-1) + EX2 + (tiles + 40) * U + EX2 * (1 + torch.log2(l[:, 0]).abs()) \
                + 2 * U * lse[r0:r1, h].abs().nan_to_num(0, 0, 0)
    return out, lse, f_out, f_lse


# ============================================================================================ device helpers
def _cuda():
    if not torch.cuda.is_available() or torch.cuda.get_device_capability()[0] != 9:
        pytest.skip("needs an sm_90 GPU")
    return torch.device("cuda")


def _fa():
    from colossalai_b200.ops import flash_attn_native as fa
    return fa


def fwd(q, k, v, *, causal, batch=1, cu=None, window=0, slopes=None, o_state=None, lse=None, has_prev=False,
        paged=None, scale=None):
    """cb_flash_attn_fwd on tensors; returns (out, lse).  `paged` = (tables, seq_lens) with k / v the caches."""
    fa = _fa()
    T, Hq, D = q.shape
    scale = D ** -0.5 if scale is None else scale
    out = torch.full_like(q, float("nan"))
    lse = torch.full((T, Hq), float("nan"), dtype=torch.float32, device=q.device) if lse is None else lse
    kw = {}
    if cu is not None:
        kw.update(cu_seqlens=cu.data_ptr(), total_tokens=T)
    if paged is not None:
        tables, lens = paged
        kw.update(block_tables=tables.data_ptr(), seq_lens=lens.data_ptr(), block_size=k.shape[1],
                  max_blocks=tables.shape[1], num_blocks=k.shape[0])
    nb = cu.numel() - 1 if cu is not None else batch
    Hkv = k.shape[-2]
    fa._fwd("fwd", q.data_ptr(), k.data_ptr(), v.data_ptr(), 0 if o_state is not None else out.data_ptr(),
            lse.data_ptr(), nb, T // batch if cu is None else 0, (k.shape[0] // batch) if cu is None else 0, Hq, Hkv,
            D, causal, scale, q.dtype, o_state=o_state.data_ptr() if o_state is not None else 0, has_prev=has_prev,
            window=window, alibi=slopes.data_ptr() if slopes is not None else 0, **kw)
    torch.cuda.synchronize()
    return out, lse


def _int_v(shape, dev, gen):
    return torch.randint(-4, 5, shape, generator=gen, device="cpu").float().to(dev)


def _cu(lens, dev):
    return torch.tensor([0] + list(itertools.accumulate(lens)), dtype=torch.int32, device=dev)


def _segments(lens):
    at = 0
    for L in lens:
        yield at, at + L
        at += L


# ============================================================================================ Tier A: forward
def _tier_a_expect(v, keep, G):
    """Mean of the visible V and ln(count) for q = 0: v [Sk, Hkv, D], keep [Sq, Sk] -> ([Sq, Hq, D], [Sq, Hq])."""
    n = keep.double().sum(-1)                                                      # [Sq]
    s = keep.double() @ v.double().flatten(1)                                      # [Sq, Hkv * D]
    mean = (s / n.clamp_min(1)[:, None]).view(keep.shape[0], v.shape[1], v.shape[2]).repeat_interleave(G, 1)
    lse = torch.where(n > 0, n.clamp_min(1).log(), torch.full_like(n, float("-inf")))
    return mean, lse[:, None].expand(-1, v.shape[1] * G)


def _check_tier_a(tag, out, lse, mean, lse_ref, dtype):
    check_exact_f32(f"fwd_lse.{_NAME[dtype]} {tag}", lse, lse_ref, 2.0 ** -21, 2.0 ** -22)
    check_count_out(f"fwd_out.{_NAME[dtype]} {tag}", out.float(), mean, dtype)


UNIFORM_S = [1, 63, 64, 127, 128, 129, 255, 256, 257, 1000, 4096]


@pytest.mark.gpu
@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("D", [64, 128])
@pytest.mark.parametrize("causal", [False, True])
def test_fwd_counting_uniform(dtype, D, causal):
    """Every length of UNIFORM_S over 3 ragged batch entries (a key tile crosses into the next entry), G cycling
    over 1..16, plus 16384 on one head."""
    dev = _cuda()
    gen = torch.Generator().manual_seed(D + causal)
    for i, S in enumerate(UNIFORM_S + [16384]):
        G = [1, 2, 4, 8, 16][i % 5]
        Hkv, B = (1, 1) if S == 16384 else (2 if G < 16 else 1, 3)
        q = torch.zeros(B * S, Hkv * G, D, dtype=dtype, device=dev)
        v = _int_v((B * S, Hkv, D), dev, gen).to(dtype)
        k = torch.randn(B * S, Hkv, D, generator=gen).to(dev, dtype)
        out, lse = fwd(q, k, v, causal=causal, batch=B)
        pos = torch.arange(S, device=dev)
        keep = visible(pos, pos, causal)
        for b in range(B):
            mean, lref = _tier_a_expect(v[b * S:(b + 1) * S], keep, G)
            _check_tier_a(f"uniform S={S} G={G} b={b}", out[b * S:(b + 1) * S], lse[b * S:(b + 1) * S], mean, lref,
                          dtype)


@pytest.mark.gpu
@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("D", [64, 128])
def test_fwd_counting_cross_attention(dtype, D):
    """Non-causal seqlen_q != seqlen_k, batch 2: 1 x 1000, 300 x 77, 129 x 4096; MQA 32 over 1 on the last."""
    dev = _cuda()
    gen = torch.Generator().manual_seed(D)
    for Sq, Sk, Hq, Hkv in [(1, 1000, 4, 2), (300, 77, 8, 2), (129, 4096, 32, 1)]:
        q = torch.zeros(2 * Sq, Hq, D, dtype=dtype, device=dev)
        k = torch.randn(2 * Sk, Hkv, D, generator=gen).to(dev, dtype)
        v = _int_v((2 * Sk, Hkv, D), dev, gen).to(dtype)
        out, lse = fwd(q, k, v, causal=False, batch=2)
        keep = torch.ones(Sq, Sk, dtype=torch.bool, device=dev)
        for b in range(2):
            mean, lref = _tier_a_expect(v[b * Sk:(b + 1) * Sk], keep, Hq // Hkv)
            _check_tier_a(f"cross {Sq}x{Sk} b={b}", out[b * Sq:(b + 1) * Sq], lse[b * Sq:(b + 1) * Sq], mean, lref,
                          dtype)


PACKED_LENS = [
    [0, 1, 127, 128, 129, 0, 300, 0],                     # empty first, in the middle and last
    [2, 1, 3] * 66 + [1, 2],                              # 200 tiny sequences: most CTAs of the grid exit at once
    [5, 3000, 64, 63],                                    # one long sequence
]


@pytest.mark.gpu
@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("D", [64, 128])
@pytest.mark.parametrize("causal", [False, True])
def test_fwd_counting_packed(dtype, D, causal):
    dev = _cuda()
    gen = torch.Generator().manual_seed(3 * D + causal)
    for lens in PACKED_LENS:
        T = sum(lens)
        Hq, Hkv = 8, 2
        q = torch.zeros(T, Hq, D, dtype=dtype, device=dev)
        k = torch.randn(T, Hkv, D, generator=gen).to(dev, dtype)
        v = _int_v((T, Hkv, D), dev, gen).to(dtype)
        out, lse = fwd(q, k, v, causal=causal, cu=_cu(lens, dev))
        for a, b in _segments(lens):
            if a == b:
                continue
            pos = torch.arange(b - a, device=dev)
            mean, lref = _tier_a_expect(v[a:b], visible(pos, pos, causal), Hq // Hkv)
            _check_tier_a(f"packed len={b - a}", out[a:b], lse[a:b], mean, lref, dtype)


@pytest.mark.gpu
@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("D", [64, 128])
def test_fwd_counting_prefill_window(dtype, D):
    """Sliding window 1, 127, 128, 129 and one beyond every length (q = 0: ALiBi is Tier B)."""
    dev = _cuda()
    gen = torch.Generator().manual_seed(D)
    lens = [1, 129, 0, 700, 128]
    T = sum(lens)
    q = torch.zeros(T, 8, D, dtype=dtype, device=dev)
    k = torch.randn(T, 2, D, generator=gen).to(dev, dtype)
    v = _int_v((T, 2, D), dev, gen).to(dtype)
    for window in (1, 127, 128, 129, 5000):
        out, lse = fwd(q, k, v, causal=True, cu=_cu(lens, dev), window=window)
        for a, b in _segments(lens):
            if a == b:
                continue
            pos = torch.arange(b - a, device=dev)
            mean, lref = _tier_a_expect(v[a:b], visible(pos, pos, True, window), 4)
            _check_tier_a(f"prefill window={window} len={b - a}", out[a:b], lse[a:b], mean, lref, dtype)


@pytest.mark.gpu
@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("D", [64, 128])
def test_fwd_counting_block_chain(dtype, D):
    """Block mode over 4 launches (a causal first block, then full blocks): o_state is the running mean of every V
    seen so far, lse the log of their count; rows not a multiple of 128."""
    dev = _cuda()
    gen = torch.Generator().manual_seed(D)
    rows, Hq, Hkv = 300, 8, 2
    q = torch.zeros(rows, Hq, D, dtype=dtype, device=dev)
    o_state = torch.empty(rows, Hq, D, dtype=torch.float32, device=dev)
    lse = torch.empty(rows, Hq, dtype=torch.float32, device=dev)
    pos = torch.arange(rows, device=dev)
    total = torch.zeros(rows, Hkv * D, dtype=torch.float64, device=dev)
    count = torch.zeros(rows, dtype=torch.float64, device=dev)
    for i in range(4):
        causal = i == 0
        k = torch.randn(rows, Hkv, D, generator=gen).to(dev, dtype)
        v = _int_v((rows, Hkv, D), dev, gen).to(dtype)
        fwd(q, k, v, causal=causal, o_state=o_state, lse=lse, has_prev=i > 0)
        keep = visible(pos, pos, causal).double()
        total += keep @ v.double().flatten(1)
        count += keep.sum(-1)
        mean = (total / count[:, None]).view(rows, Hkv, D).repeat_interleave(Hq // Hkv, 1)
        check_exact_f32(f"block_lse.{_NAME[dtype]} link={i}", lse, count.log()[:, None].expand(-1, Hq), 2.0 ** -21,
                        2.0 ** -22 + i * 2.0 ** -20)
        # a resumed launch starts from m = lse * log2(e) > 0, so its new keys weigh p = ex2(-m) ~ 1 / count instead of
        # 1: ex2.approx and the rounding of m move that weight by 2^-21 relative (times |v - mean| <= 8), and P's
        # rounding to the input dtype for the MMA by u_P (times the new keys' share of the mean, |v| <= 4)
        new = keep.sum(-1)[:, None, None] / count[:, None, None]
        tol = (5 + 4 * i) * U * mean.abs() + (i > 0) * (2.0 ** -21 * 8 + U_P[dtype] * 4 * new)
        check_exact_tol(f"block_ostate.{_NAME[dtype]} link={i}", o_state, mean, tol)


def _paged_case(lens_k, new, bs, Hkv, D, dtype, dev, gen, kv_fn, tail=0.0):
    """A paged cache holding each sequence's K/V in permuted blocks; unreferenced blocks NaN, table tails -1, the
    last block's unwritten slots `tail`."""
    nblk = [(L + bs - 1) // bs for L in lens_k]
    num_blocks = sum(nblk) + 5
    perm = torch.randperm(num_blocks, generator=gen).tolist()
    tables = torch.full((len(lens_k), max(nblk) + 2), -1, dtype=torch.int32)
    kc = torch.full((num_blocks, bs, Hkv, D), float("nan"), dtype=dtype, device=dev)
    vc = torch.full_like(kc, float("nan"))
    ks, vs, at = [], [], 0
    for b, L in enumerate(lens_k):
        ids = perm[at:at + nblk[b]]
        at += nblk[b]
        tables[b, :nblk[b]] = torch.tensor(ids, dtype=torch.int32)
        k, v = kv_fn(L)
        kk = torch.full((nblk[b] * bs, Hkv, D), tail, dtype=dtype, device=dev)
        vv = kk.clone()
        kk[:L], vv[:L] = k, v
        kc[ids] = kk.view(-1, bs, Hkv, D)
        vc[ids] = vv.view(-1, bs, Hkv, D)
        ks.append(k)
        vs.append(v)
    return kc, vc, tables.to(dev), torch.tensor(lens_k, dtype=torch.int32, device=dev), ks, vs


@pytest.mark.gpu
@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("D", [64, 128])
@pytest.mark.parametrize("bs", [8, 16, 32, 64, 128])
def test_fwd_counting_paged(dtype, D, bs):
    """Paged prefill with an lse: cached lengths off the block grid, windows, NaN tail slots."""
    dev = _cuda()
    gen = torch.Generator().manual_seed(bs + D)
    Hq, Hkv = 8, 2
    cached, new = [0, bs + 3, 5 * bs - 1, 200], [7, 129, 1, 300]
    lens_k = [c + n for c, n in zip(cached, new)]
    kc, vc, tables, lk, ks, vs = _paged_case(
        lens_k, new, bs, Hkv, D, dtype, dev, gen,
        lambda L: (torch.randn(L, Hkv, D, generator=gen).to(dev, dtype), _int_v((L, Hkv, D), dev, gen).to(dtype)),
        tail=float("nan"))
    q = torch.zeros(sum(new), Hq, D, dtype=dtype, device=dev)
    for window in (0, 1, 129, 10000):
        out, lse = fwd(q, kc, vc, causal=True, cu=_cu(new, dev), window=window, paged=(tables, lk))
        for b, (a, e) in enumerate(_segments(new)):
            L = lens_k[b]
            keep = visible(torch.arange(L - new[b], L, device=dev), torch.arange(L, device=dev), True, window)
            mean, lref = _tier_a_expect(vs[b], keep, Hq // Hkv)
            _check_tier_a(f"paged bs={bs} window={window} b={b}", out[a:e], lse[a:e], mean, lref, dtype)


# ============================================================================================ Tier B: forward
def _rand_qkv(T, Tk, Hq, Hkv, D, dtype, dev, gen, qscale=1.0):
    q = (torch.randn(T, Hq, D, generator=gen) * qscale).to(dev, dtype)
    k = torch.randn(Tk, Hkv, D, generator=gen).to(dev, dtype)
    v = (torch.rand(Tk, Hkv, D, generator=gen) + 0.5).to(dev, dtype)
    return q, k, v


def _check_b(tag, dtype, out, lse, ref, f_out, lse_ref, f_lse, keys):
    # V > 0, so P|V| = |O|: the accumulator's drift budget over the 8 k16 steps of each of the ceil(keys / 128) tiles
    drift = DRIFT16 * 8 * -(-keys // 128) * ref.abs()
    check(f"fwd_out.{_NAME[dtype]} {tag}", out, ref, dtype, floor=f_out, signed_mean=ref.shape[-1], drift=drift)
    if lse is not None:
        check(f"fwd_lse.{_NAME[dtype]} {tag}", lse, lse_ref, torch.float32, k=1.0, floor=f_lse)


def _twice(fn):
    a = fn()
    b = fn()
    for i, (x, y) in enumerate(zip(a, b)):
        if x is not None:
            check_bitwise(f"repeat[{i}]", x, y)
    return a


@pytest.mark.gpu
@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("D", [64, 128])
@pytest.mark.parametrize("causal", [False, True])
def test_fwd_random_uniform(dtype, D, causal):
    dev = _cuda()
    gen = torch.Generator().manual_seed(7 * D + causal)
    for i, S in enumerate([1, 64, 129, 257, 1000, 4096, 16384]):
        G = [1, 2, 4, 8, 16, 4, 1][i]
        Hkv, B = (1, 1) if S >= 4096 else (2, 2)
        q, k, v = _rand_qkv(B * S, B * S, Hkv * G, Hkv, D, dtype, dev, gen)
        out, lse = _twice(lambda: fwd(q, k, v, causal=causal, batch=B))
        pos = torch.arange(S, device=dev)
        keep = visible(pos, pos, causal)
        for b in range(B):
            sl = slice(b * S, (b + 1) * S)
            ref, lref, fo, fl = attn64(q[sl], k[sl], v[sl], D ** -0.5, keep, dtype=dtype)
            _check_b(f"uniform S={S} G={G}", dtype, out[sl], lse[sl], ref, fo, lref, fl, S)


@pytest.mark.gpu
@pytest.mark.parametrize("dtype", DTYPES)
def test_fwd_random_large_scores_rescale(dtype):
    """Scores up to about +-150 (q scaled by 12): exp without the running max overflows fp32; the alpha rescale is
    exercised on almost every tile.  Cross attention 129 x 4096 and causal packed."""
    dev = _cuda()
    gen = torch.Generator().manual_seed(11)
    D = 128
    q, k, v = _rand_qkv(129, 4096, 4, 2, D, dtype, dev, gen, qscale=12.0)
    out, lse = _twice(lambda: fwd(q, k, v, causal=False, batch=1))
    ref, lref, fo, fl = attn64(q, k, v, D ** -0.5, torch.ones(129, 4096, dtype=torch.bool, device=dev), dtype=dtype)
    _check_b("large 129x4096", dtype, out, lse, ref, fo, lref, fl, 4096)
    lens = [1000, 77, 513]
    q, k, v = _rand_qkv(sum(lens), sum(lens), 8, 2, D, dtype, dev, gen, qscale=12.0)
    out, lse = _twice(lambda: fwd(q, k, v, causal=True, cu=_cu(lens, dev)))
    for a, b in _segments(lens):
        pos = torch.arange(b - a, device=dev)
        ref, lref, fo, fl = attn64(q[a:b], k[a:b], v[a:b], D ** -0.5, visible(pos, pos, True), dtype=dtype)
        _check_b(f"large packed len={b - a}", dtype, out[a:b], lse[a:b], ref, fo, lref, fl, b - a)


@pytest.mark.gpu
@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("D", [64, 128])
def test_fwd_random_packed_and_prefill(dtype, D):
    """Packed causal / non-causal, then prefill with ALiBi (with and without a window) and a window alone."""
    dev = _cuda()
    gen = torch.Generator().manual_seed(13 + D)
    lens = [0, 1, 127, 128, 129, 0, 1000]
    Hq, Hkv = 8, 2
    T = sum(lens)
    q, k, v = _rand_qkv(T, T, Hq, Hkv, D, dtype, dev, gen)
    slopes = torch.tensor([2 ** (-(h + 1) / 2) for h in range(Hq)], dtype=torch.float32, device=dev)
    cases = [(False, 0, None), (True, 0, None), (True, 0, slopes), (True, 129, slopes), (True, 128, None)]
    for causal, window, sl in cases:
        out, lse = _twice(lambda: fwd(q, k, v, causal=causal, cu=_cu(lens, dev), window=window, slopes=sl))
        for a, b in _segments(lens):
            if a == b:
                continue
            pos = torch.arange(b - a, device=dev)
            ref, lref, fo, fl = attn64(q[a:b], k[a:b], v[a:b], D ** -0.5, visible(pos, pos, causal, window), sl,
                                       pos, pos, dtype=dtype)
            _check_b(f"packed causal={causal} window={window} alibi={sl is not None} len={b - a}", dtype, out[a:b],
                     lse[a:b], ref, fo, lref, fl, b - a)


@pytest.mark.gpu
@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("D", [64, 128])
def test_fwd_random_block_chain(dtype, D):
    """Block mode, 3 launches whose keys are x4 (the later block dominates) or x0.25 (dominated), causal last block,
    rows not a multiple of 128; the chain's state is checked after the last launch against the float64 attention over
    the concatenated keys."""
    dev = _cuda()
    gen = torch.Generator().manual_seed(17 + D)
    rows, Hq, Hkv = 200, 4, 2
    for ks_ in ([1.0, 4.0, 4.0], [1.0, 0.25, 0.25]):
        q = torch.randn(rows, Hq, D, generator=gen).to(dev, dtype)
        blocks = [(torch.randn(rows, Hkv, D, generator=gen) * s).to(dev, dtype) for s in ks_]
        vals = [(torch.rand(rows, Hkv, D, generator=gen) + 0.5).to(dev, dtype) for _ in ks_]

        def run():
            o_state = torch.empty(rows, Hq, D, dtype=torch.float32, device=dev)
            lse = torch.empty(rows, Hq, dtype=torch.float32, device=dev)
            for i, (k, v) in enumerate(zip(blocks, vals)):
                fwd(q, k, v, causal=i == len(blocks) - 1, o_state=o_state, lse=lse, has_prev=i > 0)
            return o_state, lse

        o_state, lse = _twice(run)
        pos = torch.arange(rows, device=dev)
        keep = torch.cat([torch.ones(rows, rows * (len(blocks) - 1), dtype=torch.bool, device=dev),
                          visible(pos, pos, True)], 1)
        ref, lref, fo, fl = attn64(q, torch.cat(blocks), torch.cat(vals), D ** -0.5, keep, dtype=dtype)
        fo = fo + len(blocks) * 8 * U * ref.abs()                                   # per-launch merge roundings
        check(f"block_ostate.{_NAME[dtype]} scale={ks_[1]}", o_state, ref, torch.float32, floor=fo,
              signed_mean=ref.shape[-1])
        check(f"block_lse.{_NAME[dtype]} scale={ks_[1]}", lse, lref, torch.float32, floor=fl + 4 * U * len(blocks))


# ============================================================================================ backward
def _bwd_operands(T, Hq, Hkv, D, dtype, dev, gen):
    c = torch.rand(T, 1, 1, generator=gen) + 0.5
    v = (c + 0.05 * torch.randn(T, Hkv, D, generator=gen)).to(dev, dtype)
    sign = 1.0 - 2.0 * (torch.arange(D) % 2)                                    # +1, -1, ... over the head dim
    k = ((c - 1) * sign + 0.05 * torch.randn(T, Hkv, D, generator=gen)).to(dev, dtype)
    q = (torch.rand(T, Hq, D, generator=gen) + 0.5).to(dev, dtype)
    do = (torch.rand(T, Hq, D, generator=gen) + 0.5).to(dev, dtype)
    return q, k, v, do


def bwd64(q, k, v, out, do, lse, keep, scale, dtype, key_tiles=None):
    """float64 gradients from the saved (out, lse), and their Tier B floors."""
    q, k, v, out, do = (t.double() for t in (q, k, v, out, do))
    lse = lse.double()
    S, Hq, D = q.shape
    Hkv = k.shape[1]
    G = Hq // Hkv
    uP, sub = U_P[dtype], SUB_P[dtype]
    dq, dk, dv = torch.zeros_like(q), torch.zeros_like(k), torch.zeros_like(v)
    fdq, fdk, fdv = torch.zeros_like(q), torch.zeros_like(k), torch.zeros_like(v)
    q_steps = G * -(-S // 64) * 4                      # k16 steps of dV / dK over the group's query tiles
    k_tiles = -(-k.shape[0] // 128) if key_tiles is None else key_tiles      # fp32 atomic adds into dQ
    kf = keep.double()
    for h in range(Hq):
        kh, vh = k[:, h // G], v[:, h // G]
        x = (q[:, h] @ kh.t()) * (scale * LOG2E) - lse[:, h:h + 1] * LOG2E
        x = x.masked_fill(~keep, float("-inf"))
        p = torch.exp2(x)
        xf = torch.where(keep, x, torch.zeros_like(x))
        a = (q[:, h].abs() @ kh.abs().t()) * scale
        eta = a * (D / 16) * G16 + LN2 * U * (4 * xf.abs() + 2 * (lse[:, h:h + 1] * LOG2E).abs()) + EX2
        eta = eta * kf
        dp = do[:, h] @ vh.t()
        e_dp = (D / 16) * G16 * (do[:, h].abs() @ vh.abs().t())
        delta = (do[:, h] * out[:, h]).sum(-1, keepdim=True)
        e_delta = (D / 8 + 5) * U * (do[:, h].abs() * out[:, h].abs()).sum(-1, keepdim=True)
        ds = p * (dp - delta)
        e_ds = p * (e_dp + e_delta) + eta * ds.abs() + uP * ds.abs() + sub * kf
        dvh = p.t() @ do[:, h]
        fdv[:, h // G] += (uP * p + eta * p + sub * kf).t() @ do[:, h].abs() + q_steps * G16 * (p.t() @ do[:, h].abs())
        dv[:, h // G] += dvh
        dk[:, h // G] += scale * (ds.t() @ q[:, h])
        fdk[:, h // G] += scale * (e_ds.t() @ q[:, h].abs() + q_steps * G16 * (ds.abs().t() @ q[:, h].abs()))
        dq[:, h] = scale * (ds @ kh)
        sk = ds.abs() @ kh.abs()
        fdq[:, h] = scale * (e_ds @ kh.abs() + 8 * G16 * sk + (k_tiles + 1) * U * sk)
    return (dq, dk, dv), (fdq, fdk + 2 * U * dk.abs(), fdv + 2 * U * dv.abs())


@pytest.mark.gpu
@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("causal", [False, True])
@pytest.mark.parametrize("packed", [False, True])
def test_bwd_random(dtype, causal, packed):
    """Lengths 1, 64, 65, 127, 128, 129 (packed: with empty sequences between them); G 1, 2, 16."""
    dev = _cuda()
    fa = _fa()
    gen = torch.Generator().manual_seed(23 + causal + 2 * packed)
    D = 128
    for G, Hkv in [(1, 2), (2, 2), (16, 1)]:
        Hq = G * Hkv
        if packed:
            lens = [1, 0, 64, 65, 0, 127, 128, 129, 0]
        else:
            lens = [129, 129]
        T = sum(lens)
        q, k, v, do = _bwd_operands(T, Hq, Hkv, D, dtype, dev, gen)
        cu = _cu(lens, dev) if packed else None
        out, lse = fwd(q, k, v, causal=causal, cu=cu, batch=1 if packed else 2)

        def run():
            r = fa.flash_bwd(q, k, v, out, do, lse, 1 if packed else 2, causal, D ** -0.5, cu_seqlens=cu)
            torch.cuda.synchronize()
            return None, r[1], r[2]

        _, dk, dv = _twice(run)
        dq = fa.flash_bwd(q, k, v, out, do, lse, 1 if packed else 2, causal, D ** -0.5, cu_seqlens=cu)[0]
        delta = fa.flash_delta(out, do)
        d64 = (do.double() * out.double()).sum(-1)
        check(f"flash_delta.{_NAME[dtype]} G={G}", delta, d64, torch.float32,
              floor=(D / 8 + 5) * U * (do.double().abs() * out.double().abs()).sum(-1))
        for a, b in _segments(lens):
            if a == b:
                continue
            pos = torch.arange(b - a, device=dev)
            (rq, rk, rv), (fq, fk, fv) = bwd64(q[a:b], k[a:b], v[a:b], out[a:b], do[a:b], lse[a:b],
                                               visible(pos, pos, causal), D ** -0.5, dtype)
            tag = f"G={G} causal={causal} len={b - a}"
            check(f"bwd_dv.{_NAME[dtype]} {tag}", dv[a:b], rv, dtype, floor=fv)
            check(f"bwd_dk.{_NAME[dtype]} {tag}", dk[a:b], rk, dtype, floor=fk)
            check(f"bwd_dq.{_NAME[dtype]} {tag}", dq[a:b], rq, dtype, floor=fq)


@pytest.mark.gpu
@pytest.mark.parametrize("dtype", DTYPES)
def test_block_bwd_chain(dtype):
    """cb_flash_attn_block_bwd over 3 key blocks (causal last), given the merged forward's lse: the fp32
    accumulators equal the float64 gradients of attention over the concatenated keys."""
    dev = _cuda()
    fa = _fa()
    gen = torch.Generator().manual_seed(29)
    rows, Hq, Hkv, D = 200, 4, 2, 128
    q, _, _, do = _bwd_operands(rows, Hq, Hkv, D, dtype, dev, gen)
    blocks = [_bwd_operands(rows, Hq, Hkv, D, dtype, dev, gen)[1:3] for _ in range(3)]
    o_state = torch.empty(rows, Hq, D, dtype=torch.float32, device=dev)
    lse = torch.empty(rows, Hq, dtype=torch.float32, device=dev)
    for i, (k, v) in enumerate(blocks):
        fwd(q, k, v, causal=i == 2, o_state=o_state, lse=lse, has_prev=i > 0)
    out = o_state.to(dtype)
    delta = fa.flash_delta(out, do)
    dq_acc = torch.zeros(rows, Hq, D, dtype=torch.float32, device=dev)
    grads = []
    for i, (k, v) in enumerate(blocks):
        dk_acc = torch.zeros(rows, Hkv, D, dtype=torch.float32, device=dev)
        dv_acc = torch.zeros_like(dk_acc)
        fa.flash_block_bwd(q.data_ptr(), k.data_ptr(), v.data_ptr(), do.data_ptr(), lse.data_ptr(), delta.data_ptr(),
                           dq_acc.data_ptr(), dk_acc.data_ptr(), dv_acc.data_ptr(), rows, Hq, Hkv, D, i == 2,
                           D ** -0.5, dtype)
        grads.append((dk_acc, dv_acc))
    torch.cuda.synchronize()
    pos = torch.arange(rows, device=dev)
    keep = torch.cat([torch.ones(rows, 2 * rows, dtype=torch.bool, device=dev), visible(pos, pos, True)], 1)
    kc = torch.cat([b[0] for b in blocks])
    vc = torch.cat([b[1] for b in blocks])
    (rq, rk, rv), (fq, fk, fv) = bwd64(q, kc, vc, out, do, lse, keep, D ** -0.5, dtype, key_tiles=3 * 2)
    check(f"block_bwd_dq.{_NAME[dtype]}", dq_acc, rq, torch.float32, floor=fq)
    for i, (dk_acc, dv_acc) in enumerate(grads):
        sl = slice(i * rows, (i + 1) * rows)
        check(f"block_bwd_dk.{_NAME[dtype]} block={i}", dk_acc, rk[sl], torch.float32, floor=fk[sl])
        check(f"block_bwd_dv.{_NAME[dtype]} block={i}", dv_acc, rv[sl], torch.float32, floor=fv[sl])


# ============================================================================================ decode / verify
def decode(q, kc, vc, tables, lens, *, q_len, splits, part_len, window=0, slopes=None, out=None, q_stride=None):
    """cb_paged_decode_attention with our own partials; returns (out, o_part, ml_part)."""
    from colossalai_b200.kernel import loader
    from colossalai_b200.ops import inference as iops
    from colossalai_b200.ops._dtypes import code

    rows, Hq, D = q.shape
    n = lens.numel()
    Hkv = kc.shape[2]
    out = torch.full((rows, Hq, D), float("nan"), dtype=q.dtype, device=q.device) if out is None else out
    o_part = torch.full((rows, Hq, splits, D), float("nan"), device=q.device)
    ml_part = torch.full((rows, Hq, splits, 2), float("nan"), device=q.device)
    rc = iops._get_lib().cb_paged_decode_attention(
        loader.ptr(q), loader.ptr(kc), loader.ptr(vc), loader.ptr(tables), loader.ptr(lens), loader.ptr(out),
        loader.ptr(o_part), loader.ptr(ml_part), n, q_len, Hq, Hkv, D, kc.shape[1], tables.shape[1], splits,
        part_len, ctypes.c_float(D ** -0.5), loader.ptr(slopes), ctypes.c_int64(q.stride(0) if q_stride is None
                                                                               else q_stride),
        ctypes.c_int64(out.stride(0)), code(q.dtype), iops._cache_code(kc), int(window), loader.stream_ptr())
    torch.cuda.synchronize()
    assert rc == 0, rc
    return out, o_part, ml_part


def _decode_cache(lens, bs, Hkv, D, dtype, dev, gen, kind):
    """kind 'int': K random, V integers; 'rand': V in [0.5, 1.5].  NaN in unreferenced blocks and the last block's
    tail slots, -1 past each table's last block."""
    def kv(L):
        k = torch.randn(L, Hkv, D, generator=gen).to(dev, dtype)
        v = _int_v((L, Hkv, D), dev, gen).to(dtype) if kind == "int" else \
            (torch.rand(L, Hkv, D, generator=gen) + 0.5).to(dev, dtype)
        return k, v
    return _paged_case([max(L, 1) for L in lens], None, bs, Hkv, D, dtype, dev, gen, kv, tail=float("nan"))


def _decode_rows(lens, q_len):
    """(sequence, query token, len_j) per output row."""
    return [(i, j, L - (q_len - 1 - j)) for i, L in enumerate(lens) for j in range(q_len)]


DECODE_CASES = [
    # D, G, q_len, bs, part_len, window
    (128, 1, 1, 64, 96, 0),
    (128, 3, 1, 128, 160, 0),
    (64, 5, 3, 64, 96, 0),
    (64, 6, 7, 16, 64, 0),
    (128, 7, 2, 64, 96, 96),
    (128, 8, 16, 128, 224, 1),
    (64, 2, 11, 32, 128, 0),
    (128, 4, 4, 64, 96, 5000),
    (256, 1, 1, 16, 96, 0),
    (256, 6, 1, 64, 96, 96),
    (256, 8, 1, 32, 64, 1),
]


def _decode_lens(part_len, q_len):
    mx = 4 * part_len + 5
    return [0, 1 + q_len - 1, part_len - 1, part_len, part_len + 1, 2 * part_len + 17, mx]


@pytest.mark.gpu
@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("case", DECODE_CASES, ids=lambda c: "D{}-G{}-q{}-bs{}-P{}-w{}".format(*c))
@pytest.mark.parametrize("fp8", [False, True])
def test_decode_counting(dtype, case, fp8):
    """Tier A: per (row, head, split) counts in ml_part; the reduced output; a length-0 slot gives exactly 0."""
    D, G, q_len, bs, part_len, window = case
    dev = _cuda()
    gen = torch.Generator().manual_seed(D + G + q_len + bs)
    Hkv = 2
    lens = _decode_lens(part_len, q_len)
    splits = -(-max(lens) // part_len)
    kc, vc, tables, _, ks, vs = _decode_cache(lens, bs, Hkv, D, dtype, dev, gen, "int")
    if fp8:
        kc, vc = kc.to(torch.float8_e5m2).view(torch.uint8), vc.to(torch.float8_e5m2).view(torch.uint8)
    lt = torch.tensor(lens, dtype=torch.int32, device=dev)
    q = torch.zeros(len(lens) * q_len, Hkv * G, D, dtype=dtype, device=dev)
    out, _, ml = decode(q, kc, vc, tables, lt, q_len=q_len, splits=splits, part_len=part_len, window=window)
    for r, (i, j, Lj) in enumerate(_decode_rows(lens, q_len)):
        ws = max(0, Lj - window) if window else 0
        want_l = torch.tensor([max(0, min(Lj, (s + 1) * part_len) - max(s * part_len, ws)) for s in range(splits)],
                              dtype=torch.float64, device=dev)
        m, l = ml[r, :, :, 0].double(), ml[r, :, :, 1].double()
        empty = want_l == 0
        assert torch.equal(l, want_l[None].expand_as(l)), \
            f"row {r} (len_j {Lj}): l {l[0].tolist()} want {want_l.tolist()}"
        assert (m[:, empty] == float("-inf")).all() and (m[:, ~empty] == 0).all(), f"row {r}: m {m[0].tolist()}"
        if Lj <= 0:
            assert (out[r] == 0).all(), f"row {r}: a slot without keys must give exactly 0"
            continue
        vv = vs[i].double() if not fp8 else vs[i].to(torch.float8_e5m2).double()
        mean = vv[ws:Lj].mean(0).repeat_interleave(G, 0)
        check_count_out(f"decode_out.{_NAME[dtype]} D={D} row={r}", out[r].float(), mean, dtype)


def _decode_ref(q, vs, ks, lens, q_len, window, slopes, dtype, fp8):
    """float64 reference and floors of every decode row."""
    refs, floors = [], []
    Hq, D = q.shape[1], q.shape[2]
    for r, (i, j, Lj) in enumerate(_decode_rows(lens, q_len)):
        L = lens[i]
        k, v = ks[i], vs[i]
        if fp8:
            k, v = k.to(torch.float8_e5m2), v.to(torch.float8_e5m2)
        keep = visible(torch.tensor([Lj - 1], device=q.device), torch.arange(k.shape[0], device=q.device), True,
                       window) & (torch.arange(k.shape[0], device=q.device) < max(Lj, 0))[None]
        if Lj <= 0:
            refs.append(torch.zeros(Hq, D, dtype=torch.float64, device=q.device))
            floors.append(torch.zeros(Hq, D, dtype=torch.float64, device=q.device))
            continue
        pos_k = torch.arange(k.shape[0], device=q.device)
        o, _, fo, _ = attn64(q[r:r + 1], k, v, D ** -0.5, keep, slopes, torch.tensor([Lj - 1], device=q.device),
                             pos_k, dtype=dtype)
        refs.append(o[0])
        floors.append(fo[0] + 8 * U * o[0].abs())          # split merge: __expf weights cancel, 8 fp32 roundings
    return torch.stack(refs), torch.stack(floors)


@pytest.mark.gpu
@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("case", DECODE_CASES, ids=lambda c: "D{}-G{}-q{}-bs{}-P{}-w{}".format(*c))
def test_decode_random(dtype, case):
    """Tier B for decode and verify, ALiBi on every other case, strided q / out; repeat bitwise; each verify row
    equals the single-token decode of that row (no window); the fp8 cache equals its decoded 16-bit cache."""
    D, G, q_len, bs, part_len, window = case
    dev = _cuda()
    gen = torch.Generator().manual_seed(31 + D + G + q_len)
    Hkv = 2
    Hq = Hkv * G
    lens = _decode_lens(part_len, q_len)
    splits = -(-max(lens) // part_len)
    kc, vc, tables, _, ks, vs = _decode_cache(lens, bs, Hkv, D, dtype, dev, gen, "rand")
    lt = torch.tensor(lens, dtype=torch.int32, device=dev)
    rows = len(lens) * q_len
    qbuf = torch.randn(rows, Hq + 1, D, generator=gen).to(dev, dtype)     # q_stride = (Hq + 1) * D
    q = qbuf[:, :Hq]
    obuf = torch.full((rows, Hq + 2, D), 7.0, dtype=dtype, device=dev)
    slopes = torch.tensor([2 ** (-(h + 1) / 2) for h in range(Hq)], dtype=torch.float32, device=dev) \
        if G % 2 == 1 else None
    kw = dict(q_len=q_len, splits=splits, part_len=part_len, window=window, slopes=slopes)

    def run():
        o = obuf.clone()
        decode(q, kc, vc, tables, lt, out=o[:, :Hq], **kw)
        return (o,)

    (o,) = _twice(run)
    assert (o[:, Hq:] == 7).all(), "columns past Hq * D of a strided output were written"
    got = o[:, :Hq]
    ref, floor = _decode_ref(q, vs, ks, lens, q_len, window, slopes, dtype, False)
    live = torch.tensor([Lj > 0 for _, _, Lj in _decode_rows(lens, q_len)], device=dev)
    assert (got[~live] == 0).all(), "a row without keys must give exactly 0"
    check(f"decode_out.{_NAME[dtype]} D={D} G={G} q_len={q_len}", got[live], ref[live], dtype, floor=floor[live],
          signed_mean=ref.shape[-1])
    if q_len > 1 and not window:
        n = len(lens)
        for j in range(q_len):
            single = decode(q.view(n, q_len, Hq, D)[:, j], kc, vc, tables, lt - (q_len - 1 - j),
                            **dict(kw, q_len=1))[0]
            check_bitwise(f"verify row j={j} == decode", got.view(n, q_len, Hq, D)[:, j], single)
    k8, v8 = kc.to(torch.float8_e5m2), vc.to(torch.float8_e5m2)
    o8 = decode(q, k8.view(torch.uint8), v8.view(torch.uint8), tables, lt, **kw)[0]
    o16 = decode(q, k8.to(dtype), v8.to(dtype), tables, lt, **kw)[0]
    check_bitwise("fp8 cache == decoded 16-bit cache", o8, o16)


# ============================================================================================ locality
def _poison(t, rows, vals=(float("nan"), float("inf"), float("-inf"))):
    t = t.clone()
    for i, r in enumerate(rows):
        t[r] = vals[i % len(vals)]
    return t


@pytest.mark.gpu
@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("D", [64, 128])
def test_fwd_sequences_do_not_see_each_other(dtype, D):
    """NaN / +Inf / -Inf in the q, k and v rows of one sequence (packed), one batch entry (uniform, causal and not),
    and a paged sequence's last-block tail slots: every other sequence's out and lse are those of a clean run, bit
    for bit."""
    dev = _cuda()
    gen = torch.Generator().manual_seed(37 + D)
    Hq, Hkv = 4, 2
    lens = [100, 77, 300, 129]
    T = sum(lens)
    q, k, v = _rand_qkv(T, T, Hq, Hkv, D, dtype, dev, gen)
    cu = _cu(lens, dev)
    segs = list(_segments(lens))
    for victim in range(1, len(lens)):
        a, b = segs[victim]
        rows = list(range(a, min(b, a + 9)))
        for causal in (False, True):
            clean = fwd(q, k, v, causal=causal, cu=cu)
            dirty = fwd(_poison(q, rows), _poison(k, rows), _poison(v, rows), causal=causal, cu=cu)
            for s, (x, y) in enumerate(segs):
                if s != victim:
                    check_bitwise(f"packed out seq {s} (poisoned {victim}, causal={causal})", dirty[0][x:y],
                                  clean[0][x:y])
                    check_bitwise(f"packed lse seq {s} (poisoned {victim})", dirty[1][x:y], clean[1][x:y])
    S, B = 200, 3
    q, k, v = _rand_qkv(B * S, B * S, Hq, Hkv, D, dtype, dev, gen)
    rows = list(range(S, S + 9))                                                  # batch entry 1
    for causal in (False, True):
        clean = fwd(q, k, v, causal=causal, batch=B)
        dirty = fwd(_poison(q, rows), _poison(k, rows), _poison(v, rows), causal=causal, batch=B)
        for bb in (0, 2):
            sl = slice(bb * S, (bb + 1) * S)
            check_bitwise(f"uniform out entry {bb} (causal={causal})", dirty[0][sl], clean[0][sl])
            check_bitwise(f"uniform lse entry {bb} (causal={causal})", dirty[1][sl], clean[1][sl])
    bs, new = 64, [30, 50]
    lens_k = [100, 150]                                                            # not block multiples
    kv = lambda L: (torch.randn(L, Hkv, D, generator=gen).to(dev, dtype),
                    (torch.rand(L, Hkv, D, generator=gen) + 0.5).to(dev, dtype))
    st = torch.random.get_rng_state()
    g_state = gen.get_state()
    kc0, vc0, tables, lk, _, _ = _paged_case(lens_k, new, bs, Hkv, D, dtype, dev, gen, kv, tail=0.0)
    gen.set_state(g_state)
    kc1, vc1, tables1, _, _, _ = _paged_case(lens_k, new, bs, Hkv, D, dtype, dev, gen, kv, tail=float("nan"))
    torch.random.set_rng_state(st)
    assert torch.equal(tables, tables1)
    qn = torch.randn(sum(new), Hq, D, generator=gen).to(dev, dtype)
    clean = fwd(qn, kc0, vc0, causal=True, cu=_cu(new, dev), paged=(tables, lk))
    dirty = fwd(qn, kc1, vc1, causal=True, cu=_cu(new, dev), paged=(tables, lk))
    check_bitwise("paged out with NaN tail slots", dirty[0], clean[0])
    check_bitwise("paged lse with NaN tail slots", dirty[1], clean[1])


@pytest.mark.gpu
@pytest.mark.xfail(strict=True, reason="the backward's ragged tiles multiply P = 0 / dS = 0 by the next sequence's "
                                       "q / k / dout rows; see cb_flash_attn_bwd")
def test_bwd_sequences_do_not_see_each_other():
    dev = _cuda()
    fa = _fa()
    gen = torch.Generator().manual_seed(41)
    dtype, D, Hq, Hkv = BF16, 128, 4, 2
    lens = [100, 77, 300]
    T = sum(lens)
    q, k, v, do = _bwd_operands(T, Hq, Hkv, D, dtype, dev, gen)
    cu = _cu(lens, dev)
    out, lse = fwd(q, k, v, causal=True, cu=cu)
    clean = fa.flash_bwd(q, k, v, out, do, lse, 1, True, D ** -0.5, cu_seqlens=cu)
    rows = list(range(100, 109))
    dirty = fa.flash_bwd(_poison(q, rows), _poison(k, rows), _poison(v, rows), out, _poison(do, rows), lse, 1, True,
                         D ** -0.5, cu_seqlens=cu)
    torch.cuda.synchronize()
    for name, c, d in zip(("dq", "dk", "dv"), clean, dirty):
        assert torch.isfinite(d[:100].float()).all(), f"{name} of sequence 0 took the next sequence's NaN / Inf"
        assert torch.isfinite(d[177:].float()).all(), f"{name} of sequence 2"


# ============================================================================================ CPU self-test
def _rejects(fn):
    try:
        fn()
    except AssertionError:
        return True
    return False


def test_comparators_reject_simulated_faults():
    """Ten kernel faults simulated in float64 on the CPU, at the GPU tests' shapes: the checks above reject each."""
    torch.manual_seed(0)
    dt = BF16
    found = {}

    # Tier A decode: the counts of every split; the newest token dropped at context 4000, a key dropped at a split
    # boundary (part_len 96)
    def counts(L, part, splits, drop_newest=False, drop_at=None):
        c = []
        for s in range(splits):
            lo, hi = s * part, min(L - (1 if drop_newest else 0), (s + 1) * part)
            n = max(0, hi - lo)
            if drop_at is not None and lo == drop_at:
                n -= 1
            c.append(float(n))
        return torch.tensor(c, dtype=torch.float64)

    splits = -(-4000 // 96)
    good = counts(4000, 96, splits)
    found[1] = not torch.equal(counts(4000, 96, splits, drop_newest=True), good)
    found[2] = not torch.equal(counts(4000, 96, splits, drop_at=96 * 7), good)
    # the l counts drive the output too: dropping the newest integer V moves O by up to 8 / 4000
    v = torch.randint(-4, 5, (4000, 128)).double()
    mean, mean_bad = v.mean(0), v[:-1].mean(0)
    found[1] &= _rejects(lambda: check_count_out("sim", mean_bad.to(dt).float(), mean, dt)) or found[1]

    # Tier A forward: the last key dropped at S = 4096 (non-causal), the window one too wide, a key of the next
    # packed sequence visible: lse must be ln(n)
    n = torch.full((4096,), 4096.0, dtype=torch.float64)
    found[3] = _rejects(lambda: check_exact_f32("sim", (n - 1).log().float(), n.log(), 2.0 ** -21, 2.0 ** -22))
    pos = torch.arange(700)
    nw = visible(pos, pos, True, 129).double().sum(-1)
    nw_bad = visible(pos, pos, True, 130).double().sum(-1)
    found[4] = _rejects(lambda: check_exact_f32("sim", nw_bad.log().float(), nw.log(), 2.0 ** -21, 2.0 ** -22))
    npk = torch.arange(1, 130, dtype=torch.float64)
    found[10] = _rejects(lambda: check_exact_f32("sim", (npk + 1).log().float(), npk.log(), 2.0 ** -21, 2.0 ** -22))

    # Tier B: ALiBi slopes 1% too large, packed prefill S = 1000, 8 heads
    S, H, D = 1000, 8, 128
    q, k = torch.randn(S, H, D).to(dt), torch.randn(S, 2, D).to(dt)
    vv = (torch.rand(S, 2, D) + 0.5).to(dt)
    sl = torch.tensor([2 ** (-(h + 1) / 2) for h in range(H)], dtype=torch.float64)
    pos = torch.arange(S)
    keep = visible(pos, pos, True)
    ref, lref, fo, fl = attn64(q, k, vv, D ** -0.5, keep, sl, pos, pos, dtype=dt)
    bad, lbad, _, _ = attn64(q, k, vv, D ** -0.5, keep, sl * 1.01, pos, pos, bounds=False, dtype=dt)
    found[5] = _rejects(lambda: _check_b("sim", dt, bad.to(dt), lbad.float(), ref, fo, lref, fl, S))
    assert not _rejects(lambda: _check_b("sim", dt, ref.to(dt), lref.float(), ref, fo, lref, fl, S))

    # Tier B: the alpha rescale skipped when the max grows (large scores, 129 x 4096): tiles accumulated with their
    # own max and never rescaled
    q, k = (torch.randn(129, 1, D) * 12).to(dt), torch.randn(4096, 1, D).to(dt)
    vv = (torch.rand(4096, 1, D) + 0.5).to(dt)
    keep = torch.ones(129, 4096, dtype=torch.bool)
    ref, lref, fo, fl = attn64(q, k, vv, D ** -0.5, keep, dtype=dt)
    x = (q[:, 0].double() @ k[:, 0].double().t()) * D ** -0.5
    o, l, m = torch.zeros(129, D, dtype=torch.float64), torch.zeros(129, 1, dtype=torch.float64), None
    for t in range(32):
        xt = x[:, 128 * t:128 * (t + 1)]
        m = xt.amax(-1, keepdim=True) if m is None else torch.maximum(m, xt.amax(-1, keepdim=True))
        e = torch.exp(xt - m)
        o, l = o + e @ vv[128 * t:128 * (t + 1), 0].double(), l + e.sum(-1, keepdim=True)
    found[6] = _rejects(lambda: _check_b("sim", dt, (o / l)[:, None].to(dt), None, ref, fo, lref, fl, 4096))

    # Tier B: P rounded toward zero before the P V MMA (S = 4096 causal, one head): within the elementwise floor but
    # caught by the signed mean
    S = 4096
    q, k = torch.randn(S, 1, 64).to(dt), torch.randn(S, 1, 64).to(dt)
    vv = (torch.rand(S, 1, 64) + 0.5).to(dt)
    pos = torch.arange(S)
    keep = visible(pos, pos, True)
    ref, lref, fo, fl = attn64(q, k, vv, 64 ** -0.5, keep, dtype=dt)
    x = ((q[:, 0].double() @ k[:, 0].double().t()) * 64 ** -0.5).masked_fill(~keep, float("-inf"))
    p = torch.exp(x - x.amax(-1, keepdim=True))
    pr = p.to(dt).double()
    pr = torch.where(pr > p, torch.nextafter(pr.to(dt), torch.zeros((), dtype=dt)).double(), pr)   # toward zero
    o_tz = (pr @ vv[:, 0].double()) / p.sum(-1, keepdim=True)
    found[7] = _rejects(lambda: _check_b("sim", dt, o_tz[:, None].to(dt), None, ref, fo, lref, fl, S))
    assert not _rejects(lambda: _check_b("sim", dt, ref.to(dt), None, ref, fo, lref, fl, S))

    # backward: dK / dV summing only the first head of a GQA group (G = 2); dQ missing the ragged last key tile (129)
    S = 129
    gen = torch.Generator().manual_seed(1)
    q, k, v, do = (t.cpu() for t in _bwd_operands(S, 4, 2, 128, dt, "cpu", gen))
    pos = torch.arange(S)
    keep = visible(pos, pos, True)
    out, lse, _, _ = attn64(q, k, v, 128 ** -0.5, keep, bounds=False, dtype=dt)
    out = out.to(dt)
    (rq, rk, rv), (fq, fk, fv) = bwd64(q, k, v, out, do, lse.float(), keep, 128 ** -0.5, dt)
    assert not _rejects(lambda: check("sim", rv.to(dt), rv, dt, floor=fv))
    assert not _rejects(lambda: check("sim", rk.to(dt), rk, dt, floor=fk))
    assert not _rejects(lambda: check("sim", rq.to(dt), rq, dt, floor=fq))
    k1 = keep.clone()
    (_, bk, bv), _ = bwd64(q[:, ::2].contiguous(), k, v, out[:, ::2].contiguous(), do[:, ::2].contiguous(),
                           lse[:, ::2].contiguous().float(), k1, 128 ** -0.5, dt)
    found[8] = _rejects(lambda: check("sim", bv.to(dt), rv, dt, floor=fv)) and \
        _rejects(lambda: check("sim", bk.to(dt), rk, dt, floor=fk))
    k2 = keep.clone()
    k2[:, 128:] = False
    (bq, _, _), _ = bwd64(q, k, v, out, do, lse.float(), k2, 128 ** -0.5, dt)
    found[9] = _rejects(lambda: check("sim", bq.to(dt), rq, dt, floor=fq))

    missed = [i for i in range(1, 11) if not found.get(i)]
    assert not missed, f"simulated faults not rejected: {missed}"
