"""The dense, fp8 and grouped wgmma GEMMs (`gemm_sm90.cuh`) against float64 references.

Every reference is a float64 matmul on the GPU of the exact operand values the kernel read (never an fp32
`torch.matmul`, whose use of TF32 depends on global settings).  Two tiers:

Tier A - exact integers.  16-bit operands are integers in [-8, 8] with |sums| < 2^24; e4m3 / e5m2 operands are
integers in [-4, 4], so a 128-deep fp8 stage sums to less than 128 * 16 = 2^11 and is exact even in a reduced-precision
accumulator.  fp8 scales are powers of two, accumulated C values are integers.  Every product and partial sum is then
exact, whatever order the tensor core adds in, and the output must equal `ref.to(out_dtype)` bit for bit.  This tier
carries the structural claims: tiles, k-blocks, operand layouts, masks, groups and epilogue order.

Tier B - random operands, derived bound.  Each element is checked against

    |got - ref| <= k * ulp_out(|ref|) + gamma * S,      S = |A| x |B|^T  (float64, per element)

with k = 1 for the single rounding to the output dtype.  gamma follows the accumulation order of the code:
  * 16-bit: K is walked in k16 `wgmma` steps into one fp32 accumulator.  The tensor core aligns the addends of a step
    to the largest exponent and truncates, so each step is budgeted at G16 = 2^-22 of the running sum of |a * b|,
    giving gamma = ceil(K / 16) * 2^-22.
  * fp8: each 128-deep stage is summed by four k32 instructions into a fresh partial whose accumulator keeps about
    14 bits (the figure published for Hopper fp8 accumulation), i.e. 2^-13 of the stage's sum of |a * b| per
    instruction, and the partial is then added to the fp32 accumulator (2^-24 of the running sum per stage):
    gamma = 4 * 2^-13 + ceil(K / 128) * 2^-24, plus 2^-23 for the fp32 product of the scales and its multiply.
  * `accumulate` adds one fp32 add: 2^-24 * (S + |C|).
Neither per-step figure is measured here; the largest error-to-tolerance ratio per kernel and output dtype is printed
at module teardown so the constants can be argued from measurement.  The comparator refuses a floor above 1% of the
median |ref|; where the floor would be larger (random signs with K far beyond 4096, random-sign fp8), the operands are
same-sign (S = |ref|) instead.  An element whose reference is exactly zero with every term zero must be exactly zero.

Every Tier B case runs twice and the two results must be bitwise identical: there are no atomics or split-K, so any
difference is a race in the mbarrier ring.

Kernel constants (gemm_sm90.cuh): 128 x 128 tiles, 64 (16-bit) or 128 (fp8) K elements per stage, STAGES = 6, tiles
rasterised in bands of GROUP_M = 8 row blocks, grid = min(tiles, SMs) persistent CTAs (grouped: always SMs).
"""
import ctypes
import math

import pytest
import torch

U = 2.0 ** -24
G16 = 2.0 ** -22                      # per k16 wgmma step, of the running sum of |a * b|
G8 = 2.0 ** -13                       # per k32 fp8 instruction into a ~14-bit partial, of the stage's sum of |a * b|
BM = BN = 128
KE16, KE8, STAGES, GROUP_M = 64, 128, 6, 8
MAX_GROUPS = 512
INVALID = 1                           # cudaErrorInvalidValue
F32, BF16, F16 = torch.float32, torch.bfloat16, torch.float16
E4M3, E5M2 = torch.float8_e4m3fn, torch.float8_e5m2
CODE = {F32: 0, F16: 1, BF16: 2, E4M3: 3, E5M2: 4}
FMT = {E4M3: 0, E5M2: 1}
_MANT = {BF16: 8, F16: 11, F32: 24}
_MIN_STEP = {BF16: 2.0 ** -133, F16: 2.0 ** -24, F32: 2.0 ** -149}
_NAME = {F32: "f32", BF16: "bf16", F16: "f16"}
_F8NAME = {E4M3: "e4m3", E5M2: "e5m2"}
_WORST = {}                           # "kernel.out_dtype" -> largest |err| / tol seen


# ============================================================================================ comparators
def ulp(ref: torch.Tensor, dtype: torch.dtype) -> torch.Tensor:
    """Spacing of `dtype` at |ref| (never below its subnormal step)."""
    _, e = torch.frexp(ref.abs().double())
    return torch.ldexp(torch.ones_like(ref, dtype=torch.float64), e - _MANT[dtype]).clamp_min(_MIN_STEP[dtype])


def check(what, got, ref, dtype, k=1.0, floor=0.0):
    """Tier B: |got - ref| <= k * ulp(|ref|) + floor elementwise."""
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


def _bits(t):
    return t.contiguous().view({4: torch.int32, 2: torch.int16, 1: torch.int8}[t.element_size()])


def check_bitwise(what, got, want):
    """Tier A: `got` must be `want` bit for bit (NaN patterns included)."""
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
        print("\nlargest error-to-tolerance ratio per kernel and output dtype:")
        for k, v in sorted(_WORST.items()):
            print(f"  {k:<24} {v:.3f}")
    if torch.cuda.is_available() and torch.cuda.is_initialized():
        print(f"peak CUDA memory allocated: {torch.cuda.max_memory_allocated() / 2**30:.2f} GiB")


# ============================================================================================ operands
def values(kind, shape, dtype, gen, device):
    """'int': exact integers (Tier A); 'rand': N(0, 1); 'pos': same-sign in [0.5, 1)."""
    lim = 4 if dtype in (E4M3, E5M2) else 8
    if kind == "int":
        v = torch.randint(-lim, lim + 1, shape, generator=gen, device="cpu").float()
    elif kind == "rand":
        v = torch.randn(shape, generator=gen, device="cpu")
    else:
        v = torch.rand(shape, generator=gen, device="cpu") * 0.5 + 0.5
    return v.to(device).to(dtype)


def operand(kind, rows, K, dtype, mn_major, gen, device, pad=0):
    """Logical [rows, K] operand.  K-major: stored [rows, ld >= K]; MN-major: stored [K, ld >= rows].  The storage
    beyond the logical extent is NaN (16-bit) and must never be read.  Returns (storage, logical view, ld)."""
    v = values(kind, (rows, K), dtype, gen, device)
    inner = K if not mn_major else rows
    align = 16 if dtype in (E4M3, E5M2) else 8
    ld = (inner + align - 1) // align * align + pad
    outer = rows if not mn_major else K
    if dtype in (E4M3, E5M2):
        st = torch.full((outer, ld), float("nan"), device=device).to(dtype)
    else:
        st = torch.full((outer, ld), float("nan"), dtype=dtype, device=device)
    if mn_major:
        st[:, :rows] = v.t()
        return st, st[:, :rows].t(), ld
    st[:, :K] = v
    return st, st[:, :K], ld


def ref_and_s(a, b):
    """float64 a @ b^T and |a| @ |b|^T on the GPU."""
    a, b = a.double(), b.double()
    return a @ b.t(), a.abs() @ b.abs().t()


def out_buffer(M, N, dtype, ldc, device):
    """A NaN-filled [M + 1, ldc] buffer and its [M, N] window (the row and the columns outside must stay NaN)."""
    buf = torch.full((M + 1, ldc), float("nan"), dtype=dtype, device=device)
    return buf, buf[:M, :N]


def assert_outside_untouched(what, buf, before, M, N):
    mask = torch.ones(buf.shape, dtype=torch.bool, device=buf.device)
    mask[:M, :N] = False
    diff = (_bits(buf) != _bits(before)) & mask
    assert not diff.any(), f"{what}: {int(diff.sum())} elements outside the [{M}, {N}] output window were written"


def _cuda():
    if not torch.cuda.is_available():
        pytest.skip("needs a GPU")
    from colossalai_b200.ops import gemm_native

    if not gemm_native.available():
        pytest.skip("needs an sm_90 GPU")
    return torch.device("cuda")


def _sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


# ============================================================================================ dense 16-bit
def run_dense(tag, M, N, K, dtype=BF16, out=F32, a_mn=0, b_mn=0, acc=False, kind="int", pad=0, ldc_pad=0, seed=0,
              nan_a=None, nan_b=None):
    """One `cb_gemm_tcgen05` problem through `gemm_native._launch`; checks the window and everything around it."""
    from colossalai_b200.ops import gemm_native

    dev = _cuda()
    gen = torch.Generator().manual_seed(seed)
    a_st, a, lda = operand(kind, M, K, dtype, a_mn, gen, dev, pad)
    b_st, b, ldb = operand(kind, N, K, dtype, b_mn, gen, dev, pad)
    if nan_a is not None:
        a[nan_a] = float("nan")
    if nan_b is not None:
        b[nan_b] = float("nan")
    ldc = N + ldc_pad
    buf, c = out_buffer(M, N, out, ldc, dev)
    c0 = None
    if acc:
        c0 = values("int" if kind == "int" else "rand", (M, N), F32, gen, dev).mul_(8).to(out)
        c.copy_(c0)
    before = buf.clone()
    ref, S = ref_and_s(a, b)
    what = f"dense.{_NAME[out]} {tag} {_NAME[dtype]} a_mn={a_mn} b_mn={b_mn} acc={int(acc)} M={M} N={N} K={K}"
    results = []
    for _ in range(1 if kind == "int" else 2):
        if acc:
            c.copy_(c0)
        gemm_native._launch(a_st, b_st, c, M, N, K, lda, ldb, a_mn, b_mn, acc)
        torch.cuda.synchronize()
        assert_outside_untouched(what, buf, before, M, N)
        results.append(c.clone())
    if len(results) == 2:
        check_bitwise(what + " (second run)", results[1], results[0])
    got = results[0]
    full = ref + (c0.double() if acc else 0)
    if nan_a is not None or nan_b is not None:
        return got, full
    if kind == "int":
        check_bitwise(what, got, full.to(out))
    else:
        floor = math.ceil(K / 16) * G16 * S
        if acc:
            floor = floor + U * (S + c0.double().abs())
        check(what, got, full, out, k=1, floor=floor)
    return got, full


# (a_mn, b_mn): (0, 0) = gemm_nt, (0, 1) = gemm_nn, (1, 1) = gemm_tn, (1, 0) = reachable only through `_launch`.
# M = 333 -> 3 row blocks with a 77-row tail; N = 136 -> a 128-column tile and an 8-column tail; K = 200 = 3 * 64 + 8
# -> 4 k-blocks, the last one 8 deep (TMA zero-fills its other 56 columns).
@pytest.mark.gpu
@pytest.mark.parametrize("layout", [(0, 0), (0, 1), (1, 0), (1, 1)], ids=["nt", "nn", "mn_a", "tn"])
@pytest.mark.parametrize("dtype", [BF16, F16], ids=["bf16", "f16"])
@pytest.mark.parametrize("out", [F32, BF16, F16], ids=["o32", "obf16", "of16"])
@pytest.mark.parametrize("acc", [False, True], ids=["set", "acc"])
def test_dense_layouts_epilogues_exact(layout, dtype, out, acc):
    run_dense("layout", 333, 136, 200, dtype, out, *layout, acc=acc, kind="int", pad=8, ldc_pad=8)


# Edges of the tile and the k-block.  M: 1 (one row of one tile), 127 / 128 / 129 (either side of a tile), 333.
# N: 8 (one column pair per thread group), 120 / 128 / 136 (either side of a tile).  K = 72 -> a full k-block and an
# 8-deep tail.
@pytest.mark.gpu
@pytest.mark.parametrize("M", [1, 127, 128, 129, 333])
@pytest.mark.parametrize("N", [8, 120, 128, 136])
def test_dense_tile_edges_exact(M, N):
    run_dense("edge", M, N, 72, BF16, BF16, 0, 0, kind="int", ldc_pad=2)
    run_dense("edge", M, N, 72, F16, F32, 1, 1, kind="int")


# K: 8 / 56 (a single partial k-block), 64 (one full), 72 (full + 8 tail), 320 = 5 blocks (< STAGES), 384 = 6 blocks
# (= STAGES: the ring wraps exactly once), 520 = 8 full + 8 tail = 9 blocks (not a multiple of STAGES, the phase flips
# mid-tile), 1000 = 15 full + 40 tail.
@pytest.mark.gpu
@pytest.mark.parametrize("K", [8, 56, 64, 72, 320, 384, 520, 1000])
@pytest.mark.parametrize("layout", [(0, 0), (1, 0)], ids=["nt", "mn_a"])
def test_dense_k_edges_exact(K, layout):
    run_dense("kedge", 129, 136, K, BF16, F32, *layout, kind="int")


# Tile count against the SM count (grid = min(tiles, SMs)): tiles = SMs - 1, SMs, SMs + 1 with N = 128 (one column
# block, so tiles = m_blocks).  3 * SMs + 5 tiles with K = 448 = 7 k-blocks: each CTA owns 3 or 4 tiles and 7 % 6 != 0,
# so the ring's stage and phase carry from one tile into the next.  M = 13 * 128 + 1 -> 14 row blocks, 14 % GROUP_M = 6:
# the raster's last band is 6 deep, with N = 1024 (8 column blocks, 112 tiles).
@pytest.mark.gpu
@pytest.mark.parametrize("case", ["sms-1", "sms", "sms+1", "multi-tile", "band-tail"])
def test_dense_tile_counts(case):
    sms = _sms()
    M, N, K = {"sms-1": ((sms - 1) * BM, BN, 136), "sms": (sms * BM, BN, 136), "sms+1": ((sms + 1) * BM, BN, 136),
               "multi-tile": ((3 * sms + 5) * BM, BN, 448), "band-tail": (13 * BM + 1, 1024, 200)}[case]
    run_dense(case, M, N, K, BF16, BF16, 0, 0, kind="int")
    run_dense(case, M, N, K, BF16, F32, 0, 1, kind="rand", seed=1)


# Tier B: random signs up to K = 4096 (floor at the median |ref| about 0.04 * K^1.5 * 2^-22 = 0.25% at K = 4096), and
# the long K = 16384 (256 k-blocks) with same-sign operands, where S = |ref|.
@pytest.mark.gpu
@pytest.mark.parametrize("M,N,K,kind", [(333, 136, 1000, "rand"), (256, 264, 4096, "rand"), (256, 256, 16384, "pos")])
@pytest.mark.parametrize("layout", [(0, 0), (0, 1), (1, 0), (1, 1)], ids=["nt", "nn", "mn_a", "tn"])
@pytest.mark.parametrize("dtype,out", [(BF16, F32), (BF16, BF16), (F16, F16)], ids=["bf16-o32", "bf16", "f16"])
def test_dense_random_bound(M, N, K, kind, layout, dtype, out):
    run_dense("rand", M, N, K, dtype, out, *layout, kind=kind, seed=2)


@pytest.mark.gpu
@pytest.mark.parametrize("out", [F32, BF16], ids=["o32", "obf16"])
def test_dense_random_accumulate(out):
    run_dense("rand-acc", 300, 264, 2048, BF16, out, 1, 1, acc=True, kind="rand", seed=3)


# Strided operands: lda / ldb 24 elements past K (K-major; the NaN columns must never be read) and past M / N
# (MN-major: TMA must zero-fill beyond M / N instead of reading the NaN columns); the output is a window into a NaN
# buffer with ldc = N + 24.
@pytest.mark.gpu
@pytest.mark.parametrize("layout", [(0, 0), (0, 1), (1, 0), (1, 1)], ids=["nt", "nn", "mn_a", "tn"])
def test_dense_strided_operands_and_output_window(layout):
    got, _ = run_dense("strided", 200, 136, 136, F16, F16, *layout, kind="int", pad=24, ldc_pad=24)
    assert torch.isfinite(got).all()


@pytest.mark.gpu
@pytest.mark.parametrize("layout", [(0, 0), (1, 1)], ids=["nt", "tn"])
def test_dense_nan_locality(layout):
    """A NaN at A[i, k] poisons exactly row i of D; a NaN at B[j, k] exactly column j."""
    M, N, K = 260, 200, 200
    i, j, k = 131, 130, 190
    got, full = run_dense("nan", M, N, K, BF16, F32, *layout, kind="int", nan_a=(i, k), nan_b=(j, 7))
    nan = torch.isnan(got)
    want = torch.zeros_like(nan)
    want[i, :] = True
    want[:, j] = True
    assert torch.equal(nan, want), f"NaN pattern: {int(nan.sum())} NaN, expected row {i} and column {j} only"
    keep = ~want
    check_bitwise("dense nan locality (finite part)", got[keep], full[keep].float())


# ============================================================================================ fp8
def fp8_call(a, b, c, M, N, K, lda, ldb, acc, sa, sb):
    from colossalai_b200.kernel import loader
    from colossalai_b200.ops import gemm_native

    return gemm_native._get_lib().cb_gemm_fp8_tcgen05(
        loader.ptr(a), loader.ptr(b), ctypes.c_void_p(c.data_ptr()), M, N, K, lda, ldb, c.stride(0), FMT[a.dtype],
        FMT[b.dtype], CODE[c.dtype], int(acc), loader.ptr(sa), loader.ptr(sb), loader.stream_ptr())


def run_fp8(tag, M, N, K, adt, bdt, out, acc=False, scales=(True, True), kind="int", seed=0):
    dev = _cuda()
    gen = torch.Generator().manual_seed(seed)
    a_st, a, lda = operand(kind, M, K, adt, False, gen, dev)
    b_st, b, ldb = operand(kind, N, K, bdt, False, gen, dev)
    if kind == "int":
        sv = (0.5, 4.0)                                        # powers of two: alpha * acc stays exact
    else:
        sv = (0.37, 1.9)
    sa = torch.tensor([sv[0]], device=dev) if scales[0] else None
    sb = torch.tensor([sv[1]], device=dev) if scales[1] else None
    alpha = (float(sa) if scales[0] else 1.0) * (float(sb) if scales[1] else 1.0)
    buf, c = out_buffer(M, N, out, N + 8, dev)
    c0 = None
    if acc:
        c0 = values("int" if kind == "int" else "rand", (M, N), F32, gen, dev).mul_(8).to(out)
    before = buf.clone()
    ref, S = ref_and_s(a, b)
    what = (f"fp8.{_NAME[out]} {tag} {_F8NAME[adt]}x{_F8NAME[bdt]} acc={int(acc)} scales={scales} "
            f"M={M} N={N} K={K}")
    results = []
    for _ in range(1 if kind == "int" else 2):
        if acc:
            c.copy_(c0)
        assert fp8_call(a_st, b_st, c, M, N, K, lda, ldb, acc, sa, sb) == 0, what
        torch.cuda.synchronize()
        assert_outside_untouched(what, buf, before, M, N)
        results.append(c.clone())
    if len(results) == 2:
        check_bitwise(what + " (second run)", results[1], results[0])
    full = alpha * ref + (c0.double() if acc else 0)         # D = alpha * AB + C, not alpha * (AB + C)
    if kind == "int":
        check_bitwise(what, results[0], full.to(out))
    else:
        floor = (4 * G8 + math.ceil(K / KE8) * U + 2 * U) * alpha * S
        if acc:
            floor = floor + U * (alpha * S + c0.double().abs())
        check(what, results[0], full, out, k=1, floor=floor)


FP8_KINDS = [(E4M3, E4M3), (E4M3, E5M2), (E5M2, E4M3), (E5M2, E5M2)]
FP8_IDS = ["e4m3xe4m3", "e4m3xe5m2", "e5m2xe4m3", "e5m2xe5m2"]


# K = 1040 = 8 * 128 + 16: 9 stages, the last 16 deep; lda = K (1040 is a multiple of 16 bytes).  M = 300 / N = 264:
# row and column tails.  All four instantiations, the scales null or not, each output dtype, accumulate or not.
@pytest.mark.gpu
@pytest.mark.parametrize("kinds", FP8_KINDS, ids=FP8_IDS)
@pytest.mark.parametrize("out", [F32, BF16, F16], ids=["o32", "obf16", "of16"])
@pytest.mark.parametrize("acc", [False, True], ids=["set", "acc"])
def test_fp8_kinds_epilogues_exact(kinds, out, acc):
    run_fp8("exact", 300, 264, 1040, *kinds, out, acc=acc)


@pytest.mark.gpu
@pytest.mark.parametrize("scales", [(False, False), (True, False), (False, True)], ids=["none", "a", "b"])
def test_fp8_null_scales_exact(scales):
    run_fp8("scales", 300, 264, 1040, E4M3, E5M2, BF16, acc=True, scales=scales)


# Tier B with same-sign operands (random-sign fp8 would need a floor above 1% of |ref|): K = 1040, and K = 16384 =
# 128 stages, where a partial that was never promoted into fp32 would lose about K / 2 * 2^-13 of the sum (see
# test_comparator_rejects_fp8_without_promotion).
@pytest.mark.gpu
@pytest.mark.parametrize("kinds", FP8_KINDS, ids=FP8_IDS)
@pytest.mark.parametrize("K", [1040, 16384])
@pytest.mark.parametrize("out", [F32, BF16], ids=["o32", "obf16"])
def test_fp8_same_sign_bound(kinds, K, out):
    run_fp8("pos", 256, 264, K, *kinds, out, kind="pos", seed=5)


@pytest.mark.gpu
def test_fp8_same_sign_accumulate():
    run_fp8("pos-acc", 256, 264, 4096, E4M3, E4M3, F32, acc=True, kind="pos", seed=6)


# Shapes below `supported_fp8_nt`'s threshold (M, N >= 128 and tiles >= SMs / 2), run through `gemm_fp8_nt`.
@pytest.mark.gpu
@pytest.mark.parametrize("M,N,K", [(1, 16, 128), (100, 136, 1040), (129, 8, 256)])
def test_fp8_small_shapes_through_wrapper(M, N, K):
    from colossalai_b200.ops import gemm_native

    dev = _cuda()
    gen = torch.Generator().manual_seed(7)
    a = values("int", (M, K), E4M3, gen, dev)
    b = values("int", (N, K), E5M2, gen, dev)
    assert not gemm_native.supported_fp8_nt(a, b)
    sa, sb = torch.tensor([2.0], device=dev), torch.tensor([0.25], device=dev)
    got = gemm_native.gemm_fp8_nt(a, b, sa, sb, torch.float32)
    ref, _ = ref_and_s(a, b)
    check_bitwise(f"gemm_fp8_nt M={M} N={N} K={K}", got, (0.5 * ref).float())


# ============================================================================================ grouped
def _glib():
    from colossalai_b200.moe import grouped_gemm

    return grouped_gemm._get_lib()


def grouped_call(x, w, y, offs, E, total_rows, N, K, transpose_b, ldx=None, ldy=None):
    from colossalai_b200.kernel import loader

    return _glib().cb_grouped_gemm(loader.ptr(x), loader.ptr(w), ctypes.c_void_p(y.data_ptr()), loader.ptr(offs), E,
                                   total_rows, N, K, ldx if ldx is not None else x.stride(0),
                                   ldy if ldy is not None else y.stride(0), int(transpose_b), CODE[x.dtype],
                                   loader.stream_ptr())


def wgrad_call(dy, x, dw, offs, E, total_rows, M, N, acc, out_code=None):
    from colossalai_b200.kernel import loader

    return _glib().cb_grouped_gemm_wgrad(loader.ptr(dy), loader.ptr(x), ctypes.c_void_p(dw.data_ptr()),
                                         loader.ptr(offs), E, total_rows, M, N, dy.stride(0), x.stride(0),
                                         CODE[dy.dtype], CODE[dw.dtype] if out_code is None else out_code, int(acc),
                                         loader.stream_ptr())


def _offs(counts, dev):
    return torch.tensor(counts, dtype=torch.int64).cumsum(0).to(torch.int32).to(dev)


def run_grouped(tag, counts, N, K, dtype=BF16, transpose_b=True, extra_rows=0, kind="int", seed=0, nan=None):
    """Variable-M NT (transpose_b) / NN.  `extra_rows` over-allocates x and y past offs[E - 1] (the buffer size the
    sorted MoE path passes).  Those x rows hold finite values like every other row, so the last group's final row tile,
    which reads them, computes finite rows there; y starts NaN, and those rows must come back bitwise NaN.  No other
    tile is stored over them, so this is the deterministic check of the row mask at the store.  `nan`: ("x", e) NaN
    in the last row of group e; ("w", e) NaN in one column (NT) / k-row (NN) of W[e]."""
    dev = _cuda()
    gen = torch.Generator().manual_seed(seed)
    E, used = len(counts), sum(counts)
    rows = used + extra_rows
    x = values(kind, (rows, K), dtype, gen, dev)
    w = values(kind, (E, N, K) if transpose_b else (E, K, N), dtype, gen, dev)
    if nan is not None:
        what_nan, e = nan
        r0 = sum(counts[:e])
        if what_nan == "x":
            x[r0 + counts[e] - 1, K // 2] = float("nan")
        else:
            w[e, N // 2 if transpose_b else K - 1, K // 2 if transpose_b else N // 2] = float("nan")
    y = torch.full((rows, N), float("nan"), dtype=dtype, device=dev)
    fill = y.clone()
    offs = _offs(counts, dev)
    ref = torch.full((rows, N), float("nan"), dtype=torch.float64, device=dev)
    S = torch.zeros((rows, N), dtype=torch.float64, device=dev)
    s = 0
    for e, n in enumerate(counts):
        if n:
            we = w[e] if transpose_b else w[e].t()
            ref[s:s + n], S[s:s + n] = ref_and_s(x[s:s + n], we)
        s += n
    mode = "nt" if transpose_b else "nn"
    what = f"grouped.{_NAME[dtype]} {tag} {mode} E={E} N={N} K={K} rows={rows}"
    results = []
    for _ in range(1 if kind == "int" else 2):
        y.copy_(fill)
        assert grouped_call(x, w, y, offs, E, rows, N, K, transpose_b) == 0, what
        torch.cuda.synchronize()
        results.append(y.clone())
    if len(results) == 2:
        check_bitwise(what + " (second run)", results[1], results[0])
    got = results[0]
    check_bitwise(f"{what}: rows after the last group", got[used:], fill[used:])
    got, ref, S = got[:used], ref[:used], S[:used]
    if nan is not None:
        return got, ref
    if kind == "int":
        check_bitwise(what, got, ref.to(dtype))
    else:
        check(what, got, ref, dtype, k=1, floor=math.ceil(K / 16) * G16 * S)
    return got, ref


# Group layouts.  Row tiles are per group: a group of n rows has ceil(n / 128) of them, and its last one reads rows of
# the next group (masked at the store).  Sizes 1, 127, 128, 129; empty first, middle and trailing groups; one group of
# 9 * 128 + 5 rows (10 row tiles: a band of GROUP_M = 8 and a band tail of 2) with N = 2048 (16 column blocks: 160 of
# its tiles alone, more than the SMs).  In every layout the last non-empty group ends inside a row tile (300 = 2 * 128
# + 44, 129 = 128 + 1, 333 = 2 * 128 + 77, 200 = 128 + 72) with 37 finite rows after it in the buffer, so that tile
# would store into the sentinel rows without its row mask.
LAYOUTS = {
    "sizes": [1, 127, 128, 129, 300],
    "empty-first-mid-last": [0, 200, 0, 129, 0, 0],
    "single": [333],
    "band-tail": [9 * 128 + 5, 64, 0, 200],
}


@pytest.mark.gpu
@pytest.mark.parametrize("layout", list(LAYOUTS), ids=list(LAYOUTS))
@pytest.mark.parametrize("dtype", [BF16, F16], ids=["bf16", "f16"])
@pytest.mark.parametrize("transpose_b", [True, False], ids=["nt", "nn"])
def test_grouped_layouts_exact(layout, dtype, transpose_b):
    counts = LAYOUTS[layout]
    N = 2048 if layout == "band-tail" else 136
    K = 256 if not transpose_b else (200 if layout != "band-tail" else 128)
    run_grouped(layout, counts, N, K, dtype, transpose_b, extra_rows=37, kind="int")


@pytest.mark.gpu
@pytest.mark.parametrize("transpose_b", [True, False], ids=["nt", "nn"])
def test_grouped_all_empty_and_max_groups(transpose_b):
    """All groups empty (nothing is written), and E = 512 = MAX_GROUPS (its 513-entry tile table ends against the end
    of the kernel's shared memory)."""
    run_grouped("all-empty", [0] * 7, 136, 128, BF16, transpose_b, extra_rows=50, kind="int")
    gen = torch.Generator().manual_seed(8)
    counts = torch.randint(0, 6, (MAX_GROUPS,), generator=gen).tolist()
    counts[3] = 300
    run_grouped("E=512", counts, 136, 128, BF16, transpose_b, extra_rows=3, kind="int")


@pytest.mark.gpu
@pytest.mark.parametrize("transpose_b", [True, False], ids=["nt", "nn"])
@pytest.mark.parametrize("dtype", [BF16, F16], ids=["bf16", "f16"])
def test_grouped_random_bound(transpose_b, dtype):
    run_grouped("rand", [300, 0, 1, 255, 256, 257, 700, 131], 264, 1024, dtype, transpose_b, extra_rows=9,
                kind="rand", seed=9)


@pytest.mark.gpu
@pytest.mark.parametrize("transpose_b", [True, False], ids=["nt", "nn"])
@pytest.mark.parametrize("where", ["x", "w"])
def test_grouped_nan_locality(transpose_b, where):
    """The exact NaN pattern, and every other element bitwise.

    where = "x": a NaN at x[r, K / 2], r the last row of group 1, must poison exactly output row r - each row is its
    own reduction, so this checks that x rows reach the right output rows and nothing else.
    where = "w": a NaN in W[1] (row N / 2 of the [N, K] matrix for NT; the last k-row, K - 1, of the [K, N] matrix for
    NN) must poison exactly column N / 2 of group 1's rows.  For NN a k-block that ran from W[1] into W[2] (or the
    other way) would carry it into group 0 or 2.  Group 1 ends 28 rows into a row tile whose other rows are group 2's,
    so an unmasked store of that tile would also put the NaN column into group 2's first rows - but only when it lands
    after group 2's own tile, which depends on CTA timing.  The deterministic check of that mask is the over-allocated
    buffer in `run_grouped`."""
    counts = [128, 100, 300, 129]
    e, N, K = 1, 256, 256
    got, ref = run_grouped(f"nan-{where}", counts, N, K, BF16, transpose_b, kind="int", nan=(where, e))
    r0, r1 = sum(counts[:e]), sum(counts[:e + 1])
    want = torch.zeros(got.shape, dtype=torch.bool, device=got.device)
    if where == "x":
        want[r1 - 1, :] = True
    else:
        want[r0:r1, N // 2] = True
    nan = torch.isnan(got)
    if not torch.equal(nan, want):
        extra, missing = (nan & ~want).nonzero(), (want & ~nan).nonzero()
        raise AssertionError(f"NaN pattern: {len(extra)} unexpected NaN (first {extra[:4].tolist()}), "
                             f"{len(missing)} expected NaN missing (first {missing[:4].tolist()})")
    check_bitwise("grouped nan locality (finite part)", got[~want], ref[~want].to(BF16))


# ---- variable-K weight gradient
def run_wgrad(tag, counts, M, N, dtype=BF16, out=F32, acc=False, extra_rows=0, kind="int", seed=0, nan_e=None):
    """dw[e] (+)= dy[rows e]^T x[rows e].  Group row ranges are multiples of 128.  Rows after offs[E - 1] are NaN."""
    dev = _cuda()
    gen = torch.Generator().manual_seed(seed)
    E, used = len(counts), sum(counts)
    assert all(n % 128 == 0 for n in counts)
    rows = used + extra_rows
    dy = values(kind, (rows, M), dtype, gen, dev)
    x = values(kind, (rows, N), dtype, gen, dev)
    if extra_rows:
        dy[used:] = float("nan")
        x[used:] = float("nan")
    if nan_e is not None:
        x[sum(counts[:nan_e]) + counts[nan_e] // 2, N // 2] = float("nan")
    offs = _offs(counts, dev)
    c0 = values("int" if kind == "int" else "rand", (E, M, N), F32, gen, dev).mul_(8).to(out) if acc else None
    ref = torch.zeros((E, M, N), dtype=torch.float64, device=dev)
    S = torch.zeros_like(ref)
    s = 0
    for e, n in enumerate(counts):
        if n:
            ref[e], S[e] = ref_and_s(dy[s:s + n].t(), x[s:s + n].t())
        s += n
    what = f"wgrad.{_NAME[out]} {tag} {_NAME[dtype]} acc={int(acc)} E={E} M={M} N={N} rows={rows}"
    dw = torch.full((E, M, N), float("nan"), dtype=out, device=dev)
    results = []
    for _ in range(1 if kind == "int" else 2):
        if acc:
            dw.copy_(c0)
        else:
            dw.fill_(float("nan"))
        assert wgrad_call(dy, x, dw, offs, E, rows, M, N, acc) == 0, what
        torch.cuda.synchronize()
        results.append(dw.clone())
    if len(results) == 2:
        check_bitwise(what + " (second run)", results[1], results[0])
    got = results[0]
    full = ref + (c0.double() if acc else 0)
    if nan_e is not None:
        return got, full
    if kind == "int":
        check_bitwise(what, got, full.to(out))
    else:
        kmax = max(counts)
        floor = math.ceil(kmax / 16) * G16 * S
        if acc:
            floor = floor + U * (S + c0.double().abs())
        check(what, got, full, out, k=1, floor=floor)
    return got, full


# Expert row ranges 0 (dW = 0, or C unchanged), 128, 384 (6 k-blocks of 64 = STAGES), 512 (8), at the first, middle
# and last position; M = 264 / N = 136 leave row and column tails; 37 NaN rows after the last group.
WGRAD_COUNTS = [0, 128, 0, 384, 512, 0]


@pytest.mark.gpu
@pytest.mark.parametrize("dtype", [BF16, F16], ids=["bf16", "f16"])
@pytest.mark.parametrize("out", [F32, BF16, F16], ids=["o32", "obf16", "of16"])
@pytest.mark.parametrize("acc", [False, True], ids=["set", "acc"])
def test_wgrad_epilogues_exact(dtype, out, acc):
    run_wgrad("exact", WGRAD_COUNTS, 264, 136, dtype, out, acc=acc, extra_rows=37, kind="int")


@pytest.mark.gpu
@pytest.mark.parametrize("acc", [False, True], ids=["set", "acc"])
def test_wgrad_all_empty_and_max_groups(acc):
    """No rows anywhere: dW is exactly zero (or C unchanged); and E = 512."""
    run_wgrad("all-empty", [0] * 5, 136, 128, BF16, F32, acc=acc, extra_rows=40, kind="int")
    counts = [0] * MAX_GROUPS
    counts[0], counts[200], counts[MAX_GROUPS - 1] = 128, 256, 128
    run_wgrad("E=512", counts, 16, 24, BF16, BF16, acc=acc, kind="int")


@pytest.mark.gpu
@pytest.mark.parametrize("out", [F32, BF16], ids=["o32", "obf16"])
@pytest.mark.parametrize("acc", [False, True], ids=["set", "acc"])
def test_wgrad_random_bound(out, acc):
    run_wgrad("rand", [256, 0, 1024, 128], 264, 392, BF16, out, acc=acc, extra_rows=5, kind="rand", seed=10)


@pytest.mark.gpu
def test_wgrad_nan_locality():
    """NaN in expert e's x rows reaches only dW[e]: no k-block mixes two experts, and the NaN rows after the last
    group never reach any dW."""
    counts = [128, 256, 0, 128]
    got, full = run_wgrad("nan", counts, 136, 264, BF16, F32, extra_rows=64, kind="int", nan_e=1)
    bad = torch.isnan(got).flatten(1).any(1)
    assert bad.tolist() == [False, True, False, False], bad.tolist()
    for e in (0, 2, 3):
        check_bitwise(f"wgrad nan locality dW[{e}]", got[e], full[e].float())


# ============================================================================================ launcher envelope
def _nan(shape, dtype, dev):
    return torch.full(shape, float("nan"), dtype=dtype, device=dev)


def _assert_all_nan(bufs):
    torch.cuda.synchronize()
    for name, t in bufs.items():
        assert torch.isnan(t.float()).all(), f"a rejected call wrote {name}"


@pytest.mark.gpu
def test_launchers_reject_unknown_out_dtype():
    """An out_dtype other than fp32 / fp16 / bf16 is refused; it used to be stored as fp16."""
    from colossalai_b200.kernel import loader
    from colossalai_b200.ops import gemm_native

    dev = _cuda()
    a, b = torch.ones(128, 128, dtype=BF16, device=dev), torch.ones(128, 128, dtype=BF16, device=dev)
    a8, b8 = a.to(E4M3), b.to(E4M3)
    c = _nan((128, 128), F16, dev)
    offs = _offs([128], dev)
    lib, st = gemm_native._get_lib(), loader.stream_ptr()
    P = loader.ptr
    for bad in (CODE[E4M3], CODE[E5M2], 7, -1):
        rc = lib.cb_gemm_tcgen05(P(a), P(b), P(c), 128, 128, 128, 128, 128, 128, 0, 0, CODE[BF16], bad, 0, 0, st)
        assert rc == INVALID, f"cb_gemm_tcgen05 out_dtype={bad}: returned {rc}"
        rc = lib.cb_gemm_fp8_tcgen05(P(a8), P(b8), P(c), 128, 128, 128, 128, 128, 128, 0, 0, bad, 0, None, None, st)
        assert rc == INVALID, f"cb_gemm_fp8_tcgen05 out_dtype={bad}: returned {rc}"
        rc = _glib().cb_grouped_gemm_wgrad(P(a), P(b), P(c), P(offs), 1, 128, 128, 128, 128, 128, CODE[BF16], bad, 0,
                                           st)
        assert rc == INVALID, f"cb_grouped_gemm_wgrad out_dtype={bad}: returned {rc}"
    _assert_all_nan({"C": c})


@pytest.mark.gpu
def test_launchers_reject_k_zero():
    """K <= 0 is refused with cudaErrorInvalidValue (no tensor map can describe an empty operand)."""
    from colossalai_b200.kernel import loader
    from colossalai_b200.ops import gemm_native

    dev = _cuda()
    a = torch.ones(128, 128, dtype=BF16, device=dev)
    a8 = a.to(E4M3)
    c = _nan((128, 128), F32, dev)
    y = _nan((128, 128), BF16, dev)
    offs = _offs([128], dev)
    lib, st, P = gemm_native._get_lib(), loader.stream_ptr(), loader.ptr
    for K in (0, -64):
        for acc in (0, 1):
            rc = lib.cb_gemm_tcgen05(P(a), P(a), P(c), 128, 128, K, 128, 128, 128, 0, 0, CODE[BF16], CODE[F32], acc,
                                     0, st)
            assert rc == INVALID, f"cb_gemm_tcgen05 K={K} accumulate={acc}: returned {rc}"
        rc = lib.cb_gemm_fp8_tcgen05(P(a8), P(a8), P(c), 128, 128, K, 128, 128, 128, 0, 0, CODE[F32], 0, None, None,
                                     st)
        assert rc == INVALID, f"cb_gemm_fp8_tcgen05 K={K}: returned {rc}"
        rc = _glib().cb_grouped_gemm(P(a), P(a), P(y), P(offs), 1, 128, 128, K, 128, 128, 1, CODE[BF16], st)
        assert rc == INVALID, f"cb_grouped_gemm K={K}: returned {rc}"
    _assert_all_nan({"C": c, "y": y})


@pytest.mark.gpu
def test_launchers_reject_out_of_envelope():
    """Every call outside a launcher's envelope returns cudaErrorInvalidValue and writes nothing, including outputs
    the two-element epilogue store cannot write (a base not aligned to two elements, an odd or short ldc)."""
    from colossalai_b200.kernel import loader
    from colossalai_b200.ops import gemm_native

    dev = _cuda()
    lib, glib, st, P = gemm_native._get_lib(), _glib(), loader.stream_ptr(), loader.ptr
    a = torch.ones(256, 256, dtype=BF16, device=dev)
    a8 = a.to(E4M3)
    c32 = _nan((130, 136), F32, dev)
    c16 = _nan((130, 136), BF16, dev)
    y = _nan((300, 136), BF16, dev)
    dw = _nan((2 * 128 * 136 + 8,), F32, dev)
    offs = _offs([128, 128], dev)
    off = lambda t, n: ctypes.c_void_p(t.data_ptr() + n * t.element_size())   # noqa: E731

    def dense(C=None, ldc=136, out=CODE[F32], K=128, ind=CODE[BF16]):
        return lib.cb_gemm_tcgen05(P(a), P(a), C if C is not None else P(c32), 128, 128, K, 256, 256, ldc, 0, 0, ind,
                                   out, 0, 0, st)

    def fp8(C=None, ldc=136, out=CODE[F32], lda=256):
        return lib.cb_gemm_fp8_tcgen05(P(a8), P(a8), C if C is not None else P(c32), 128, 128, 128, lda, 256, ldc, 0,
                                       0, out, 0, None, None, st)

    def grouped(E=2, N=128, K=128, ldy=136, Y=None, tb=1, dtype=CODE[BF16]):
        return glib.cb_grouped_gemm(P(a), P(a), Y if Y is not None else P(y), P(offs), E, 256, N, K, 256, ldy, tb,
                                    dtype, st)

    def wgrad(E=2, M=128, N=136, out=CODE[F32], DW=None):
        return glib.cb_grouped_gemm_wgrad(P(a), P(a), DW if DW is not None else P(dw), P(offs), E, 256, M, N, 256,
                                          256, CODE[BF16], out, 0, st)

    rejected = {
        "dense fp32 input": lambda: dense(ind=CODE[F32]),
        "dense fp32 C 4 bytes off": lambda: dense(C=off(c32, 1)),
        "dense bf16 C 2 bytes off": lambda: dense(C=off(c16, 1), out=CODE[BF16]),
        "dense odd ldc": lambda: dense(ldc=135),
        "dense ldc < N": lambda: dense(ldc=126),
        "dense empty M, bad out_dtype": lambda: lib.cb_gemm_tcgen05(P(a), P(a), P(c32), 0, 128, 128, 256, 256, 136, 0,
                                                                   0, CODE[BF16], 9, 0, 0, st),
        "fp8 lda % 16": lambda: fp8(lda=248 + 4),
        "fp8 fp32 C 4 bytes off": lambda: fp8(C=off(c32, 1)),
        "fp8 odd ldc": lambda: fp8(ldc=137),
        "grouped E = 513": lambda: grouped(E=MAX_GROUPS + 1),
        "grouped fp32": lambda: grouped(dtype=CODE[F32]),
        "grouped N % 8": lambda: grouped(N=124, ldy=124),
        "grouped K % 8": lambda: grouped(K=100),
        "grouped NN K % 128": lambda: grouped(K=192, tb=0),
        "grouped y 2 bytes off": lambda: grouped(Y=off(y, 1)),
        "grouped odd ldy": lambda: grouped(ldy=135),
        "wgrad E = 513": lambda: wgrad(E=MAX_GROUPS + 1),
        "wgrad M % 8": lambda: wgrad(M=124),
        "wgrad fp32 dW 4 bytes off": lambda: wgrad(DW=off(dw, 1)),
        "wgrad total_rows 0": lambda: glib.cb_grouped_gemm_wgrad(P(a), P(a), P(dw), P(offs), 2, 0, 128, 136, 256, 256,
                                                                CODE[BF16], CODE[F32], 0, st),
    }
    for name, call in rejected.items():
        rc = call()
        assert rc == INVALID, f"{name}: returned {rc}"
    _assert_all_nan({"C fp32": c32, "C bf16": c16, "y": y, "dW": dw})
    # the same buffers are written by calls inside the envelope
    assert dense() == 0 and grouped() == 0 and wgrad() == 0
    torch.cuda.synchronize()
    assert torch.isfinite(c32[:128, :128]).all() and torch.isfinite(y[:256, :128]).all()


def test_out_ok_predicate():
    """`gemm_native.out_ok` accepts exactly the outputs the epilogue's two-element stores can write (runs on CPU)."""
    from colossalai_b200.ops.gemm_native import out_ok

    for dt in (F32, BF16, F16):
        flat = torch.zeros(64 * 40 + 8, dtype=dt)
        base = flat[:64 * 40].view(64, 40)
        assert out_ok(base)
        assert out_ok(flat[2:2 + 64 * 40].view(64, 40))                      # two elements off: still a pair
        assert not out_ok(flat[1:1 + 64 * 40].view(64, 40)), dt              # one element off
        assert out_ok(flat[:63 * 40 + 38].as_strided((64, 38), (40, 1)))     # window, even ldc
        assert not out_ok(flat[:64 * 39].view(64, 39)), dt                   # odd ldc
        assert not out_ok(base.t())                                          # column stride != 1
    assert not out_ok(torch.zeros(8, 8, dtype=torch.float64))
    assert not out_ok(torch.zeros(64, dtype=F32))


@pytest.mark.gpu
def test_gemm_wrappers_check_out():
    """`gemm_nt` / `gemm_nn` / `gemm_tn` / `gemm_fp8_nt` refuse an output of the wrong shape or one the epilogue
    cannot store into, before launching."""
    from colossalai_b200.ops import gemm_native as g

    dev = _cuda()
    a = torch.ones(256, 128, dtype=BF16, device=dev)
    flat = _nan((256 * 258,), BF16, dev)
    shifted = flat[1:1 + 256 * 256].view(256, 256)
    odd = flat.as_strided((256, 256), (257, 1))
    for out in (shifted, odd, _nan((256, 128), BF16, dev), _nan((256, 256), torch.float64, dev)):
        with pytest.raises(ValueError, match="gemm output"):
            g.gemm_nt(a, a.new_ones(256, 128), out=out)
        with pytest.raises(ValueError, match="gemm output"):
            g.gemm_nn(a.new_ones(256, 256), a.new_ones(256, 256), out=out)
        with pytest.raises(ValueError, match="gemm output"):
            g.gemm_tn(a.new_ones(128, 256), a.new_ones(128, 256), out=out, accumulate=True)
    with pytest.raises(ValueError, match="gemm output"):
        g.gemm_fp8_nt(a.to(E4M3), a.to(E4M3), None, None, out=_nan((256, 257), BF16, dev)[:, 1:])
    torch.cuda.synchronize()
    assert torch.isnan(flat.float()).all()


@pytest.mark.gpu
@pytest.mark.parametrize("out_dtype", [F32, BF16], ids=["o32", "obf16"])
@pytest.mark.parametrize("accumulate", [False, True], ids=["set", "acc"])
def test_matmul_tn_misaligned_out_stays_native(out_dtype, accumulate):
    """`ops.matmul_tn` with an output view one element off alignment (a parameter's slice of a flat gradient buffer)
    runs the native GEMM into an aligned copy and writes the exact result into the view."""
    from colossalai_b200 import ops
    from colossalai_b200.kernel import loader
    from colossalai_b200.ops import gemm as gemm_ops

    dev = _cuda()
    gen = torch.Generator().manual_seed(11)
    red, M, N = 1024, 256, 384
    a = values("int", (red, M), BF16, gen, dev)
    b = values("int", (red, N), BF16, gen, dev)
    flat = torch.zeros(M * N + 3, dtype=out_dtype, device=dev)
    flat[0], flat[-2:] = 7, 7
    out = flat[1:1 + M * N].view(M, N)
    c0 = values("int", (M, N), F32, gen, dev).to(out_dtype)
    out.copy_(c0)
    old = gemm_ops.get_gemm_backend()
    gemm_ops.set_gemm_backend("native")
    before = loader.launch_counter.by_name.get("gemm_tcgen05", 0)
    try:
        r = ops.matmul_tn(a, b, out=out, accumulate=accumulate)
    finally:
        gemm_ops.set_gemm_backend(old)
    torch.cuda.synchronize()
    assert loader.launch_counter.by_name.get("gemm_tcgen05", 0) == before + 1, "the native GEMM did not run"
    assert r.data_ptr() == out.data_ptr()
    ref = a.double().t() @ b.double() + (c0.double() if accumulate else 0)
    check_bitwise(f"matmul_tn misaligned {_NAME[out_dtype]} acc={accumulate}", out, ref.to(out_dtype))
    assert flat[0].item() == 7 and flat[-2:].tolist() == [7, 7], "matmul_tn wrote outside its output view"


# ============================================================================================ comparator (CPU)
def _trunc_bits(x: torch.Tensor, bits: int) -> torch.Tensor:
    """x truncated (toward zero) to `bits` significant bits."""
    m, e = torch.frexp(x)
    return torch.ldexp(torch.trunc(torch.ldexp(m, torch.full_like(e, bits))), e - bits)


def _bf16_truncate(x: torch.Tensor) -> torch.Tensor:
    return (x.float().view(torch.int32) & ~0xFFFF).view(torch.float32).to(BF16)


def _emulate_dense(a, b, *, drop=None, twice=None):
    """float64 A @ B^T over the K columns `keep`, optionally leaving out or repeating a K range."""
    K = a.shape[1]
    w = torch.ones(K, dtype=torch.float64)
    if drop is not None:
        w[drop[0]:drop[1]] = 0
    if twice is not None:
        w[twice[0]:twice[1]] = 2
    return (a.double() * w) @ b.double().t()


def _emulate_fp8(a, b, bits, promote):
    """fp8 products summed in k32 instructions into an accumulator kept to `bits` significant bits (truncating); with
    `promote`, the partial restarts every 128-deep stage and is added to an fp32 accumulator."""
    prod = a.double()[:, None, :] * b.double()[None, :, :]                   # [M, N, K]
    K = prod.shape[-1]
    acc = torch.zeros(prod.shape[:2], dtype=torch.float64)
    part = torch.zeros_like(acc)
    for k0 in range(0, K, 32):
        part = _trunc_bits(part + prod[..., k0:k0 + 32].sum(-1), bits)
        if promote and ((k0 + 32) % 128 == 0 or k0 + 32 >= K):
            acc = (acc + part).float().double()
            part = torch.zeros_like(acc)
    return acc if promote else part


FAULTS = ["dropped 64-wide k-block", "dropped 8-element K tail", "k-block counted twice",
          "tile stored one column block off", "next group's rows unmasked", "alpha applied to C as well",
          "scale_b ignored", "accumulate ignored", "bf16 output truncated instead of rounded"]


def _faulty(fault, gen, kind):
    """(what the kernel would store, the float64 reference, floor) for one injected fault; bf16 output."""
    M, N, K = 256, 264, 200
    a = values(kind, (M, K), BF16, gen, "cpu")
    b = values(kind, (N, K), BF16, gen, "cpu")
    ref, S = ref_and_s(a, b)
    c = values("int" if kind == "int" else "rand", (M, N), F32, gen, "cpu").mul_(8).to(BF16).double()
    floor = math.ceil(K / 16) * G16 * S
    alpha = 0.5 if kind == "int" else 0.37
    if fault == "dropped 64-wide k-block":
        return _emulate_dense(a, b, drop=(64, 128)), ref, floor
    if fault == "dropped 8-element K tail":
        return _emulate_dense(a, b, drop=(192, 200)), ref, floor
    if fault == "k-block counted twice":
        return _emulate_dense(a, b, twice=(128, 192)), ref, floor
    if fault == "tile stored one column block off":
        got = ref.clone()
        got[:128, 128:256] = ref[:128, :128]
        return got, ref, floor
    if fault == "next group's rows unmasked":
        # groups of 100 and 156 rows, W[0] = b, W[1] = -b + 1: group 0's only row tile also stores rows 100..127
        b1 = (1 - b.double()).to(BF16)
        want = torch.cat([ref[:100], ref_and_s(a[100:], b1)[0]])
        s1 = torch.cat([S[:100], ref_and_s(a[100:], b1)[1]])
        got = want.clone()
        got[100:128] = ref[100:128]
        return got, want, math.ceil(K / 16) * G16 * s1
    if fault == "alpha applied to C as well":
        return alpha * (ref + c), alpha * ref + c, alpha * floor + U * (alpha * S + c.abs())
    if fault == "scale_b ignored":
        return 0.5 * ref, 0.5 * 4.0 * ref, 2.0 * floor
    if fault == "accumulate ignored":
        return ref, ref + c, floor + U * (S + c.abs())
    assert fault == "bf16 output truncated instead of rounded"
    return ref, ref, floor


@pytest.mark.parametrize("fault", FAULTS)
def test_comparator_rejects_gemm_faults(fault):
    """Each fault is rejected by the exact tier (integer operands), and, except the rounding mode, which only the exact
    tier can see, by the bound tier (random operands) as well."""
    gen = torch.Generator().manual_seed(12)
    got, ref, _ = _faulty(fault, gen, "int")
    stored = _bf16_truncate(got) if fault.startswith("bf16") else got.to(BF16)
    with pytest.raises(AssertionError, match="differ bitwise"):
        check_bitwise(fault, stored, ref.to(BF16))
    if fault.startswith("bf16"):
        return
    got, ref, floor = _faulty(fault, gen, "rand")
    with pytest.raises(AssertionError, match=f"^{fault}: .*out of tolerance"):
        check(fault, got.to(BF16), ref, BF16, k=1, floor=floor)


def test_comparator_rejects_fp8_without_promotion():
    """fp8 at K = 16384 with same-sign operands: a 13-bit accumulator never promoted into fp32 is rejected; the
    promoted 14-bit accumulation the bound is derived from is accepted."""
    gen = torch.Generator().manual_seed(13)
    M, N, K = 4, 4, 16384
    a = values("pos", (M, K), E4M3, gen, "cpu")
    b = values("pos", (N, K), E4M3, gen, "cpu")
    ref, S = ref_and_s(a, b)
    floor = (4 * G8 + math.ceil(K / KE8) * U + 2 * U) * S
    fault = "fp8 13-bit accumulator without per-stage promotion"
    with pytest.raises(AssertionError, match=f"^{fault}: .*out of tolerance"):
        check(fault, _emulate_fp8(a, b, 13, promote=False).float(), ref, F32, k=1, floor=floor)
    check("selftest.fp8 promoted 14-bit", _emulate_fp8(a, b, 14, promote=True).float(), ref, F32, k=1, floor=floor)


@pytest.mark.parametrize("out", [F32, BF16, F16], ids=["o32", "obf16", "of16"])
def test_comparator_accepts_correct_gemms(out):
    """The reference rounded to the output dtype, and an fp32 accumulation in a shuffled K order, are accepted."""
    gen = torch.Generator().manual_seed(14)
    M, N, K = 256, 264, 4096
    a = values("rand", (M, K), BF16, gen, "cpu")
    b = values("rand", (N, K), BF16, gen, "cpu")
    ref, S = ref_and_s(a, b)
    floor = math.ceil(K / 16) * G16 * S
    check("selftest.rounded", ref.to(out), ref, out, k=1, floor=floor)
    perm = torch.randperm(K, generator=gen)
    shuffled = torch.zeros(M, N, dtype=torch.float32)
    for k0 in range(0, K, 16):                                  # sequential fp32 adds of k16 partial sums
        idx = perm[k0:k0 + 16]
        shuffled += a[:, idx].float() @ b[:, idx].float().t()
    check("selftest.shuffled_f32", shuffled.to(out), ref, out, k=1, floor=floor)
    ai = values("int", (M, 200), BF16, gen, "cpu")
    bi = values("int", (N, 200), BF16, gen, "cpu")
    refi, _ = ref_and_s(ai, bi)
    check_bitwise("selftest.exact", refi.to(out), refi.to(out))
