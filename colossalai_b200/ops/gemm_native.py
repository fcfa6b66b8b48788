"""ctypes face of the wgmma GEMM (kernel/csrc/gemm_wgmma.cu)."""
from __future__ import annotations

import ctypes
import os
from typing import Optional

import torch

from ..kernel import loader
from ._dtypes import code

_lib = None
_MIN_FLOPS = int(os.environ.get("CB200_GEMM_MIN_FLOPS", str(1 << 24)))
_DISABLED = os.environ.get("CB200_DISABLE_TCGEN05_GEMM", "0") == "1"


def _get_lib():
    global _lib
    if _lib is None:
        _lib = loader.load("cb200_gemm")
    return _lib


def available() -> bool:
    if _DISABLED or not torch.cuda.is_available():
        return False
    if torch.cuda.get_device_capability()[0] != 9:
        return False
    try:
        _get_lib()
        return True
    except Exception:
        return False


def _ok2d(t: torch.Tensor) -> bool:
    return (t.dim() == 2 and t.dtype in (torch.bfloat16, torch.float16) and t.stride(1) == 1
            and t.stride(0) % 8 == 0 and t.data_ptr() % 16 == 0 and t.stride(0) >= t.shape[1])


def out_ok(c: torch.Tensor) -> bool:
    """True if the epilogue can store into `c`: fp32/bf16/fp16 rows of unit stride, and since two adjacent columns
    go out as one 2-element store, a base aligned to two elements and an even row stride."""
    return (c.dim() == 2 and c.dtype in (torch.float32, torch.bfloat16, torch.float16) and c.stride(1) == 1
            and c.stride(0) % 2 == 0 and c.stride(0) >= c.shape[1] and c.data_ptr() % (2 * c.element_size()) == 0)


def _check_out(c: torch.Tensor, M: int, N: int, like: torch.Tensor) -> None:
    if c.device != like.device or tuple(c.shape) != (M, N) or not out_ok(c):
        raise ValueError(f"gemm output must be a [{M}, {N}] fp32/bf16/fp16 tensor on {like.device} with unit column "
                         f"stride, an even row stride and a base aligned to two elements; got {tuple(c.shape)} "
                         f"{c.dtype} stride {c.stride()} at offset {c.data_ptr() % 16} mod 16 on {c.device}")


def _big(m: int, n: int, k: int) -> bool:
    return 2 * m * n * k >= _MIN_FLOPS and k >= 64 and n >= 64


def _launch(a, b, c, M, N, K, lda, ldb, a_mn, b_mn, accumulate, block_n=0) -> None:
    lib = _get_lib()
    rc = lib.cb_gemm_tcgen05(loader.ptr(a), loader.ptr(b), loader.ptr(c), M, N, K, lda, ldb, c.stride(0), a_mn, b_mn,
                             code(a.dtype), code(c.dtype), int(accumulate), block_n, loader.stream_ptr())
    loader.check(rc, "gemm_tcgen05")
    loader.launch_counter.add("gemm_tcgen05")


# ---- y[M,N] = x[M,K] @ w[N,K]^T
def supported_nt(x: torch.Tensor, w: torch.Tensor) -> bool:
    x2 = x.reshape(-1, x.shape[-1]) if x.dim() != 2 else x
    return (x.dtype == w.dtype and _ok2d(x2) and _ok2d(w) and w.shape[0] % 8 == 0
            and _big(x2.shape[0], w.shape[0], w.shape[1]))


def gemm_nt(x: torch.Tensor, w: torch.Tensor, out: Optional[torch.Tensor] = None, block_n: int = 0) -> torch.Tensor:
    M, K = x.shape
    N = w.shape[0]
    y = out if out is not None else torch.empty(M, N, dtype=x.dtype, device=x.device)
    _check_out(y, M, N, x)
    _launch(x, w, y, M, N, K, x.stride(0), w.stride(0), 0, 0, False, block_n)
    return y


# ---- c[M,N] = a[M,K] @ b[K,N]       (dgrad: b = W stored [N_out, K_in] is the MN-major "B")
def supported_nn(a: torch.Tensor, b: torch.Tensor) -> bool:
    return (a.dtype == b.dtype and _ok2d(a) and _ok2d(b) and b.shape[1] % 8 == 0
            and _big(a.shape[0], b.shape[1], a.shape[1]))


def gemm_nn(a: torch.Tensor, b: torch.Tensor, out: Optional[torch.Tensor] = None, block_n: int = 0) -> torch.Tensor:
    M, K = a.shape
    N = b.shape[1]
    c = out if out is not None else torch.empty(M, N, dtype=a.dtype, device=a.device)
    _check_out(c, M, N, a)
    _launch(a, b, c, M, N, K, a.stride(0), b.stride(0), 0, 1, False, block_n)
    return c


# ---- c[N,K] = a[M,N]^T @ b[M,K]     (wgrad: contraction over the token dim M; both operands MN-major)
def supported_tn(a: torch.Tensor, b: torch.Tensor) -> bool:
    return (a.dtype == b.dtype and _ok2d(a) and _ok2d(b) and a.shape[1] % 8 == 0 and b.shape[1] % 8 == 0
            and _big(a.shape[1], b.shape[1], a.shape[0]))


def gemm_tn(a: torch.Tensor, b: torch.Tensor, out: Optional[torch.Tensor] = None, accumulate: bool = False,
            block_n: int = 0) -> torch.Tensor:
    red, M = a.shape
    N = b.shape[1]
    if out is None:
        out = torch.empty(M, N, dtype=a.dtype, device=a.device)
        accumulate = False
    _check_out(out, M, N, a)
    _launch(a, b, out, M, N, red, a.stride(0), b.stride(0), 1, 1, accumulate, block_n)
    return out


# ---- fp8: c[M,N] = scale_a * scale_b * (a[M,K] @ b[N,K]^T), operands e4m3 / e5m2, both K-major
_FP8_FMT = {getattr(torch, "float8_e4m3fn", None): 0, getattr(torch, "float8_e5m2", None): 1}
_FP8_BACKEND = os.environ.get("CB200_FP8_GEMM", "native")      # "native" -> wgmma m64n128k32 fp8 kernel


def fp8_backend() -> str:
    return _FP8_BACKEND


def set_fp8_backend(name: str) -> None:
    global _FP8_BACKEND
    assert name in ("native", "cublaslt")
    _FP8_BACKEND = name


def supported_fp8_nt(a: torch.Tensor, b: torch.Tensor) -> bool:
    def ok(t):
        return (t.dim() == 2 and t.dtype in _FP8_FMT and t.stride(1) == 1 and t.stride(0) % 16 == 0
                and t.data_ptr() % 16 == 0 and t.stride(0) >= t.shape[1])

    if not (a.is_cuda and ok(a) and ok(b) and a.shape[1] == b.shape[1]):
        return False
    M, K, N = a.shape[0], a.shape[1], b.shape[0]
    # the kernel runs one persistent CTA per SM on 128 x 128 output tiles: shapes with fewer tiles than half the SMs
    # would leave most of the GPU idle, and go to cuBLASLt instead
    sms = torch.cuda.get_device_properties(a.device).multi_processor_count
    return M >= 128 and N >= 128 and K >= 128 and N % 8 == 0 and ((M + 127) // 128) * ((N + 127) // 128) >= sms // 2


def gemm_fp8_nt(a: torch.Tensor, b: torch.Tensor, scale_a: Optional[torch.Tensor], scale_b: Optional[torch.Tensor],
                out_dtype: torch.dtype = torch.bfloat16, out: Optional[torch.Tensor] = None) -> torch.Tensor:
    """a [M, K] fp8, b [N, K] fp8 (rows contiguous); scales are fp32 device scalars (dequantisation factors)."""
    M, K = a.shape
    N = b.shape[0]
    c = out if out is not None else torch.empty(M, N, dtype=out_dtype, device=a.device)
    _check_out(c, M, N, a)
    sa = None if scale_a is None else scale_a.reshape(1).to(device=a.device, dtype=torch.float32)
    sb = None if scale_b is None else scale_b.reshape(1).to(device=a.device, dtype=torch.float32)
    lib = _get_lib()
    rc = lib.cb_gemm_fp8_tcgen05(loader.ptr(a), loader.ptr(b), loader.ptr(c), M, N, K, a.stride(0), b.stride(0),
                                 c.stride(0), _FP8_FMT[a.dtype], _FP8_FMT[b.dtype], code(c.dtype), 0,
                                 loader.ptr(sa), loader.ptr(sb), loader.stream_ptr())
    loader.check(rc, "gemm_fp8_tcgen05")
    loader.launch_counter.add("gemm_fp8_tcgen05")
    return c
