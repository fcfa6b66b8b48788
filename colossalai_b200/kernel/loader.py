"""Native kernel build + load.

Parity: reference `colossalai/kernel/kernel_loader.py:31-131` + `extensions/{base,cpp,cuda}_extension.py`
(AOT/JIT build of op families, `KernelLoader.load()`).  H100-first differences:
  * ONE arch: every `.cu` is compiled with `-gencode arch=compute_90a,code=sm_90a -lineinfo`;
  * kernels export plain C launchers (`extern "C"`, raw pointers + cudaStream_t) and are loaded with ctypes —
    no torch headers in the CUDA translation units, so a full rebuild takes seconds and the `.so` files live
    IN-TREE (`colossalai_b200/kernel/_build/`) so they travel to the GPU box with the repo snapshot;
  * on a GPU box a missing/unloadable library is a hard error (no silent eager fallback); on a CPU-only box the
    python ops use their torch reference path (the plumbing tier of the test-suite).
"""
from __future__ import annotations

import ctypes
import hashlib
import os
import shutil
import subprocess
import threading
from pathlib import Path
from typing import Dict, List, Optional

import torch

__all__ = ["KernelLoader", "load", "build_all", "native_available", "launch_counter", "LIBS"]

_HERE = Path(__file__).resolve().parent
CSRC = _HERE / "csrc"
BUILD = _HERE / "_build"

NVCC_FLAGS = [
    "-gencode", "arch=compute_90a,code=sm_90a", "-lineinfo", "-O3", "-std=c++17", "--use_fast_math",
    "--expt-relaxed-constexpr", "--expt-extended-lambda", "-Xcompiler", "-fPIC", "-shared",
    "-U__CUDA_NO_HALF_OPERATORS__", "-U__CUDA_NO_HALF_CONVERSIONS__", "-U__CUDA_NO_BFLOAT16_CONVERSIONS__",
    "-U__CUDA_NO_HALF2_OPERATORS__",
]
CXX_FLAGS = ["-O3", "-std=c++17", "-fPIC", "-shared", "-fopenmp", "-ffast-math", "-fno-finite-math-only"]

# library name -> (sources, kind)
LIBS: Dict[str, dict] = {
    "cb200_elementwise": {"sources": ["elementwise.cu"], "kind": "cuda"},
    "cb200_norm": {"sources": ["norm.cu"], "kind": "cuda"},
    "cb200_optim": {"sources": ["multi_tensor_optim.cu"], "kind": "cuda"},
    "cb200_softmax": {"sources": ["softmax.cu"], "kind": "cuda"},
    "cb200_loss": {"sources": ["cross_entropy.cu"], "kind": "cuda"},
    "cb200_gemm": {"sources": ["gemm_wgmma.cu"], "kind": "cuda"},
    "cb200_grouped_gemm": {"sources": ["grouped_gemm_wgmma.cu"], "kind": "cuda"},
    "cb200_attn": {"sources": ["flash_attn_wgmma.cu"], "kind": "cuda"},
    "cb200_comm": {"sources": ["fused_comm_gemm.cu"], "kind": "cuda"},
    "cb200_moe": {"sources": ["moe.cu"], "kind": "cuda"},
    "cb200_infer": {"sources": ["inference.cu"], "kind": "cuda"},
    "cb200_quant": {"sources": ["quant.cu"], "kind": "cuda"},
    "cb200_wq_gemm": {"sources": ["wq_gemm_wgmma.cu"], "kind": "cuda"},
    "cb200_cpu_adam": {"sources": ["cpu_adam.cpp"], "kind": "cpp"},
    "cb200_aio": {"sources": ["async_file_io.cpp"], "kind": "cpp", "extra": ["-lpthread"]},
}


class _LaunchCounter:
    """Counts launches of OUR kernels (reported by bench.py as `gpu_launches`)."""

    def __init__(self) -> None:
        self.count = 0
        self.by_name: Dict[str, int] = {}
        self.enabled = True

    def add(self, name: str, n: int = 1) -> None:
        if self.enabled:
            self.count += n
            self.by_name[name] = self.by_name.get(name, 0) + n

    def reset(self) -> None:
        self.count = 0
        self.by_name.clear()


launch_counter = _LaunchCounter()
_loaded: Dict[str, ctypes.CDLL] = {}
_lock = threading.Lock()


def _nvcc() -> Optional[str]:
    cand = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    return cand if os.path.exists(cand) else None


def _src_hash(name: str) -> str:
    h = hashlib.sha1()
    spec = LIBS[name]
    for s in spec["sources"]:
        h.update((CSRC / s).read_bytes())
    for hdr in sorted(CSRC.glob("*.cuh")) + sorted(CSRC.glob("*.h")):
        h.update(hdr.read_bytes())
    h.update(" ".join(NVCC_FLAGS if spec["kind"] == "cuda" else CXX_FLAGS).encode())
    return h.hexdigest()[:16]


def lib_path(name: str) -> Path:
    return BUILD / f"lib{name}.so"


def is_stale(name: str) -> bool:
    p, stamp = lib_path(name), BUILD / f"{name}.hash"
    if not p.exists() or not stamp.exists():
        return True
    return stamp.read_text().strip() != _src_hash(name)


def build(name: str, verbose: bool = False, force: bool = False) -> Path:
    spec = LIBS[name]
    srcs = [str(CSRC / s) for s in spec["sources"]]
    for s in srcs:
        if not os.path.exists(s):
            raise FileNotFoundError(s)
    BUILD.mkdir(parents=True, exist_ok=True)
    out = lib_path(name)
    if not force and not is_stale(name):
        return out
    if spec["kind"] == "cuda":
        nvcc = _nvcc()
        if nvcc is None:
            raise RuntimeError("nvcc not found; cannot build CUDA kernels")
        cmd = [nvcc] + NVCC_FLAGS + ["-I", str(CSRC)] + (["-Xptxas", "-v"] if verbose else []) + srcs + \
              ["-o", str(out), "-lcuda"] + spec.get("extra", [])
        # libcuda may be absent on the build box: resolve driver entry points at run time instead
        cmd = [c for c in cmd if c != "-lcuda"]
    else:
        cmd = ["g++"] + CXX_FLAGS + ["-I", str(CSRC)] + srcs + ["-o", str(out)] + spec.get("extra", [])
    tmp = str(out) + f".tmp{os.getpid()}"
    cmd[cmd.index(str(out))] = tmp
    res = subprocess.run(cmd, capture_output=True, text=True)
    if res.returncode != 0:
        raise RuntimeError(f"build of {name} failed:\n{' '.join(cmd)}\n{res.stdout}\n{res.stderr}")
    os.replace(tmp, out)
    (BUILD / f"{name}.hash").write_text(_src_hash(name))
    if verbose:
        print(res.stderr)
    return out


def build_all(verbose: bool = False, force: bool = False, parallel: int = 8) -> List[Path]:
    from concurrent.futures import ThreadPoolExecutor

    names = [n for n, s in LIBS.items() if all((CSRC / x).exists() for x in s["sources"])]
    with ThreadPoolExecutor(max_workers=parallel) as ex:
        return list(ex.map(lambda n: build(n, verbose=verbose, force=force), names))


def native_available(name: str) -> bool:
    """True when the library can be used for CUDA tensors (GPU present and .so present/buildable)."""
    if LIBS[name]["kind"] == "cuda" and not torch.cuda.is_available():
        return False
    return lib_path(name).exists() or all((CSRC / s).exists() for s in LIBS[name]["sources"])


def load(name: str) -> ctypes.CDLL:
    with _lock:
        if name in _loaded:
            return _loaded[name]
        p = lib_path(name)
        if not p.exists() or (is_stale(name) and _nvcc() is not None and os.environ.get("CB200_NO_REBUILD") != "1"):
            try:
                build(name)
            except Exception:
                if not p.exists():
                    raise
        lib = ctypes.CDLL(str(p), mode=ctypes.RTLD_GLOBAL)
        _loaded[name] = lib
        return lib


class KernelLoader:
    """Reference-style façade: `KernelLoader("cb200_norm").load()`."""

    def __init__(self, name: str) -> None:
        if name not in LIBS:
            raise KeyError(f"unknown kernel library {name!r}; known: {list(LIBS)}")
        self.name = name

    def is_available(self) -> bool:
        return native_available(self.name)

    def load(self) -> ctypes.CDLL:
        return load(self.name)


# --------------------------------------------------------------------------------------- ctypes helpers
def ptr(t: Optional[torch.Tensor]) -> ctypes.c_void_p:
    return ctypes.c_void_p(0 if t is None else t.data_ptr())


def stream_ptr() -> ctypes.c_void_p:
    return ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)


def check(err: int, what: str) -> None:
    if err != 0:
        raise RuntimeError(f"{what}: native launcher returned CUDA error {err}")
