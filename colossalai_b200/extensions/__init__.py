"""Extension registry: one entry per native library, with ahead-of-time (`build_aot`) and on-demand (`build_jit`)
builds and an availability probe.

Parity: reference `extensions/{base_extension.py:8-82 (_Extension ABC), cpp_extension.py:13-138, cuda_extension.py:18-118,
__init__.py:13-25 (ALL_EXTENSIONS)}` — there the builds go through `torch.utils.cpp_extension` + pybind; here every
library is a plain C ABI `.so` compiled by `nvcc -gencode arch=compute_90a,code=sm_90a` (or `g++`) straight into the
source tree and bound with ctypes (`kernel/loader.py`), so the extension objects are thin descriptors over that loader.
"""
from __future__ import annotations

from abc import ABC
from pathlib import Path
from typing import Dict, List

from ..kernel import loader

__all__ = ["_Extension", "CudaExtension", "CppExtension", "ALL_EXTENSIONS", "get_extension", "build_all_extensions"]


class _Extension(ABC):
    def __init__(self, name: str, lib: str, support_aot: bool = True, support_jit: bool = True, priority: int = 1):
        self._name, self._lib = name, lib
        self._support_aot, self._support_jit, self.priority = support_aot, support_jit, priority

    @property
    def name(self) -> str:
        return self._name

    @property
    def lib_name(self) -> str:
        return self._lib

    @property
    def support_aot(self) -> bool:
        return self._support_aot

    @property
    def support_jit(self) -> bool:
        return self._support_jit

    def sources(self) -> List[Path]:
        return [loader.CSRC / s for s in loader.LIBS[self._lib]["sources"]]

    def is_available(self) -> bool:
        """Sources present and the matching compiler on PATH (nvcc cross-compiles sm_90a without a GPU)."""
        import shutil

        kind = loader.LIBS[self._lib]["kind"]
        return all(p.exists() for p in self.sources()) and shutil.which("nvcc" if kind == "cuda" else "g++") is not None

    def assert_compatibility(self) -> None:
        if not self.is_available():
            raise RuntimeError(f"extension {self._name}: sources or compiler missing")

    def build_aot(self) -> Path:
        self.assert_compatibility()
        return loader.build(self._lib)

    def build_jit(self):
        return self.load()

    def load(self):
        return loader.load(self._lib)


class CudaExtension(_Extension):
    """sm_90a CUDA library (`-gencode arch=compute_90a,code=sm_90a -lineinfo -O3`)."""


class CppExtension(_Extension):
    """Host library (`g++ -O3 -march=native -fopenmp`)."""


def _make(name: str, lib: str) -> _Extension:
    cls = CudaExtension if loader.LIBS[lib]["kind"] == "cuda" else CppExtension
    return cls(name, lib)


# reference extension names -> our libraries (plus the ones the reference does not have)
ALL_EXTENSIONS: Dict[str, _Extension] = {n: _make(n, lib) for n, lib in {
    "cpu_adam_x86": "cb200_cpu_adam",
    "cpu_adam_arm": "cb200_cpu_adam",
    "fused_optim_cuda": "cb200_optim",
    "layernorm_cuda": "cb200_norm",
    "moe_cuda": "cb200_moe",
    "scaled_masked_softmax_cuda": "cb200_softmax",
    "scaled_upper_triangle_masked_softmax_cuda": "cb200_softmax",
    "inference_ops_cuda": "cb200_infer",
    "activation_cuda": "cb200_elementwise",
    "cross_entropy_cuda": "cb200_loss",
    "gemm_tcgen05": "cb200_gemm",
    "fused_comm_gemm": "cb200_comm",
    "fp8_quant_cuda": "cb200_quant",
    "async_file_io": "cb200_aio",
}.items() if lib in loader.LIBS}


def get_extension(name: str) -> _Extension:
    return ALL_EXTENSIONS[name]


def build_all_extensions(verbose: bool = False) -> List[Path]:
    """`BUILD_EXT=1 pip install` equivalent: compile every library into the tree."""
    return loader.build_all(verbose=verbose)
