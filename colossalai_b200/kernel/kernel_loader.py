"""`KernelLoader` façade over the native library loader.

Parity: reference `colossalai/kernel/kernel_loader.py:32-120` (`KernelLoader.load()` picks the first available
extension for the device; one subclass per kernel family).  Here every family maps to one in-tree sm_90a library
(`kernel/loader.py`); `load()` returns the ctypes handle and raises if the library cannot be built/loaded.
"""
from __future__ import annotations

from typing import List

from . import loader

__all__ = ["KernelLoader", "CPUAdamLoader", "FusedOptimizerLoader", "LayerNormLoader", "MoeLoader",
           "ScaledMaskedSoftmaxLoader", "ScaledUpperTriangleMaskedSoftmaxLoader", "InferenceOpsLoader",
           "FlashAttentionLoader", "FlashAttentionWithCustomMaskLoader", "FlashAttentionForFloatAndCustomMaskLoader",
           "GemmLoader", "FusedCommLoader", "QuantLoader"]


class KernelLoader:
    """`KernelLoader().load()` -> handle of the first usable library in `LIBS`."""

    LIBS: List[str] = []

    def __init__(self) -> None:
        self._lib = None

    def fetch_kernel(self, lib_name: str = None):
        names = [lib_name] if lib_name else list(self.LIBS)
        errors = []
        for n in names:
            try:
                return loader.load(n)
            except Exception as e:  # try the next candidate
                errors.append(f"{n}: {e}")
        raise RuntimeError(f"No usable kernel found for {type(self).__name__} on the current machine: {errors}")

    def load(self, ext_name: str = None):
        if self._lib is None:
            self._lib = self.fetch_kernel(ext_name)
        return self._lib

    @classmethod
    def is_available(cls) -> bool:
        try:
            return all(loader.lib_path(n).exists() or loader.build(n) for n in cls.LIBS)
        except Exception:
            return False


class CPUAdamLoader(KernelLoader):
    LIBS = ["cb200_cpu_adam"]


class FusedOptimizerLoader(KernelLoader):
    LIBS = ["cb200_optim"]


class LayerNormLoader(KernelLoader):
    LIBS = ["cb200_norm"]


class MoeLoader(KernelLoader):
    LIBS = ["cb200_moe"]


class ScaledMaskedSoftmaxLoader(KernelLoader):
    LIBS = ["cb200_softmax"]


class ScaledUpperTriangleMaskedSoftmaxLoader(KernelLoader):
    LIBS = ["cb200_softmax"]


class InferenceOpsLoader(KernelLoader):
    LIBS = ["cb200_infer"]


class GemmLoader(KernelLoader):
    LIBS = ["cb200_gemm"]


class FusedCommLoader(KernelLoader):
    LIBS = ["cb200_comm"]


class QuantLoader(KernelLoader):
    LIBS = ["cb200_quant"]


class FlashAttentionLoader(KernelLoader):
    """Attention dispatch: returns a callable `(q, k, v, **kw)` over token-major tensors (`ops.attention`)."""

    def load(self, ext_name: str = None):
        from ..ops import attention

        return attention


class FlashAttentionWithCustomMaskLoader(FlashAttentionLoader):
    pass


class FlashAttentionForFloatAndCustomMaskLoader(FlashAttentionLoader):
    pass
