"""Ahead-of-time build of the two native extensions the reference's own benchmark optimizer (`HybridAdam`,
`examples/language/llama/benchmark.py`) loads: `cpu_adam_x86` and `fused_optim_cuda`.

This is the reference's own `BUILD_EXT=1` recipe (`setup.py:72-96`: `ext.build_aot()` for every extension) restricted to
those two, executed against the UNMODIFIED sources installed in `baseline/_ref`; the built modules land in
`baseline/_ref/colossalai/_C/` where the reference's `KernelLoader` looks first (`extensions/cpp_extension.py:57-61,130`).
There is no GPU on the build box, so the arch list is pinned to sm_90 (the cross-compile branch of the reference's
`set_cuda_arch_list` only knows architectures up to 8.6) and `torch.cuda.get_device_capability` is answered with (9, 0)
for `get_cuda_cc_flag()`.  `-march=native` of the CPU Adam is replaced by an explicit `-march=x86-64-v3` (AVX2) so the
binary does not depend on the build host's CPU.

    python baseline/build_ref_ext.py          # idempotent; ~3-6 minutes of nvcc
"""
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
REF = os.path.join(ROOT, "baseline", "_ref")


def main() -> int:
    out_dir = os.path.join(REF, "colossalai", "_C")
    want = ["cpu_adam_x86", "fused_optim_cuda"]
    if all(any(f.startswith(n) and f.endswith(".so") for f in os.listdir(out_dir)) for n in want) \
            and "--force" not in sys.argv:
        print("[build_ref_ext] already built:", sorted(os.listdir(out_dir)))
        return 0
    os.environ.setdefault("FORCE_CUDA", "1")
    os.environ.setdefault("TORCH_CUDA_ARCH_LIST", "9.0")
    os.environ.setdefault("MAX_JOBS", str(os.cpu_count() or 4))
    sys.path[:] = [p for p in sys.path if os.path.abspath(p or ".") != ROOT]
    sys.path.insert(0, REF)
    sys.path.insert(0, os.path.join(ROOT, "baseline"))
    import reference_arm as ra          # stub finder for the packages the reference hard-imports

    sys.meta_path.append(ra._StubFinder())
    import torch

    if not torch.cuda.is_available():
        torch.cuda.get_device_capability = lambda *a, **k: (9, 0)      # cross-compiling for the H100 boxes
        torch.cuda.get_arch_list = lambda: ["sm_90"]
    from setuptools import setup
    from torch.utils.cpp_extension import BuildExtension

    from colossalai.kernel.extensions.pybind.cpu_adam import CpuAdamX86Extension
    from colossalai.kernel.extensions.pybind.optimizer import FusedOptimizerCudaExtension

    mods = []
    for cls in (CpuAdamX86Extension, FusedOptimizerCudaExtension):
        ext = cls()
        ext.assert_compatible()
        m = ext.build_aot()
        for key in ("cxx", "nvcc"):
            m.extra_compile_args[key] = [("-march=x86-64-v3" if a == "-march=native" else a)
                                         for a in m.extra_compile_args[key]]
        mods.append(m)
    build_tmp = os.path.join(ROOT, "baseline", "_build_tmp")
    setup(name="colossalai_ref_ext", ext_modules=mods, cmdclass={"build_ext": BuildExtension.with_options(use_ninja=True)},
          script_args=["build_ext", "--build-lib", REF, "--build-temp", build_tmp])
    print("[build_ref_ext] built:", sorted(os.listdir(out_dir)))
    return 0


if __name__ == "__main__":
    sys.exit(main())
