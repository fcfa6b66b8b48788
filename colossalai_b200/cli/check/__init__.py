"""`colossalai_b200 check -i`: installation report.  Parity: reference `colossalai/cli/check/check_installation.py`."""
from __future__ import annotations

import argparse
import subprocess

__all__ = ["add_check_parser", "check_installation"]


def _nvcc_version() -> str:
    try:
        out = subprocess.run(["nvcc", "--version"], capture_output=True, text=True, timeout=20).stdout
        for tok in out.replace(",", " ").split():
            if tok.startswith("V") and tok[1:2].isdigit():
                return tok[1:]
    except Exception:
        pass
    return "N/A"


def check_installation() -> dict:
    import torch

    from ... import __version__ as ver
    from ...kernel import loader

    built = {name: loader.lib_path(name).exists() for name in loader.LIBS}
    info = {
        "colossalai_b200": ver,
        "torch": torch.__version__,
        "torch CUDA": torch.version.cuda,
        "system CUDA (nvcc)": _nvcc_version(),
        "CUDA available": torch.cuda.is_available(),
        "device": torch.cuda.get_device_name(0) if torch.cuda.is_available() else "N/A",
        "compute capability": ".".join(map(str, torch.cuda.get_device_capability(0))) if torch.cuda.is_available() else "N/A",
        "NCCL": ".".join(map(str, torch.cuda.nccl.version())) if torch.cuda.is_available() else "N/A",
        "native libraries built": f"{sum(built.values())}/{len(built)}",
        "missing native libraries": [k for k, v in built.items() if not v],
    }
    return info


def _run(args: argparse.Namespace, extra) -> int:
    if not args.installation:
        print("Usage: colossalai_b200 check -i")
        return 0
    info = check_installation()
    print("#### Installation Report ####")
    for k, v in info.items():
        print(f"{k}: {v}")
    if info["torch CUDA"] and info["system CUDA (nvcc)"] != "N/A":
        same = info["system CUDA (nvcc)"].split(".")[0] == str(info["torch CUDA"]).split(".")[0]
        print(f"CUDA major version match (system vs torch): {'yes' if same else 'NO'}")
    print("Target architecture: sm_90a (kernels are compiled with -gencode arch=compute_90a,code=sm_90a)")
    return 0


def add_check_parser(sub) -> None:
    p = sub.add_parser("check", help="check the installation")
    p.add_argument("-i", "--installation", action="store_true", help="print the installation report")
    p.set_defaults(func=_run)
