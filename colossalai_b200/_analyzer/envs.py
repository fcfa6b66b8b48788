"""Hardware constants the analyzers price things with (reference `_analyzer/envs.py` `MeshConfig`: TFLOPS, bandwidth,
PCIe).  Defaults are one GPU inside an NVSwitch domain; `from_measured` reads the repo's `MEASURED_PEAKS.json`."""
from __future__ import annotations

import json
import os
from dataclasses import dataclass

__all__ = ["MeshConfig"]


@dataclass
class MeshConfig:
    TFLOPS: float = 1400.0            # dense bf16 through cuBLAS (measured order of magnitude; nominal 2250)
    BANDWIDTH: float = 6.0e12         # HBM3e copy bytes/s (nominal 7.7e12)
    NVLINK_BANDWIDTH: float = 770e9   # per direction through NVSwitch
    PCIE_BANDWIDTH: float = 55e9      # host <-> device, Gen5 x16 effective
    HBM_BYTES: float = 180e9

    @staticmethod
    def from_measured(path: str = "MEASURED_PEAKS.json") -> "MeshConfig":
        cfg = MeshConfig()
        if os.path.exists(path):
            with open(path) as f:
                d = json.load(f)
            for k, v in d.items():
                if not isinstance(v, (int, float)):
                    continue
                lk = k.lower()
                if "tflop" in lk and "bf16" in lk:
                    cfg.TFLOPS = float(v)
                elif "copy" in lk or "hbm" in lk:
                    cfg.BANDWIDTH = float(v) * (1e9 if v < 1e6 else 1.0)
        return cfg
