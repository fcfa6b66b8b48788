import os
import sys

import pytest

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
os.environ.setdefault("MASTER_ADDR", "127.0.0.1")


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: test needs a CUDA device (an H100)")
    config.addinivalue_line("markers", "dist: spawns multiple processes (gloo on CPU, NCCL on GPU)")


@pytest.fixture(autouse=True)
def _clear_cuda_cache():
    yield
    try:
        import torch

        if torch.cuda.is_available():
            torch.cuda.empty_cache()
    except Exception:
        pass
