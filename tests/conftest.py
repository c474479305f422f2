import os
import sys

import numpy as np
import pytest

# several replicas on ONE GPU (tests/test_data_parallel_one_gpu.py) wait for each other inside kernels: every stream needs its
# own hardware queue, otherwise a kernel can be queued behind the one that waits for it (must be set before CUDA initialises)
os.environ.setdefault("CUDA_DEVICE_MAX_CONNECTIONS", "32")

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs an H100 (sm_90a); run with -m gpu on a machine that has one")


def _have_gpu() -> bool:
    try:
        import shifu_tensorflow_b200 as sb
        return sb.capi.device_count() > 0
    except Exception:
        return False


_HAVE_GPU = None


def pytest_collection_modifyitems(config, items):
    global _HAVE_GPU
    gpu_items = [it for it in items if "gpu" in it.keywords]
    if not gpu_items:
        return
    if _HAVE_GPU is None:
        _HAVE_GPU = _have_gpu()
    if not _HAVE_GPU:
        skip = pytest.mark.skip(reason="no sm_90 GPU on this machine")
        for it in gpu_items:
            it.add_marker(skip)


def bf16_round(a: np.ndarray) -> np.ndarray:
    """fp32 -> nearest-even bf16 -> fp32 (what __float2bfloat16_rn does)."""
    a = np.ascontiguousarray(a, dtype=np.float32)
    u = a.view(np.uint32).astype(np.uint64)
    u = (u + 0x7FFF + ((u >> 16) & 1)) & 0xFFFF0000
    return u.astype(np.uint32).view(np.float32).reshape(a.shape)


@pytest.fixture(scope="session")
def sb():
    import shifu_tensorflow_b200 as m
    return m
