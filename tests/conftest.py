import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (an H100)")
    config.addinivalue_line("markers", "small_path: keep the library's default low-latency path for tiny batches")


@pytest.fixture(autouse=True)
def _batched_kernels_by_default(request, monkeypatch):
    """Test batches are tiny, and tiny batches (B * nprobes <= 1024 probe slots) take the library's low-latency path
    (small.cu).  The parity suite is about the batched kernels, so it switches that path off; the tests marked
    `small_path` (tests/test_gpu_small.py) run with the library's default."""
    if "small_path" not in request.keywords:
        monkeypatch.setenv("LGPU_SMALL_SLOTS", "0")
