import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def pytest_configure(config):
    import torch

    # the oracle's torch-CPU convs crawl when 128+ host threads fight over small layers (GPU box): cap the pool
    torch.set_num_threads(max(1, min(16, os.cpu_count() or 1)))
    config.addinivalue_line("markers", "gpu: needs a CUDA device (run on an H100 with -m gpu)")


@pytest.fixture(scope="session")
def built_lib():
    """Build (incrementally) and load liby5b200.so; the GPU box receives the prebuilt .so with the snapshot."""
    from yolov5_b200 import _lib, build

    if not os.path.exists(_lib.LIB_PATH):
        build.build()
    return _lib.lib()


@pytest.fixture(scope="session")
def cuda(built_lib):
    import torch

    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    return torch.device("cuda:0")
