import os
import sys
from pathlib import Path

import pytest

ROOT = Path(__file__).resolve().parent.parent
if str(ROOT) not in sys.path:
    sys.path.insert(0, str(ROOT))


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (run on an H100 with -m gpu)")


@pytest.fixture(scope="session", autouse=True)
def _built_library():
    """Build libmm_b200.so when it is missing (nvcc needs no GPU); a library that build() already
    compiled in-tree is used as is."""
    from models_b200 import _cabi

    if not _cabi.LIB_PATH.exists():
        from models_b200.csrc import build

        build.build()
    yield


@pytest.fixture()
def device():
    import torch

    if not torch.cuda.is_available():
        pytest.skip("needs CUDA")
    return torch.device("cuda", 0)
