import importlib.util
import os
import sys
from pathlib import Path

import pytest

ROOT = Path(__file__).resolve().parents[1]
if str(ROOT) not in sys.path:
    sys.path.insert(0, str(ROOT))


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (run on an H100 with -m gpu)")
    config.addinivalue_line("markers", "slow: multi-second CPU test")


@pytest.fixture(scope="session")
def oracle():
    from oracle import oracle as O
    O.lib()
    return O


@pytest.fixture(scope="session")
def ft():
    """The product package (ctypes mirror over libftsgemm.so), loaded from its in-tree directory."""
    import __graft_entry__ as ge
    return ge.load_package()


@pytest.fixture(scope="session")
def cuda():
    import torch
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    return torch
