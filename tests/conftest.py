import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests", "emul"))
DATA = os.path.join(ROOT, "tests", "data")
# thread emulator of the CPU suite (tests/emul): a launch that makes no progress for this many seconds dumps what every
# lane waits on and aborts, instead of hanging the suite
os.environ.setdefault("JB_EMUL_WATCHDOG", "900")


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (run on an H100 with -m gpu)")


@pytest.fixture(scope="session")
def data_dir():
    return DATA


def has_cuda() -> bool:
    try:
        import torch
        return torch.cuda.is_available()
    except Exception:
        return False
