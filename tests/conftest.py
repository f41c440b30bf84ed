import os
import sys
from pathlib import Path

import pytest

ROOT = Path(__file__).resolve().parent.parent
if str(ROOT) not in sys.path:
    sys.path.insert(0, str(ROOT))
os.environ.setdefault("MASTER_ADDR", "127.0.0.1")


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA (sm_90a) device; select with -m gpu")


@pytest.fixture(scope="session")
def golden_dir():
    return Path(__file__).resolve().parent / "golden"
