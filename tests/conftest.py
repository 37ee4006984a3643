import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (H100, sm_90a)")
    config.addinivalue_line("markers", "slow: long-running CPU test")


@pytest.fixture(scope="session")
def report_dir():
    d = os.path.join(ROOT, "gpurun_out")
    os.makedirs(d, exist_ok=True)
    return d
