import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)
GOLDEN = os.path.join(ROOT, "tests", "golden")
if GOLDEN not in sys.path:
    sys.path.insert(0, GOLDEN)


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: test needs a CUDA device (run with -m gpu on an H100)")
    config.addinivalue_line("markers", "slow: longer CPU test")


@pytest.fixture(scope="session")
def golden_dir():
    return GOLDEN
