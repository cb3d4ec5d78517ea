import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "oracle"))


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: test needs a CUDA device (an H100, sm_90a)")


@pytest.fixture(scope="session")
def oracle():
    import vloracle
    vloracle.lib()
    return vloracle
