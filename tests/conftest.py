import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (run with -m gpu on an H100)")


@pytest.fixture(scope="session", autouse=True)
def _build_everything():
    """Build the CUDA library (nvcc cross-compiles without a GPU), the CPU checkers and the host KAT binaries once."""
    from urban_road_filter_b200 import build
    build.build_lib()
    build.build_oracle()
    build.build_kat()
    build.build_glue()
    yield
