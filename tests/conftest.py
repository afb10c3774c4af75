import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: test needs a CUDA device (an H100: the library is built for sm_90a)")


@pytest.fixture(scope="session")
def oracle_mod():
    import oracle
    oracle.build()
    return oracle


@pytest.fixture(scope="session")
def gpu_ctx():
    from jepsen_tigerbeetle_b200 import native
    ctx = native.Context(device=0)
    yield ctx
    ctx.close()
