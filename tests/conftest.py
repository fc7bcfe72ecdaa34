import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (run on an H100 with -m gpu)")


def _has_gpu():
    try:
        from mitsuba_b200 import api
        return api.device_count() > 0
    except Exception:
        return False


@pytest.fixture(scope="session")
def b2ctx():
    from mitsuba_b200 import api
    if not _has_gpu():
        pytest.fail("GPU test selected but no CUDA device / libb2mts.so: the product has no CPU fallback")
    ctx = api.Context(0)
    yield ctx
    ctx.close()
