import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (an H100; select with -m gpu)")


def _have_gpu():
    try:
        from opencorr_b200 import _capi
        return _capi.load().ocb_device_count() > 0
    except Exception:
        return False


HAVE_GPU = _have_gpu() or bool(os.environ.get("OCB_TEST_FAKE_GPU"))  # the env switch is for dry runs of the test logic only


def pytest_collection_modifyitems(config, items):
    if HAVE_GPU:
        return
    skip = pytest.mark.skip(reason="no CUDA device in this process")
    for item in items:
        if "gpu" in item.keywords:
            item.add_marker(skip)


@pytest.fixture(scope="session")
def engine():
    import opencorr_b200 as ob
    return ob.default_engine(0)
