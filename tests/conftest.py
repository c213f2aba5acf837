import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (an H100)")
    config.addinivalue_line("markers", "reference: needs the read-only reference at /root/reference")


@pytest.fixture(scope="session")
def golden_dir():
    return os.path.join(ROOT, "tests", "golden")


@pytest.fixture(scope="session")
def native_lib():
    """Build (if needed) and dlopen the C-ABI library; no GPU required for this."""
    from torchrl_b200 import build, _lib
    if not os.path.exists(build.LIBPATH):
        build.build()
    return _lib.load()


def pytest_collection_modifyitems(config, items):
    from oracle import reference_loader
    if not reference_loader.available():
        skip = pytest.mark.skip(reason="/root/reference not present on this box")
        for it in items:
            if "reference" in it.keywords:
                it.add_marker(skip)
