import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (an H100)")


@pytest.fixture(scope="session")
def oracle():
    from oracle import ef_oracle
    ef_oracle.lib()
    return ef_oracle


@pytest.fixture(scope="session")
def E():
    """The product binding, with the library built if it is missing."""
    import edge_fuse_b200
    from edge_fuse_b200 import build as _b
    if not os.path.exists(edge_fuse_b200.library_path()):
        _b.build()
    edge_fuse_b200.lib()
    return edge_fuse_b200


@pytest.fixture(scope="session")
def gpu(E):
    """GPU tests must run the CUDA path: fail (not skip) when no device is visible."""
    n = E.device_count()
    assert n > 0, f"no CUDA device visible to libcachemap: {E.last_error()}"
    return n
