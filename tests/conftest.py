import json
import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a real H100 (run with -m gpu)")


@pytest.fixture(scope="session")
def kats():
    with open(os.path.join(ROOT, "tests", "golden", "reference_kats.json")) as f:
        return json.load(f)


@pytest.fixture(scope="session")
def oracle_mod():
    import oracle
    oracle.build()
    return oracle


@pytest.fixture(scope="session")
def knn_lib():
    """The CUDA library, built in-tree.  Never replaced by a CPU path."""
    from nornicdb_b200 import _lib, build
    build.build()
    return _lib.load()


@pytest.fixture(scope="session")
def gpu_device(knn_lib):
    from nornicdb_b200 import cuda
    if not cuda.IsAvailable():
        pytest.fail("-m gpu tests need a CUDA device; none is visible")
    dev = cuda.NewDevice(0)
    yield dev
    dev.Release()
