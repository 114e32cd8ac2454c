import os, sys
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (run on an H100 with `pytest -m gpu`)")


@pytest.fixture(scope="session")
def hostsim_lib():
    """CPU stand-in of the C-ABI library (tests only)."""
    from arriba_b200 import _build
    return _build.build_hostsim()


@pytest.fixture(scope="session")
def cuda_lib():
    from arriba_b200 import _build
    return _build.build_product()   # no-op when the library is newer than every source


@pytest.fixture(scope="session")
def worlds(tmp_path_factory):
    import worldutil
    return worldutil.WorldCache(str(tmp_path_factory.mktemp("worlds")))
