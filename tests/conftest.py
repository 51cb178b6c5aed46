import os
import sys

import pytest

# tests/test_sharding_gpu.py runs two ranks of the peer exchange in ONE process on one GPU: a rank that has to lazily load a
# kernel while the other rank spins inside the exchange would wait for it forever (CUDA lazy loading synchronises the
# context).  Eager loading must be chosen before CUDA initialises; separate processes / GPUs (the real layout) are unaffected.
os.environ["CUDA_MODULE_LOADING"] = "EAGER"

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs an H100 (sm_90a); select with -m gpu")


@pytest.fixture(scope="session")
def pkg():
    import __graft_entry__ as g
    return g.load_package()


@pytest.fixture(scope="session")
def oracle():
    import oracle_lib
    oracle_lib.lib()
    return oracle_lib


@pytest.fixture(scope="session")
def ctx(pkg):
    """One b200rl context on cuda:0 — fails loudly (no fallback) when the GPU or the .so is missing."""
    c = pkg.Context(0)
    yield c
    c.close()
