import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

GOLDEN = os.path.join(ROOT, "tests", "golden")


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (H100)")
    # The oracle's ARPACK / BLAS problems are 511 x 511: on a 200-thread GPU host the default
    # thread pool only spins (test_c3_cs_and_sweep: 77 oracle eigenvalues took 100-380 s
    # depending on the box, 5 s per eigsh call; 0.03 s with one thread).
    try:
        from threadpoolctl import threadpool_limits
        config._sb_blas_limit = threadpool_limits(limits=4)
    except Exception:           # noqa: BLE001 -- test speed only
        pass


@pytest.fixture(scope="session")
def golden_dir():
    return GOLDEN
