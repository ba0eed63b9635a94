import os
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (run on an H100 with -m gpu)")


@pytest.fixture(scope="session")
def checker():
    """Strongest CPU checker available: compiled reference (oracle/_ref) or the C restatement."""
    from oracle import checker as ck

    return ck.best()


@pytest.fixture(scope="session")
def port_checker():
    from oracle import checker as ck

    return ck.port()


@pytest.fixture(scope="session")
def gpu():
    """The CUDA library; GPU tests fail loudly (not skip) when it cannot run."""
    from whatshap_b200 import _lib

    assert _lib.device_count() > 0, "no CUDA device visible: GPU tests must run on an H100"
    return _lib


def solve_or_error(fn, prob):
    try:
        return fn(prob), None
    except RuntimeError as e:  # MendelianConflict is a RuntimeError
        return None, str(e)
