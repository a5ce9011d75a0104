import os
import subprocess
import sys

import pytest

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if REPO not in sys.path:
    sys.path.insert(0, REPO)


def pytest_configure(config):
    config.addinivalue_line('markers', 'gpu: needs a real H100 (run with -m gpu)')


@pytest.fixture(scope='session')
def oracle():
    """The CPU oracle (C, oracle/eld_oracle.c) behind ctypes.  Test infrastructure only."""
    from tests import oracle_lib
    return oracle_lib.load()


@pytest.fixture(scope='session')
def golden_dir():
    return os.path.join(REPO, 'tests', 'golden')


def has_gpu():
    try:
        import torch
        return torch.cuda.is_available()
    except Exception:
        return False
