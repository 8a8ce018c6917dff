import os
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)
GOLDEN = os.path.join(ROOT, 'tests', 'golden')


def pytest_configure(config):
    config.addinivalue_line('markers', 'gpu: needs a CUDA device (run on the H100 box with -m gpu)')
    # make sure the C-ABI library matches the sources in the tree (no-op when the build stamp is current;
    # falls back to the prebuilt .so when no nvcc is available)
    from parl_b200.build import build
    build()


@pytest.fixture(scope='session')
def golden():
    def _load(name):
        return np.load(os.path.join(GOLDEN, name + '.npz'), allow_pickle=False)
    return _load


def has_cuda():
    try:
        import torch
        return torch.cuda.is_available()
    except Exception:
        return False
