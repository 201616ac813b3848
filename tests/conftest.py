import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

GOLDEN = os.path.join(ROOT, 'tests', 'golden')


def pytest_configure(config):
    config.addinivalue_line('markers', 'gpu: needs a CUDA H100 device (select with -m gpu)')


def reference_golden():
    """Outputs of the unmodified reference (naver/dust3r) for the tests that compare with it, stored by
    tests/golden/make_reference_golden.py."""
    import numpy as np
    return np.load(os.path.join(GOLDEN, 'reference_live.npz'))


@pytest.fixture(scope='session')
def cuda_device():
    import torch
    if not torch.cuda.is_available():
        pytest.skip('no CUDA device')
    return torch.device('cuda:0')
