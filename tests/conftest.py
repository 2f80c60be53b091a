import os
import sys

import numpy as np
import pytest

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if REPO not in sys.path:
    sys.path.insert(0, REPO)

GOLDEN = os.path.join(REPO, 'tests', 'golden')


def pytest_configure(config):
    config.addinivalue_line('markers', 'gpu: needs a CUDA device (an H100; run with -m gpu)')


def load_golden(name):
    return np.load(os.path.join(GOLDEN, name + '.npz'))


@pytest.fixture(scope='session')
def golden():
    return load_golden
