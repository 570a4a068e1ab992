import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

GOLDEN_DIR = os.path.join(ROOT, 'tests', 'golden')


def pytest_configure(config):
    config.addinivalue_line('markers', 'gpu: needs a CUDA device (an H100: run with -m gpu)')


def golden_files():
    return sorted(f for f in os.listdir(GOLDEN_DIR) if f.endswith('.npz')) if os.path.isdir(GOLDEN_DIR) else []


@pytest.fixture(scope='session')
def oracle_lib():
    from oracle import oracle
    oracle.build()
    return oracle
