import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, 'tests')):
    if p not in sys.path:
        sys.path.insert(0, p)


def pytest_configure(config):
    config.addinivalue_line('markers', 'gpu: needs a CUDA device (an H100: the library is built for sm_90a)')


@pytest.fixture(scope='session')
def golden():
    import torch
    import cases
    return cases.load_golden(cases.GOLDEN_PATH)
