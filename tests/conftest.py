import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

GOLD = os.path.join(ROOT, 'tests', 'golden')


def pytest_configure(config):
    config.addinivalue_line('markers', 'gpu: test needs a CUDA device (run on an H100 with -m gpu)')


@pytest.fixture(scope='session')
def oracle():
    """The CPU oracle (test infrastructure).  Built on demand with gcc."""
    from oracle import oracle as orc
    orc.build()
    return orc


@pytest.fixture(scope='session')
def gold_dir():
    return GOLD


@pytest.fixture(scope='session')
def engine():
    import torch
    if not torch.cuda.is_available():
        pytest.skip('no CUDA device')
    from lidar_snow_sim_b200.engine import SnowfallEngine
    eng = SnowfallEngine(0)
    yield eng
    eng.close()
