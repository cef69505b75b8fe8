import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: test needs a CUDA device (run on the H100 with -m gpu)")


@pytest.fixture(scope="session")
def orc():
    from oracle import orc as _orc
    _orc.build()
    return _orc


@pytest.fixture(scope="session")
def synth():
    import dmvio_b200.synth as s
    return s
