import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs an H100 (sm_90a); run with -m gpu on a machine that has one")


@pytest.fixture(scope="session")
def oracle():
    from oracle import oracle as o
    o.build()
    return o


@pytest.fixture(scope="session")
def ctx():
    from kaito_b200 import _native
    c = _native.Context(device_id=0)
    yield c
    c.close()


@pytest.fixture(scope="session")
def ctx_scan():
    """context pinned to the exact fp32 scan kernel (K1)"""
    from kaito_b200 import _native
    c = _native.Context(device_id=0, dense_mode=_native.DENSE_SCAN)
    yield c
    c.close()
