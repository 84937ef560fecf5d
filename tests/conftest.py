import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs an H100 (sm_90a); run with -m gpu")


@pytest.fixture(scope="session")
def oracle_built():
    """Build the CPU oracles (the C restatement; oracle/_ref too where the reference sources are present)."""
    from oracle import pyoracle
    if not pyoracle.available("port") or (pyoracle.reference_present() and not pyoracle.available("ref")):
        pyoracle.build()
    return pyoracle
