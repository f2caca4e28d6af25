import json
import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a real H100 (run with -m gpu)")


@pytest.fixture(scope="session")
def golden():
    with open(os.path.join(ROOT, "tests", "golden", "coast_golden.json")) as f:
        return json.load(f)


@pytest.fixture(scope="session")
def oracle():
    from oracle import pyoracle
    pyoracle.build()
    return pyoracle


@pytest.fixture(scope="session")
def built_lib():
    import coast_b200
    return coast_b200.build_library()


@pytest.fixture(scope="session")
def rt(built_lib):
    """The CUDA path.  No fallback: if the extension or the driver is missing this raises."""
    import coast_b200
    return coast_b200.Runtime(0)
