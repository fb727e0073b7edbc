import os
import subprocess
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (run with -m gpu)")


@pytest.fixture(scope="session", autouse=True)
def _build_test_infrastructure():
    # the oracle and the test-only host build of the kernel functors (never loaded by the product)
    subprocess.check_call(["make", "-s", "-C", os.path.join(ROOT, "oracle")])
    subprocess.check_call(["make", "-s", "-C", os.path.join(ROOT, "tests", "hostsim")])
    yield
