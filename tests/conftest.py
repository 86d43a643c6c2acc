import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (run with -m gpu on an H100)")


@pytest.fixture(scope="session")
def oracle():
    from oracle_lib import Oracle, build_oracle
    build_oracle()
    return Oracle()


@pytest.fixture(scope="session")
def reflib():
    from oracle_lib import RefLib
    if not RefLib.available():
        pytest.skip("oracle/_ref/libeigenmat_ref.so not built (needs /root/reference)")
    return RefLib()
