import importlib
import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (an H100: the library is built for sm_90a)")


@pytest.fixture(scope="session")
def pkg():
    return importlib.import_module("microservice-matchmaking_b200")


@pytest.fixture(scope="session")
def oracle():
    mod = importlib.import_module("oracle.oracle")
    mod.build()
    return mod
