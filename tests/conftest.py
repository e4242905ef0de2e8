import importlib
import os
import sys

import pytest

ROOT = os.path.abspath(os.path.join(os.path.dirname(__file__), ".."))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (run on an H100 with -m gpu)")


@pytest.fixture(scope="session")
def syn():
    return importlib.import_module("pretrain-gnns_b200.synthetic")


@pytest.fixture(scope="session")
def pkg():
    return importlib.import_module("pretrain-gnns_b200")
