"""pytest configuration: registers the `gpu` marker and puts the repo root on sys.path.

`-m "not gpu"` runs everywhere (oracle vs golden vectors, host logic, C-ABI symbols);
`-m gpu` needs an H100 and calls the CUDA kernels through the C-ABI.
"""
import os
import sys

import pytest

ROOT = os.path.abspath(os.path.join(os.path.dirname(__file__), ".."))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

GOLDEN = os.path.join(ROOT, "tests", "golden")


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (an H100)")


@pytest.fixture(scope="session")
def golden_dir():
    return GOLDEN
