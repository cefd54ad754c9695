import os
import sys

# cuSOLVER's host stages use OpenMP; these must be in the environment before libgomp is loaded (i.e. before torch is
# imported by any test module) -- see dftk_b200/__init__.py
os.environ.setdefault("OMP_WAIT_POLICY", "passive")

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: test needs a CUDA device (an H100, sm_90a)")
    config.addinivalue_line("markers", "slow: longer CPU test")
