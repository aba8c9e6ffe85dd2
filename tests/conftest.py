import json
import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


try:  # the oracle's torch-CPU ops oversubscribe badly on many-core shared hosts
    import torch
    torch.set_num_threads(min(8, os.cpu_count() or 1))
except Exception:
    pass


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (an H100; select with -m gpu)")


@pytest.fixture(scope="session")
def kats():
    with open(os.path.join(ROOT, "tests", "golden", "reference_kats.json")) as f:
        return json.load(f)
