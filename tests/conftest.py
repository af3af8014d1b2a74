import os
import sys

import pytest
import torch

# The CPU oracle is eager PyTorch on small GEMMs: it collapses on a 100+ core host (barrier overhead); 16 is plenty.
torch.set_num_threads(max(1, min(16, os.cpu_count() or 1)))

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (run on an H100 with -m gpu)")
    config.addinivalue_line("markers", "slow: multi-second CPU test (large model presets)")


@pytest.fixture(scope="session")
def golden_dir():
    return os.path.join(ROOT, "tests", "golden")
