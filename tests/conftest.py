import os
import random
import sys

import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


def pytest_configure(config):
    if not torch.cuda.is_available():
        # the CPU suite runs tiny matmuls: many intra-op threads only add scheduling overhead (and fight with the spawned
        # gloo workers, which use one thread each)
        torch.set_num_threads(min(4, os.cpu_count() or 1))
    config.addinivalue_line("markers", "gpu: test needs a CUDA device (an H100)")
    config.addinivalue_line("markers", "dist: spawns multiple processes (gloo on CPU)")


def pytest_collection_modifyitems(config, items):
    if torch.cuda.is_available():
        return
    skip = pytest.mark.skip(reason="no CUDA device")
    for item in items:
        if "gpu" in item.keywords:
            item.add_marker(skip)


@pytest.fixture(autouse=True)
def fixed_seed():
    torch.manual_seed(1234)
    random.seed(1234)
    yield
