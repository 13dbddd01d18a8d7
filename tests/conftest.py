import os
import sys

import pytest

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if REPO not in sys.path:
    sys.path.insert(0, REPO)


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs an H100 (sm_90a) GPU; run with -m gpu")


def pytest_collection_modifyitems(config, items):
    import torch
    if torch.cuda.is_available():
        return
    skip = pytest.mark.skip(reason="no CUDA device in this container")
    for item in items:
        if "gpu" in item.keywords:
            item.add_marker(skip)


@pytest.fixture(scope="session")
def built_lib():
    """Path of libcotr_b200.so, (re)built in-tree if sources are newer."""
    from cotr_b200 import build
    return build.build()


@pytest.fixture(scope="session")
def golden_dir():
    return os.path.join(REPO, "tests", "golden")
