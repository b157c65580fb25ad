import os
import sys
from pathlib import Path

import pytest

ROOT = Path(__file__).resolve().parent.parent
for p in (str(ROOT), str(ROOT / "tests")):
    if p not in sys.path:
        sys.path.insert(0, p)


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (run on an H100 with -m gpu)")


def _has_gpu() -> bool:
    if os.environ.get("LCD_FORCE_NO_GPU"):
        return False
    try:
        import torch

        return torch.cuda.is_available()
    except Exception:
        return False


HAS_GPU = _has_gpu()


@pytest.fixture(scope="session")
def has_gpu():
    return HAS_GPU


def pytest_collection_modifyitems(config, items):
    if HAS_GPU:
        return
    skip = pytest.mark.skip(reason="no CUDA device in this container")
    for item in items:
        if "gpu" in item.keywords:
            item.add_marker(skip)
