import sys
from pathlib import Path

import pytest

ROOT = Path(__file__).resolve().parents[1]
if str(ROOT) not in sys.path:
    sys.path.insert(0, str(ROOT))


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (an H100; select with `-m gpu`)")


def pytest_collection_modifyitems(config, items):
    """`pytest tests` on a box without a GPU: gpu-marked tests are skipped instead of erroring in their fixtures."""
    try:
        import torch
        have_gpu = torch.cuda.is_available()
    except Exception:
        have_gpu = False
    if have_gpu:
        return
    skip = pytest.mark.skip(reason="needs a CUDA device (H100); run with -m gpu on a machine with one")
    for item in items:
        if "gpu" in item.keywords:
            item.add_marker(skip)


@pytest.fixture(scope="session")
def repo_root():
    return ROOT


@pytest.fixture(scope="session")
def weights_npz():
    return ROOT / "genomad_b200" / "data" / "nn_classifier.npz"


@pytest.fixture(scope="session")
def golden_dir():
    return ROOT / "tests" / "golden"
