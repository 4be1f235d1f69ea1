import importlib
import os
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs an H100 (sm_90) GPU")


def _have_h100():
    try:
        import torch
        return torch.cuda.is_available() and torch.cuda.get_device_capability(0) == (9, 0)
    except Exception:
        return False


def pytest_collection_modifyitems(config, items):
    """a plain `pytest` on a machine without an sm_90 GPU skips the gpu-marked tests instead of erroring in the fixture
    (the product itself still fails loudly there: tests/test_abi.py::test_create_fails_loudly_without_gpu)."""
    if _have_h100():
        return
    skip = pytest.mark.skip(reason="needs an H100 (sm_90) GPU")
    for it in items:
        if "gpu" in it.keywords:
            it.add_marker(skip)


@pytest.fixture(scope="session")
def npe():
    return importlib.import_module("neural-photo-editor_b200")


@pytest.fixture(scope="session")
def golden():
    return dict(np.load(os.path.join(ROOT, "tests", "golden", "ian_simple_golden.npz")))


@pytest.fixture(scope="session")
def weights(golden):
    from oracle import weights as ow
    return ow.make_simple_weights(int(golden["weight_seed"]))


@pytest.fixture(scope="session")
def model(npe, weights):
    """the product: API.IAN on cuda:0 through the C-ABI library (GPU tests only)."""
    m = npe.IAN("IAN_simple.py", dnn=True, weights=weights, device=0)
    yield m
    m.close()
