import os
import sys

import pytest

os.environ.setdefault("GW_B200_CHECK", "1")  # tests always read the device status word after a forward

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)
GOLDEN = os.path.join(ROOT, "tests", "golden")


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (an H100: run with -m gpu)")
    config.addinivalue_line("markers", "training: the test differentiates through the model (autograd stays enabled)")


def pytest_collection_modifyitems(config, items):
    import torch

    if torch.cuda.is_available():
        return
    skip = pytest.mark.skip(reason="no CUDA device")
    for item in items:
        if "gpu" in item.keywords:
            item.add_marker(skip)


@pytest.fixture(scope="session")
def golden_dir():
    return GOLDEN


@pytest.fixture(autouse=True)
def _inference_by_default(request):
    """Forward-parity tests run like an evaluation loop (autograd off: the tensor-core path); tests of the training step
    mark themselves with `@pytest.mark.training` and get autograd back."""
    import torch

    if "training" in request.keywords:
        yield
        return
    with torch.no_grad():
        yield
