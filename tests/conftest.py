import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (run on an H100)")


def pytest_collection_modifyitems(config, items):
    import torch
    if torch.cuda.is_available():
        return
    skip = pytest.mark.skip(reason="no CUDA device in this container")
    for item in items:
        if "gpu" in item.keywords:
            item.add_marker(skip)


@pytest.fixture(scope="session")
def cuda_lib():
    """Build (if needed) and load the C-ABI library; GPU tests call through it."""
    from speech_b200.csrc import build
    build.build()
    from speech_b200 import _lib
    return _lib.load()


@pytest.fixture(autouse=True)
def _reset_grad_plumbing():
    """optim.FlatSGD switches on process-wide hooks of speech_b200.ops (in-place gradient sink,
    grad-ready announcements); no test may leak them into the next one."""
    yield
    from speech_b200 import ops
    ops.set_grad_sink(False)
    ops.set_grad_ready_hook(None)
