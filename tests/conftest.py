import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs an H100 (run with -m gpu)")


@pytest.fixture(scope="session")
def cuda():
    import torch
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    from speecht5_b200 import _lib
    lib = _lib.load()
    assert lib.st5_device_ok() == 0, lib.st5_last_error()
    return torch.device("cuda")


@pytest.fixture(autouse=True)
def _reset_runtime_hints():
    """Process-wide hints a B200Trainer leaves behind (it owns model + criterion, so it may tell the attention backward
    that only the first n heads of the returned probabilities carry a gradient) must not leak into the next test."""
    yield
    try:
        from speecht5_b200.ops import RT
        RT.probs_grad_heads = 0
        RT.probs_read_heads = 0
        RT.stage_callback = None
        RT.clear_static()  # (flat-buffer views keyed by id(parameter): a later test's parameters may reuse the ids)
        RT.wgrad_stream = None
        RT._side_keep.clear()
    except Exception:  # noqa: BLE001  (package not importable in a collection-only run)
        pass
