import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

# lets tests install oracle/ref_ops.py as the op table of pydreamer_b200 (never set by product code)
os.environ.setdefault("PD_B200_TESTING", "1")


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA sm_90a (H100) device")


def pytest_collection_modifyitems(config, items):
    """`gpu`-marked tests need an sm_90a device: on a box without CUDA a plain `pytest tests` skips them instead of
    failing inside torch's CUDA initialisation."""
    import torch

    if torch.cuda.is_available():
        return
    skip = pytest.mark.skip(reason="needs a CUDA sm_90a (H100) device")
    for item in items:
        if "gpu" in item.keywords:
            item.add_marker(skip)


@pytest.fixture(scope="session")
def native_ops():
    import torch

    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    from pydreamer_b200.ops import NativeOps

    return NativeOps("cuda:0")
