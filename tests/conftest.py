import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def pytest_configure(config):
    if os.environ.get("PTGNN_TOOLS_LIB"):      # kernel experiments: run the parity tests against another build of the library (tools/)
        from ptgnn_b200 import _native

        _native.LIB_PATH = os.path.join(ROOT, os.environ["PTGNN_TOOLS_LIB"])
    config.addinivalue_line("markers", "gpu: needs a CUDA device (an H100: `-m gpu`)")


def pytest_collection_modifyitems(config, items):
    import torch

    torch.backends.cuda.matmul.allow_tf32 = False       # torch-on-GPU references in the tests are true fp32
    torch.backends.cudnn.allow_tf32 = False

    if torch.cuda.is_available():
        return
    skip = pytest.mark.skip(reason="no CUDA device")
    for item in items:
        if "gpu" in item.keywords:
            item.add_marker(skip)
