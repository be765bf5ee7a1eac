import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

GOLDEN = os.path.join(ROOT, "tests", "golden")


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (run with -m gpu on a machine with an H100)")


@pytest.fixture(scope="session")
def golden():
    import numpy as np

    def load(name):
        return np.load(os.path.join(GOLDEN, name))
    return load


@pytest.fixture(scope="session")
def golden_json():
    import json

    def load(name):
        with open(os.path.join(GOLDEN, name)) as fh:
            return json.load(fh)
    return load


@pytest.fixture(scope="session")
def cuda():
    import torch
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    # the product path has no fallback: the extension must be the thing that runs
    from d3feat_b200 import _lib
    _lib.lib()
    return torch.device("cuda", 0)
