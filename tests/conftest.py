import os
import sys
from pathlib import Path

import pytest

ROOT = Path(__file__).resolve().parent.parent
if str(ROOT) not in sys.path:
    sys.path.insert(0, str(ROOT))


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a real H100 (run with -m gpu on a GPU machine)")


@pytest.fixture(scope="session")
def oracle():
    from oracle import oracle as O

    O.lib()
    return O


@pytest.fixture(scope="session")
def cuda_dev():
    import torch

    if not torch.cuda.is_available():
        pytest.fail("GPU test selected but no CUDA device is visible (no CPU fallback exists)")
    from ka9q_radio_b200 import capi

    capi.load()
    return torch.device("cuda:0")


def rel_err(a, b):
    """max|a-b| / max|b| : the parity metric of BASELINE.md section 3 (outputs cross zero)."""
    import numpy as np

    den = float(np.abs(b).max())
    return float(np.abs(a - b).max()) / (den if den > 0 else 1.0)
