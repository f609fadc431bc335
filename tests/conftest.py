import os
import sys
from pathlib import Path

import pytest

ROOT = Path(__file__).resolve().parent.parent
if str(ROOT) not in sys.path:
    sys.path.insert(0, str(ROOT))


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a real H100 (run with -m gpu)")


def _has_gpu():
    try:
        import torch
        return torch.cuda.is_available()
    except Exception:
        return False


@pytest.fixture(scope="session")
def blob():
    from headtrackr_b200 import load_cascade_blob
    return load_cascade_blob()


@pytest.fixture(scope="session")
def ctx():
    """One C-ABI context for the whole GPU session.  Fails loudly when the CUDA library cannot be used."""
    if not _has_gpu():
        pytest.fail("gpu-marked test selected but no CUDA device is visible")
    from headtrackr_b200 import Context
    c = Context(max_width=1280, max_height=720, max_frames=16, max_raw_per_frame=4096)
    yield c
    c.close()
