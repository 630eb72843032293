import os
import sys
from pathlib import Path

import pytest

ROOT = Path(__file__).resolve().parents[1]
if str(ROOT) not in sys.path:
    sys.path.insert(0, str(ROOT))


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA H100 (compute capability 9.0)")


@pytest.fixture(scope="session")
def golden():
    import numpy as np
    return np.load(ROOT / "tests" / "golden" / "reference_vectors.npz")


@pytest.fixture(scope="session")
def lib_built():
    """The C-ABI library, built on demand (nvcc cross-compiles without a GPU)."""
    sys.path.insert(0, str(ROOT))
    import __graft_entry__ as g
    if not g.LIB.exists():
        g.build()
    return g.LIB
