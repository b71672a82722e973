import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (an H100)")


@pytest.fixture(scope="session")
def golden():
    import numpy as np

    return np.load(os.path.join(ROOT, "tests", "golden", "elodin_ci_baseline.npz"))


@pytest.fixture(scope="session")
def oracle():
    """The CPU oracle (test infrastructure).  Built on demand with gcc."""
    from oracle import oracle as O

    O.build()
    O.set_dot_mode(0)
    return O


@pytest.fixture(scope="session", autouse=True)
def _built_extension():
    """Test harness convenience: compile libb200_sixdof.so in-tree if it is not there yet (nvcc
    cross-compiles without a GPU).  The product itself never builds or falls back on demand."""
    import subprocess

    so = os.path.join(ROOT, "elodin_b200", "libb200_sixdof.so")
    if not os.path.exists(so):
        subprocess.run(["make", "-s", "-C", os.path.join(ROOT, "elodin_b200", "csrc")], check=True)
