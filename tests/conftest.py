import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

GOLDEN = os.path.join(ROOT, "tests", "golden")


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA GPU (an H100, sm_90a; select with -m gpu)")
    # CPU oracle legs of the GPU tests: use the cores this process really has (cgroup quota), not the node's
    try:
        import torch
        from ln3diff_b200.utils import host_cores
        torch.set_num_threads(host_cores())
    except Exception:
        pass


@pytest.fixture(scope="session")
def golden():
    import numpy as np

    def load(name):
        return np.load(os.path.join(GOLDEN, name))
    return load


@pytest.fixture(scope="session")
def built_lib():
    """The in-tree CUDA library (nvcc cross-compiles without a GPU)."""
    from ln3diff_b200 import build
    return build.build()
