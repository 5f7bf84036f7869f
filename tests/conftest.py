import glob
import os
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)
GOLDEN = os.path.join(ROOT, "tests", "golden")


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (an H100: the kernels are built for sm_90a)")


def pytest_collection_modifyitems(config, items):
    import torch

    if torch.cuda.is_available():
        return
    skip = pytest.mark.skip(reason="no CUDA device")
    for item in items:
        if "gpu" in item.keywords:
            item.add_marker(skip)


@pytest.fixture(scope="session", autouse=True)
def _built():
    """CPU-side build products every test may rely on: the product library (cross-compiled)
    and the oracle."""
    from det3d_b200 import build as d3b_build
    from oracle import build as oracle_build

    d3b_build.build()
    oracle_build.build()


def golden_voxel_cases():
    return sorted(os.path.basename(p)[len("voxel_"):-len(".npz")] for p in glob.glob(os.path.join(GOLDEN, "voxel_*.npz")))


def load_golden(name):
    return dict(np.load(os.path.join(GOLDEN, name + ".npz")))
