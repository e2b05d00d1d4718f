import os
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (an H100)")


def _has_gpu():
    try:
        import torch

        return torch.cuda.is_available()
    except Exception:
        return False


def pytest_collection_modifyitems(config, items):
    if _has_gpu():
        return
    skip = pytest.mark.skip(reason="no CUDA device in this container")
    for item in items:
        if "gpu" in item.keywords:
            item.add_marker(skip)


@pytest.fixture(scope="session")
def K():
    from elasticfusion_b200 import synth

    return synth.K_DEFAULT


@pytest.fixture(scope="session")
def frames(K):
    """8 noisy synthetic frames (rgb, depth, T_gt) of the S2 room sequence."""
    from elasticfusion_b200 import synth

    return list(synth.sequence(8, K, seed=42, noise=True))


@pytest.fixture(scope="session")
def small_K():
    from elasticfusion_b200 import synth

    return synth.Intrinsics(160, 120, 132.0, 132.0, 80.0, 60.0)


@pytest.fixture(scope="session")
def small_frames(small_K):
    from elasticfusion_b200 import synth

    return list(synth.sequence(6, small_K, seed=7, noise=True))
