import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)
GOLDEN = os.path.join(ROOT, "tests", "golden")


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (select with -m gpu)")


@pytest.fixture(scope="session")
def golden_dir():
    return GOLDEN


@pytest.fixture(scope="session")
def synthetic_weights():
    from demon_b200 import weights as W
    return W.synthetic_weights(0)


@pytest.fixture(scope="session")
def sculpture(golden_dir):
    """The reference's example pair, prepared like examples/example.py:15-42 (channels_first)."""
    import numpy as np
    z = np.load(os.path.join(golden_dir, "sculpture_inputs.npz"))

    def prep(a):
        return (a.astype(np.float32) / 255 - 0.5).transpose(2, 0, 1)
    return {
        "image_pair": np.concatenate((prep(z["img1"]), prep(z["img2"])), axis=0)[None],
        "image1": prep(z["img1"])[None],
        "image2_2": prep(z["img2_2"])[None],
        "depth1_l2": z["depth1_l2"], "Rt1": z["Rt1"], "Rt2": z["Rt2"],
    }
