import os
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (run on an H100 with -m gpu)")


@pytest.fixture(scope="session")
def golden():
    # one fixture set stored in two files (each under 1 MB)
    out = {}
    for name in ("reference_cpu.npz", "reference_cpu_resize.npz"):
        with np.load(os.path.join(ROOT, "tests", "golden", name)) as z:
            out.update({k: z[k] for k in z.files})
    return out


@pytest.fixture(scope="session")
def golden_extra():
    return np.load(os.path.join(ROOT, "tests", "golden", "reference_cpu_extra.npz"))


@pytest.fixture(scope="session")
def oracle():
    import oracle as O   # test infrastructure only

    O.build()
    return O


@pytest.fixture(scope="session")
def vb():
    """vision_b200 with the CUDA extension loaded; GPU tests fail (not skip) if it is missing."""
    import torch

    assert torch.cuda.is_available(), "GPU test collected without a CUDA device"
    import vision_b200

    vision_b200._lib.load_ops()
    return vision_b200
