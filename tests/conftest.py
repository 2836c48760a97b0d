import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for sub in ("gpu-dpf_b200", "oracle", "tests"):
    p = os.path.join(ROOT, sub)
    if p not in sys.path:
        sys.path.insert(0, p)


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (select with `-m gpu`)")


@pytest.fixture(scope="session")
def oracle():
    import oracle as O
    return O.Oracle()


@pytest.fixture(scope="session")
def ref():
    import oracle as O
    if not O.Ref.available():
        pytest.skip("oracle/_ref/libdpfref.so not built (reference tree absent)")
    return O.Ref()


@pytest.fixture(scope="session")
def golden():
    import numpy as np
    return np.load(os.path.join(ROOT, "tests", "golden", "golden_v1.npz"))
