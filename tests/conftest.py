import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

GOLDEN = os.path.join(ROOT, "tests", "golden")


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (run on an H100 with `-m gpu`)")


@pytest.fixture(scope="session")
def golden():
    import numpy as np

    class G:
        def __init__(self):
            self._c = {}

        def __call__(self, name):
            # a fixture may be stored in several files (name.npz, name.part2.npz, ...) to keep every file small
            if name not in self._c:
                d = {}
                for f in sorted(os.listdir(GOLDEN)):
                    if f == name + ".npz" or (f.startswith(name + ".part") and f.endswith(".npz")):
                        d.update(np.load(os.path.join(GOLDEN, f)))
                self._c[name] = d
            return self._c[name]
    return G()


@pytest.fixture(scope="session")
def cuda():
    import torch
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    return torch.device("cuda:0")
