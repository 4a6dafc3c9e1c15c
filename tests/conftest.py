import os
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)
GOLDEN = os.path.join(ROOT, "tests", "golden")


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs an H100 (sm_90a) GPU")


def load_golden(name):
    # a fixture too large for one file is stored as parts <name>.<part>.npz and merged here
    path = os.path.join(GOLDEN, name + ".npz")
    parts = [path] if os.path.exists(path) else sorted(
        os.path.join(GOLDEN, f) for f in os.listdir(GOLDEN) if f.startswith(name + ".") and f.endswith(".npz"))
    assert parts, name
    out = {}
    for p in parts:
        with np.load(p) as z:
            out.update({k: z[k] for k in z.files})
    return out


def golden_params(fx, dtype=None):
    out = {}
    for k, v in fx.items():
        if k.startswith("p:"):
            out[k[2:]] = v.astype(dtype) if dtype is not None else v
    return out


@pytest.fixture(scope="session")
def golden():
    return load_golden
