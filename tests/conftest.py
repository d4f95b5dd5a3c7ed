import os
import sys

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)
GOLDEN = os.path.join(ROOT, "tests", "golden")


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (an H100)")


def pytest_collection_modifyitems(config, items):
    if torch.cuda.is_available():
        return
    skip = pytest.mark.skip(reason="no CUDA device")
    for item in items:
        if "gpu" in item.keywords:
            item.add_marker(skip)


def load_golden(name):
    g = np.load(os.path.join(GOLDEN, name))
    sd = {k[3:]: torch.from_numpy(g[k]) for k in g.files if k.startswith("sd.")}
    return g, sd


def rel_err(got, want):
    got = np.asarray(got, dtype=np.float64)
    want = np.asarray(want, dtype=np.float64)
    return float(np.abs(got - want).max() / max(np.abs(want).max(), 1e-6))


def rel_err_elem(got, want, floor_frac=1e-2):
    """PER-ELEMENT relative error: max_i |got_i - want_i| / max(|want_i|, floor_frac * max|want|).  The floor only
    keeps logits that happen to sit next to zero from dividing by ~0 (they are judged against 1 % of the batch scale)."""
    got = np.asarray(got, dtype=np.float64)
    want = np.asarray(want, dtype=np.float64)
    den = np.maximum(np.abs(want), floor_frac * max(np.abs(want).max(), 1e-30))
    return float((np.abs(got - want) / den).max())


@pytest.fixture(scope="session")
def golden5():
    return load_golden("mycnn5_xtestinput.npz")
