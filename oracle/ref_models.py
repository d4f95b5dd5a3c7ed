"""TEST INFRASTRUCTURE ONLY -- access to the UNMODIFIED reference class ``bin/models.py:MyCNN``.

``__graft_entry__.build()`` copies ``/root/reference/bin/models.py`` (35 lines, torch only) into the
git-ignored ``oracle/_ref/models.py`` whenever the reference tree is present (the authoring container);
``oracle/_ref/`` travels with the built tree to the GPU machine the way a
built ``.so`` does, and is never committed.  ``bench.py --impl reference`` and the ``cpu_baseline`` leg
time THIS class (``cpu_baseline.kind = "reference"``); when the copy is absent they fall back to the
restatement in ``oracle/mycnn_torch.py`` (``kind = "port"``).

``stretched()`` re-instantiates the reference class for a synthetic shape exactly the way
``tests/golden/make_golden.py`` does for the committed fixtures (SURVEY.md appendix 5): the class and
its ``forward`` are the reference's own code, only ``conv1`` / ``lstm`` / ``MAGICNUM`` are replaced.
"""
from __future__ import annotations

import importlib.util
import os

import torch
import torch.nn as nn

_HERE = os.path.dirname(os.path.abspath(__file__))
REF_COPY = os.path.join(_HERE, "_ref", "models.py")
REF_SOURCE = "/root/reference/bin/models.py"


def install_copy() -> bool:
    """Called by build(): refresh oracle/_ref/models.py from the reference tree when it exists."""
    if not os.path.exists(REF_SOURCE):
        return os.path.exists(REF_COPY)
    os.makedirs(os.path.dirname(REF_COPY), exist_ok=True)
    with open(REF_SOURCE, "rb") as f:
        data = f.read()
    if not os.path.exists(REF_COPY) or open(REF_COPY, "rb").read() != data:
        with open(REF_COPY, "wb") as f:
            f.write(data)
    return True


def reference_class():
    """The reference's ``MyCNN`` class object, or None when the copy is not available."""
    if not os.path.exists(REF_COPY):
        return None
    spec = importlib.util.spec_from_file_location("b2cnn_reference_models", REF_COPY)
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod.MyCNN


def stretched(MyCNN, kind: str, C: int, W: int, seed: int = 0):
    """make_golden.py's ``stretched``: MyCNN5 geometry (k1=10, pool(3,2)) or the older one (k1=5, pool(2,2))."""
    torch.manual_seed(seed)
    g = MyCNN()
    if kind == "mycnn5":
        k1, pk, ps = 10, 3, 2
    else:
        k1, pk, ps = 5, 2, 2
        g.pool = nn.MaxPool1d(kernel_size=pk, stride=ps)
    l1 = W - k1 + 1
    p1 = (l1 - pk) // ps + 1
    l2 = p1 - 5 + 1
    L = (l2 - pk) // ps + 1
    g.MAGICNUM = L
    g.conv1 = nn.Conv1d(C, 4, k1)
    g.lstm = nn.LSTM(L, 16, 2)
    g.eval()
    return g
