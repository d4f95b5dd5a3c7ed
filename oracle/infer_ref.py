"""TEST INFRASTRUCTURE ONLY -- the inference forward of ``RefMyCNN`` (oracle/mycnn_torch.py) at a chosen precision.

In float64 it is the truth the inference kernels are compared with element by element
(oracle/train_ref.py::assert_close_elem); in float32 it is, operation for operation, the existing oracle
(:func:`oracle.mycnn_torch.ref_independent` / :func:`oracle.mycnn_torch.ref_sequence`), the yardstick for "as accurate
as the reference".

Batch modes: "independent" starts every window from the zero LSTM state (``predict()``, the reference's per-row loop);
"sequence" is ``model(x, age)``, where the LSTM scans the batch axis.
"""
from __future__ import annotations

import copy

import torch

from .mycnn_torch import RefMyCNN

# Floor of the per-element bound granted to the tensor-core features (tests/test_gpu_infer_elem.py).  Measured worst on
# an H100: 2.3e-6 on saturated physio windows (the exact generic kernel: 1.2e-6 there) and 1.5e-6 on windows scaled
# by 1e-3, where the epilogue's tanh, 1 - 2 / (1 + 2^(2x log2 e)) on ex2.approx / rcp.approx, has an absolute error of
# ~1e-7 against features of ~0.1 (the generic kernel's tanhf passes there at 2^-20).  Conv1 weights missing their
# third bf16 piece (tc_splits=2) need 4e-6 on normal windows and 2e-4 on physio ones: the CPU negative control in
# tests/test_oracle_infer.py and the GPU one in tests/test_gpu_infer_elem.py show this bound rejects them.
TC_FEATURES_BETA = 3e-6


@torch.no_grad()
def infer_reference(ref: RefMyCNN, x, age, mode: str = "independent", dtype=torch.float64) -> dict:
    """``{"features": [B, L_out], "z": [B]}`` in ``dtype``; ``ref`` is left untouched (a copy is cast to ``dtype``).

    ``x``: [B, C, W] of any float dtype (bf16 and float32 windows upcast exactly); ``age``: B values or one, broadcast
    over the batch like the reference."""
    if mode not in ("sequence", "independent"):
        raise ValueError("mode must be 'sequence' or 'independent'")
    m = copy.deepcopy(ref).to(dtype).eval()
    x = torch.as_tensor(x).detach().cpu().to(dtype)
    age = torch.as_tensor(age).detach().cpu().to(dtype).reshape(-1)
    f = m.features(x)
    if mode == "sequence":
        z = m(x, age)
    else:
        h, _ = m.lstm(f.unsqueeze(0))
        y = m.out(h.squeeze(0))
        z = (y * torch.relu(age.unsqueeze(1) * m.arch.age_coef + 1)).squeeze(1)
    return {"features": f, "z": z}
