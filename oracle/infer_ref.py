"""TEST INFRASTRUCTURE ONLY -- the inference forward of ``RefMyCNN`` (oracle/mycnn_torch.py) at a chosen precision.

In float64 it is the truth the inference kernels are compared with element by element
(oracle/train_ref.py::assert_close_elem); in float32 it is, operation for operation, the existing oracle
(:func:`oracle.mycnn_torch.ref_independent` / :func:`oracle.mycnn_torch.ref_sequence`), the yardstick for "as accurate
as the reference".

Batch modes: "independent" starts every window from the zero LSTM state (``predict()``, the reference's per-row loop);
"sequence" is ``model(x, age)``, where the LSTM scans the batch axis.

Beyond the reference's own layer stack (tanh, no affine) it takes the other activations and the folded eval-BatchNorm
the C ABI accepts (``b2cnn_config.act``, ``B2CNN_FLAG_AFFINE``), applied literally in the order the model defines:
``conv -> +bias -> * scale + shift -> act -> MaxPool`` for each conv.
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

ACTS = {"tanh": torch.tanh, "relu": torch.relu, "identity": lambda v: v}


def random_affine(seed: int, c_mid: int = 4) -> tuple:
    """A folded eval-BatchNorm ``(scale1[c_mid], shift1[c_mid], scale2[1], shift2[1])`` in float32 whose scales
    alternate in sign (scale2 < 0): a max pool taken before a negative scale picks the minimum, so only a kernel that
    applies the affine before pooling matches the reference."""
    g = torch.Generator().manual_seed(seed)
    s1 = (0.5 + torch.rand(c_mid, generator=g)) * torch.tensor([1.0, -1.0] * (c_mid // 2) + [1.0] * (c_mid % 2))
    t1 = 0.3 * torch.randn(c_mid, generator=g)
    s2 = -(0.5 + torch.rand(1, generator=g))
    t2 = 0.3 * torch.randn(1, generator=g)
    return s1, t1, s2, t2


@torch.no_grad()
def centre_affine(ref: RefMyCNN, x, act: str, affine) -> tuple:
    """``affine`` with its shifts replaced so that the median pre-activation of each channel over the finite values of
    ``x`` is 0, as a BatchNorm's running mean would: features under relu are then neither all 0 nor all positive"""
    m = copy.deepcopy(ref).double().eval()
    x = torch.as_tensor(x).detach().cpu().double()
    s1, _, s2, _ = (torch.as_tensor(a).double() for a in affine)

    def median(v):                                            # per channel, over windows and positions
        v = v.transpose(0, 1).reshape(v.shape[1], -1)
        return torch.stack([r[torch.isfinite(r)].median() for r in v])

    v1 = m.conv1(x) * s1.view(1, -1, 1)
    t1 = -median(v1)
    v2 = m.conv2(m.pool(ACTS[act](v1 + t1.view(1, -1, 1)))) * s2
    t2 = -median(v2)
    return affine[0], t1.float(), affine[2], t2.float()


def _features(m: RefMyCNN, x, act: str, affine):
    """conv1 -> (* scale1 + shift1) -> act -> pool -> conv2 -> (* scale2 + shift2) -> act -> pool -> view(-1, L);
    with tanh and no affine these are the very operations of ``RefMyCNN.features`` (dropout is the identity in eval)"""
    f = ACTS[act]
    v = m.conv1(x)
    if affine is not None:
        v = v * affine[0].view(1, -1, 1) + affine[1].view(1, -1, 1)
    v = m.pool(f(v))
    v = m.conv2(v)
    if affine is not None:
        v = v * affine[2] + affine[3]
    return m.pool(f(v)).view(-1, m.MAGICNUM)


@torch.no_grad()
def infer_reference(ref: RefMyCNN, x, age, mode: str = "independent", dtype=torch.float64, act: str = "tanh",
                    affine=None) -> dict:
    """``{"features": [B, L_out], "z": [B]}`` in ``dtype``; ``ref`` is left untouched (a copy is cast to ``dtype``).

    ``x``: [B, C, W] of any float dtype (bf16 and float32 windows upcast exactly); ``age``: B values or one, broadcast
    over the batch like the reference.  ``act``: "tanh" (the reference), "relu" or "identity"; ``affine``: None or
    ``(scale1[4], shift1[4], scale2, shift2)``, the folded eval-BatchNorm after conv1 and conv2."""
    if mode not in ("sequence", "independent"):
        raise ValueError("mode must be 'sequence' or 'independent'")
    if act not in ACTS:
        raise ValueError("act must be 'tanh', 'relu' or 'identity'")
    m = copy.deepcopy(ref).to(dtype).eval()
    x = torch.as_tensor(x).detach().cpu().to(dtype)
    age = torch.as_tensor(age).detach().cpu().to(dtype).reshape(-1)
    if affine is not None:
        affine = tuple(torch.as_tensor(a).detach().cpu().to(dtype).reshape(-1) for a in affine)
        assert [a.numel() for a in affine] == [m.arch.c_mid, m.arch.c_mid, 1, 1], "affine: (scale1[4], shift1[4], scale2, shift2)"
    f = _features(m, x, act, affine)
    if mode == "sequence":
        h, _ = m.lstm(f)                      # 2-D input: the LSTM scans the batch axis (RefMyCNN.forward)
        y = m.out(h)
    else:
        h, _ = m.lstm(f.unsqueeze(0))
        y = m.out(h.squeeze(0))
    z = (y * torch.relu(age.unsqueeze(1) * m.arch.age_coef + 1)).squeeze(1)
    return {"features": f, "z": z}
