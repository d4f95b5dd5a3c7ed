"""TEST INFRASTRUCTURE ONLY -- one training step of ``RefMyCNN`` (oracle/mycnn_torch.py) differentiated by torch autograd
at a chosen precision.

In float64 it is the truth the training kernels (csrc/b2cnn_train.cu) are compared with element by element; the same
function in float32 is the yardstick for "as accurate as the reference" (:func:`assert_close_elem`).  Dropout
masks are explicit (torch's Philox stream cannot be shared with another implementation): the module's ``nn.Dropout`` is
swapped for :class:`MaskDropout`, so the module's own ``forward`` is what gets differentiated.

Batch modes: "sequence" is ``model(x, age)`` (the LSTM scans the batch axis); "independent" is one ``model(x[i:i+1],
age[i:i+1])`` call per window, every window from the zero state.
"""
from __future__ import annotations

import copy

import numpy as np
import torch
import torch.nn.functional as F
from torch import nn

from .mycnn_c import BLOB_KEYS
from .mycnn_torch import RefMyCNN


class MaskDropout(nn.Module):
    """``nn.Dropout`` with given masks (already scaled by 1/(1-p)), used in call order: conv1's pool, then conv2's."""

    def __init__(self):
        super().__init__()
        self.masks, self.i = [None, None], 0

    def set(self, m1, m2):
        self.masks, self.i = [m1, None if m2 is None else m2.unsqueeze(1)], 0

    def forward(self, x):
        m = self.masks[self.i]
        self.i += 1
        return x if m is None else x * m


def _cast(t, dtype):
    return None if t is None else torch.as_tensor(t).detach().to(dtype)


def train_reference(ref: RefMyCNN, x, age, mode: str = "sequence", mask1=None, mask2=None, target=None,
                    pos_weight=None, dz=None, dtype=torch.float64) -> dict:
    """Logits and, per loss head, the loss and the gradients of the 14 ``BLOB_KEYS``, of ``x`` and of ``age``.

    ``ref`` is left untouched (a copy is cast to ``dtype``).  ``age``: B values or one, broadcast over the batch like
    the reference; ``d age`` has the shape given.  Heads, each present when its inputs are:

    - ``"bce"``: ``BCEWithLogitsLoss()(z, target)``;
    - ``"bce_pw"``: ``BCEWithLogitsLoss(pos_weight=pos_weight)(z, target)``;
    - ``"dz"``: an arbitrary upstream gradient d loss / d z, i.e. ``loss = (z * dz).sum()``.

    Returns ``{"z": z, head: {"loss", "grads": {key: tensor}, "dx", "dage"}}``, all detached, in ``dtype``."""
    if mode not in ("sequence", "independent"):
        raise ValueError("mode must be 'sequence' or 'independent'")
    m = copy.deepcopy(ref).to(dtype)
    m.dropout = MaskDropout()
    m.train()
    x = _cast(x, dtype).clone().requires_grad_()
    age = _cast(age, dtype).reshape(-1).clone().requires_grad_()
    mask1, mask2 = _cast(mask1, dtype), _cast(mask2, dtype)
    B = x.shape[0]
    if mode == "sequence":
        m.dropout.set(mask1, mask2)
        z = m(x, age)
    else:
        outs = []
        for i in range(B):
            m.dropout.set(None if mask1 is None else mask1[i:i + 1], None if mask2 is None else mask2[i:i + 1])
            outs.append(m(x[i:i + 1], age[i:i + 1] if age.numel() > 1 else age))
        z = torch.cat(outs)
    heads = {}
    if target is not None:
        target = _cast(target, dtype)
        heads["bce"] = F.binary_cross_entropy_with_logits(z, target)
        if pos_weight is not None:
            heads["bce_pw"] = F.binary_cross_entropy_with_logits(z, target, pos_weight=torch.tensor(pos_weight, dtype=dtype))
    if dz is not None:
        heads["dz"] = (z * _cast(dz, dtype)).sum()
    named = dict(m.named_parameters())
    leaves = [named[k] for k in BLOB_KEYS] + [x, age]
    out = {"z": z.detach()}
    for name, loss in heads.items():
        g = torch.autograd.grad(loss, leaves, retain_graph=True)
        out[name] = {"loss": loss.detach(), "grads": dict(zip(BLOB_KEYS, g[:len(BLOB_KEYS)])), "dx": g[-2], "dage": g[-1]}
    return out


@torch.no_grad()
def pool_gaps(ref: RefMyCNN, x, mask1=None, dtype=torch.float64) -> tuple:
    """Per pooling window, the gap between the two largest pre-activations divided by max(1, |largest|):
    ``(gap1 [B, c_mid, P1], gap2 [B, L_out])`` for the pools after conv1 and conv2 (+inf where a window has one
    element).  A gap of 0 is an exact tie (routed to the first maximum); a gap near the rounding error of float32 is a
    near-tie, where a float32 implementation and the float64 truth may route the gradient to different positions."""
    m = copy.deepcopy(ref).to(dtype)
    a = m.arch
    x = _cast(x, dtype)

    def gaps(v):
        w = v.unfold(-1, a.pool_k, a.pool_s)
        if a.pool_k == 1:
            return torch.full(w.shape[:-1], float("inf"), dtype=dtype), w[..., 0]
        top = w.topk(2, dim=-1).values
        return (top[..., 0] - top[..., 1]) / top[..., 0].abs().clamp(min=1.0), top[..., 0]

    gap1, m1 = gaps(m.conv1(x))
    d1 = torch.tanh(m1) if mask1 is None else torch.tanh(m1) * _cast(mask1, dtype)
    gap2, _ = gaps(m.conv2(d1))
    return gap1, gap2.squeeze(1)


ALPHA, BETA, BETA_MAX = 8.0, 2.0 ** -20, 2e-5


def assert_close_elem(name, got, truth, ref32, alpha=ALPHA, beta=BETA):
    """Element by element: |got_i - truth_i| <= alpha * |ref32_i - truth_i| + beta * max|truth|.

    ``truth`` is a float64 computation, ``ref32`` the same computation in float32 (how far an honest float32
    implementation lands from the truth at that element); ``beta`` covers elements where the float32 reference happens
    to be exact.  Non-finite entries must match the truth exactly (same NaN pattern, same infinities)."""
    assert beta <= BETA_MAX, (name, beta)
    got = np.asarray(torch.as_tensor(got).detach().cpu().double(), dtype=np.float64)
    truth = np.asarray(torch.as_tensor(truth).detach().cpu().double(), dtype=np.float64)
    ref32 = np.asarray(torch.as_tensor(ref32).detach().cpu().double(), dtype=np.float64)
    assert got.shape == truth.shape == ref32.shape, (name, got.shape, truth.shape, ref32.shape)
    nan_g, nan_t = np.isnan(got), np.isnan(truth)
    if not np.array_equal(nan_g, nan_t):
        i = np.unravel_index(np.argmax(nan_g != nan_t), got.shape)
        raise AssertionError(f"{name}: NaN pattern differs ({int(nan_g.sum())} NaN vs {int(nan_t.sum())} in the truth); "
                             f"first at {i}: got {got[i]!r}, truth {truth[i]!r}, ref32 {ref32[i]!r}")
    inf_t = np.isinf(truth)
    bad_inf = (np.isinf(got) | inf_t) & ~nan_t & (got != truth)
    if bad_inf.any():
        i = np.unravel_index(np.argmax(bad_inf), got.shape)
        raise AssertionError(f"{name}: infinity differs at {i}: got {got[i]!r}, truth {truth[i]!r}")
    fin = np.isfinite(truth)
    if not fin.any():
        return
    scale = np.abs(truth[fin]).max()
    with np.errstate(invalid="ignore"):                                   # inf - inf where the infinities agree
        slack = np.nan_to_num(np.abs(ref32 - truth), nan=0.0, posinf=0.0)    # a non-finite yardstick gives no slack
        err = np.where(fin, np.abs(got - truth), 0.0)
    bound = alpha * slack + beta * scale
    bad = err > bound
    if bad.any():
        i = np.unravel_index(np.argmax(np.where(bad, err / np.maximum(bound, 1e-300), 0.0)), got.shape)
        need = float(((err - alpha * slack) / scale)[bad].max())
        raise AssertionError(f"{name}: {int(bad.sum())} of {got.size} elements off; worst at {i}: got {got[i]!r}, "
                             f"truth {truth[i]!r}, ref32 {ref32[i]!r} (bound {bound[i]:.3e}, max|truth| {scale:.3e}, "
                             f"beta would have to be {need:.2e})")


def smallest_beta(got, truth, ref32, alpha=ALPHA):
    """(the smallest beta :func:`assert_close_elem` would accept, the number of finite elements it judges); the beta is
    <= 0 where every element lies inside alpha |ref32 - truth|, and 0.0 when no element is finite"""
    got, truth, ref32 = (np.asarray(torch.as_tensor(t).detach().cpu().double()) for t in (got, truth, ref32))
    fin = np.isfinite(truth) & np.isfinite(got)
    if not fin.any():
        return 0.0, 0
    slack = np.nan_to_num(np.abs(ref32[fin] - truth[fin]), nan=0.0, posinf=0.0)
    return float(((np.abs(got[fin] - truth[fin]) - alpha * slack) / np.abs(truth[fin]).max()).max()), int(fin.sum())


def check_elems(pairs, label=""):
    """:func:`assert_close_elem` on every ``(name, got, truth, ref32, beta)``, all failures reported together.  Prints,
    per comparison, the smallest beta it would pass with and how many of its elements are finite (pytest -s shows it)."""
    errors = []
    for name, got, truth, ref32, beta in pairs:
        b, n = smallest_beta(got, truth, ref32)
        print(f"{label} {name}: smallest beta {b:.2e} (granted {beta:.2e}; {n} of {torch.as_tensor(truth).numel()} finite)")
        try:
            assert_close_elem(name, got, truth, ref32, beta=beta)
        except AssertionError as e:
            errors.append(str(e))
    assert not errors, "\n".join(errors)
