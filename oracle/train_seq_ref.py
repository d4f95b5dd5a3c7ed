"""TEST INFRASTRUCTURE ONLY -- the reference graph over many sequences in one batch (the ``seq_lengths`` calls of the
training and inference kernels), differentiated by torch autograd at a chosen precision.

A batch ``x [B, C, W]`` holds N consecutive sequences ``seq_lengths = [n_0, ..., n_{N-1}]``; sequence s is rows
``o_s .. o_s + n_s - 1``.  The truth is one ``model(x[o:o+n], age[o:o+n])`` call of the reference module in train() mode
per sequence (bin/models.py:22-36: the LSTM scans that sequence from the zero state), concatenated, with the loss over all
B windows as in bin/utils.py:200-208.  Returns what :func:`oracle.train_ref.train_reference` returns, so
:func:`oracle.train_ref.assert_close_elem` compares it the same way.
"""
from __future__ import annotations

import copy

import torch
import torch.nn.functional as F

from .mycnn_c import BLOB_KEYS
from .mycnn_torch import RefMyCNN
from .train_ref import MaskDropout


def _cast(t, dtype):
    return None if t is None else torch.as_tensor(t).detach().to(dtype)


def train_reference_seq(ref: RefMyCNN, x, age, seq_lengths, mask1=None, mask2=None, target=None, pos_weight=None, dz=None,
                        dtype=torch.float64) -> dict:
    """``train_reference(ref, x, age, "sequence", ...)`` with the LSTM started afresh at every sequence of
    ``seq_lengths``: ``z = torch.cat([ref(x[o:o+n], age[o:o+n]) for o, n in ...])`` with the same dropout masks, then
    the heads ``"bce"``, ``"bce_pw"`` and ``"dz"`` of ``train_reference`` (means over all B windows).  ``age``: B values
    or one, broadcast."""
    lens = [int(n) for n in seq_lengths]
    m = copy.deepcopy(ref).to(dtype)
    m.dropout = MaskDropout()
    m.train()
    x = _cast(x, dtype).clone().requires_grad_()
    age = _cast(age, dtype).reshape(-1).clone().requires_grad_()
    mask1, mask2 = _cast(mask1, dtype), _cast(mask2, dtype)
    B = x.shape[0]
    if min(lens) < 1 or sum(lens) != B:
        raise ValueError(f"seq_lengths {lens} do not split a batch of {B}")
    outs, o = [], 0
    for n in lens:
        m.dropout.set(None if mask1 is None else mask1[o:o + n], None if mask2 is None else mask2[o:o + n])
        outs.append(m(x[o:o + n], age[o:o + n] if age.numel() > 1 else age).reshape(-1))
        o += n
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
