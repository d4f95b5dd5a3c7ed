"""TEST INFRASTRUCTURE ONLY -- the sequence-mode LSTM head of ``RefMyCNN`` started from a given state, at a chosen
precision: the truth ``predict_record(mode="sequence", state=...)`` and a warm-started ``SlidingScorer`` are compared
with element by element.

One state format: a tensor ``[B, 2, 2, 16]`` indexed [recording][layer][h | c][unit], ``SlidingScorer.export()["lstm"]``'s
layout.  As ``nn.LSTM``'s ``(h, c)`` tuple: ``h = state[:, :, 0].transpose(0, 1)``, ``c = state[:, :, 1].transpose(0, 1)``,
each ``[layers, B, hidden]`` (:func:`to_lstm_tuple`, :func:`from_lstm_tuple`).  The scan itself is ``nn.LSTM`` called with
that tuple on the window features, so without ``torch.no_grad`` autograd gives the gradient of the initial state too;
:func:`train_record_state_reference` is the training graph of the ``_record`` calls with a state in and out.
"""
from __future__ import annotations

import copy

import torch
import torch.nn.functional as F

from .infer_ref import _features
from .mycnn_c import BLOB_KEYS
from .mycnn_torch import RefMyCNN
from .train_record_ref import cut
from .train_ref import MaskDropout


def to_lstm_tuple(state: torch.Tensor):
    """[B, 2, 2, 16] -> (h, c), each [2, B, 16]"""
    return state[:, :, 0].transpose(0, 1), state[:, :, 1].transpose(0, 1)


def from_lstm_tuple(h: torch.Tensor, c: torch.Tensor) -> torch.Tensor:
    """(h, c), each [2, B, 16] -> [B, 2, 2, 16]"""
    return torch.stack([h.transpose(0, 1), c.transpose(0, 1)], dim=2)


def sequence_with_state(ref: RefMyCNN, windows, age, state=None, dtype=torch.float64, act: str = "tanh", affine=None) -> dict:
    """One recording's windows ``[n, C, W]`` scanned as one LSTM sequence from ``state`` ``[2, 2, 16]`` (None: zeros),
    as ``model(windows, age)`` with ``(h0, c0)``; ``{"z": [n], "state": [2, 2, 16]}`` in ``dtype``, ``state`` the one
    after the last window (``state`` itself for n = 0).  ``age``: one value.  ``ref`` is left untouched."""
    m = copy.deepcopy(ref).to(dtype).eval()
    x = torch.as_tensor(windows).detach().cpu().to(dtype)
    a = torch.as_tensor(age).detach().cpu().to(dtype).reshape(-1)[:1]
    H = m.lstm.hidden_size
    s = torch.zeros(1, 2, 2, H, dtype=dtype) if state is None else torch.as_tensor(state).cpu().to(dtype).reshape(1, 2, 2, H)
    if affine is not None:
        affine = tuple(torch.as_tensor(t).detach().cpu().to(dtype).reshape(-1) for t in affine)
    if x.shape[0] == 0:
        return {"z": torch.zeros(0, dtype=dtype), "state": s[0]}
    h0, c0 = to_lstm_tuple(s)
    f = _features(m, x, act, affine)                                   # [n, L]
    h, (hn, cn) = m.lstm(f.unsqueeze(1), (h0, c0))                     # batch of one sequence, time along the windows
    z = (m.out(h[:, 0]) * torch.relu(a * m.arch.age_coef + 1)).squeeze(1)
    return {"z": z, "state": from_lstm_tuple(hn, cn)[0]}


def train_record_state_reference(ref: RefMyCNN, records, stride, age, counts, state=None, mask1=None, mask2=None, dz=None, dstate=None,
                                 target=None, pos_weight=None, dtype=torch.float64) -> dict:
    """The sequence-mode ``_record`` training graph with an initial state, in train() mode with the given dropout masks
    (:func:`oracle.train_record_ref.cut`): recording b's counted windows scanned by ``nn.LSTM`` from ``state[b]``
    ``[2, 2, 16]`` (None: zeros), a recording without windows passing its state through.  The loss is ``(z * dz).sum() +
    (state_out * dstate).sum()`` plus, with ``target``, ``BCEWithLogitsLoss(pos_weight=pos_weight)(z, target)`` (the
    mean over the M windows; a None term left out), differentiated by autograd.  Returns, detached and in
    ``dtype``: ``z`` [M], ``state`` (the final states) [B, 2, 2, 16], ``grads`` {key: tensor}, ``drecords`` [B, C, N],
    ``dage`` (one per recording) and ``dstate`` (the gradient of the initial state)."""
    arch = ref.arch
    counts = [int(c) for c in counts]
    m = copy.deepcopy(ref).to(dtype)
    m.dropout = MaskDropout()
    m.train()
    rec = torch.as_tensor(records).detach().to(dtype).requires_grad_()
    B, H = rec.shape[0], m.lstm.hidden_size
    age_r = torch.as_tensor(age).detach().to(dtype).reshape(-1).expand(B).clone().requires_grad_()
    s0 = torch.zeros(B, 2, 2, H, dtype=dtype) if state is None else torch.as_tensor(state).detach().cpu().to(dtype)
    s0 = s0.clone().requires_grad_()
    cast = (lambda t: None if t is None else torch.as_tensor(t).detach().cpu().to(dtype))
    x, m1, m2 = cut(rec, arch.window, stride, counts, arch.pool_s, cast(mask1), cast(mask2))
    zs, outs, o = [], [], 0
    for b, n in enumerate(counts):
        if n == 0:
            outs.append(s0[b])
            continue
        m.dropout.set(None if m1 is None else m1[o:o + n], None if m2 is None else m2[o:o + n])
        f = m.features(x[o:o + n])
        h, (hn, cn) = m.lstm(f.unsqueeze(1), to_lstm_tuple(s0[b:b + 1]))
        zs.append((m.out(h[:, 0]) * torch.relu(age_r[b] * arch.age_coef + 1)).squeeze(1))
        outs.append(from_lstm_tuple(hn, cn)[0])
        o += n
    z, s_out = torch.cat(zs), torch.stack(outs)
    loss = 0.0
    if dz is not None:
        loss = loss + (z * cast(dz)).sum()
    if dstate is not None:
        loss = loss + (s_out * cast(dstate)).sum()
    if target is not None:
        pw = None if pos_weight is None else torch.tensor(pos_weight, dtype=dtype)
        loss = loss + F.binary_cross_entropy_with_logits(z, cast(target), pos_weight=pw)
    named = dict(m.named_parameters())
    leaves = [named[k] for k in BLOB_KEYS] + [rec, age_r, s0]
    g = torch.autograd.grad(loss, leaves, allow_unused=True)
    g = [torch.zeros_like(t) if d is None else d for t, d in zip(leaves, g)]
    return {"z": z.detach(), "state": s_out.detach(), "loss": torch.as_tensor(loss).detach(), "grads": dict(zip(BLOB_KEYS, g[:len(BLOB_KEYS)])), "drecords": g[-3],
            "dage": g[-2], "dstate": g[-1]}
