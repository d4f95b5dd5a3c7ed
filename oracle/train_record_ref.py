"""TEST INFRASTRUCTURE ONLY -- the reference graph over the sliding windows of whole recordings (the ``_record`` training
calls), differentiated by torch autograd at a chosen precision.

Recordings ``[B, C, N]``; window w of recording b is samples ``[w S, w S + W)`` for w < ``counts[b]``.  The truth cuts
those windows out of a float64 recording that requires grad (``unfold``), cuts the recording's dropout masks the same
way (window w: ``mask1[b, :, wS/pool_s : wS/pool_s + P1]`` and ``mask2[b, wS/pool_s^2 : wS/pool_s^2 + L]``), runs
:func:`oracle.train_seq_ref.train_reference_seq` on them -- one sequence per recording with windows in sequence mode, one
per window in independent mode -- and carries the windows' input gradient back onto the recording by autograd.
"""
from __future__ import annotations

import torch

from .train_seq_ref import train_reference_seq


def cut(records, W, S, counts, pool_s, mask1=None, mask2=None):
    """``(windows [M, C, W], mask1 [M, 4, P1] or None, mask2 [M, L] or None)`` of the counted windows, recording-major.
    Differentiable in ``records``."""
    sel = [(b, w) for b, n in enumerate(counts) for w in range(int(n))]
    x = torch.stack([records[b, :, w * S:w * S + W] for b, w in sel])
    m1 = m2 = None
    N = records.shape[2]
    if mask1 is not None:
        P1 = mask1.shape[2] - (N - W) // pool_s
        m1 = torch.stack([mask1[b, :, w * S // pool_s:w * S // pool_s + P1] for b, w in sel])
    if mask2 is not None:
        L = mask2.shape[1] - (N - W) // pool_s ** 2
        m2 = torch.stack([mask2[b, w * S // pool_s ** 2:w * S // pool_s ** 2 + L] for b, w in sel])
    return x, m1, m2


def train_reference_record(ref, records, stride, age, counts, mode="sequence", mask1=None, mask2=None, target=None,
                           pos_weight=None, dz=None, dtype=torch.float64) -> dict:
    """What :func:`oracle.train_seq_ref.train_reference_seq` returns for the cut windows, with per head ``"drecords"``
    (d loss / d records [B, C, N]) and ``"dage_rec"`` (d loss / d age of each recording: the sum over its windows); its
    ``"dx"`` / ``"dage"`` stay per window.  ``age``: a scalar or one per recording."""
    arch = ref.arch
    counts = [int(c) for c in counts]
    rec = torch.as_tensor(records).detach().to(dtype).requires_grad_()
    x, m1, m2 = cut(rec, arch.window, stride, counts, arch.pool_s, mask1, mask2)
    B = rec.shape[0]
    age_r = torch.as_tensor(age, dtype=torch.float64).reshape(-1).expand(B)
    age_w = age_r.repeat_interleave(torch.tensor(counts))
    lens = [c for c in counts if c > 0] if mode == "sequence" else [1] * x.shape[0]
    out = train_reference_seq(ref, x.detach(), age_w, lens, m1, m2, target=target, pos_weight=pos_weight, dz=dz, dtype=dtype)
    owner = torch.arange(B).repeat_interleave(torch.tensor(counts))
    for name in ("bce", "bce_pw", "dz"):
        if name in out:
            h = out[name]
            h["drecords"] = torch.autograd.grad(x, rec, h["dx"].to(dtype), retain_graph=True)[0]
            h["dage_rec"] = torch.zeros(B, dtype=h["dage"].dtype).index_add_(0, owner, h["dage"].reshape(-1))
    out["windows"], out["mask1"], out["mask2"] = x.detach(), m1, m2
    return out
