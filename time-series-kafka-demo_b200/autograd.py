"""The device model under torch autograd: any loss, any optimizer, gradients for the input too.

The reference trains with ``utils.train`` (bin/utils.py:183-227)::

    model.train()
    for input, age, target in loader:
        optimizer.zero_grad(); output = model(input, age); loss = criterion(output, target)
        loss.backward(); optimizer.step()

with ``criterion = nn.BCEWithLogitsLoss(pos_weight=pos_weight)`` and ``optim.Adam(lr=1e-5)``
(bin/explore_torch.ipynb:3170,3204-3205).  :class:`B200TrainableMyCNN` is a :class:`B200MyCNN` whose parameters
take part in that loop unchanged: in ``train()`` mode its forward is ``b2cnn_train_forward`` (the training kernels of
csrc/b2cnn_train.cu, keeping the activations the backward pass needs) and autograd's backward is
``b2cnn_train_backward_ex`` (BPTT over the batch axis, pooling / conv backward, and the input gradient) driven by whatever
upstream gradient the loss produces.  With ``conv1`` / ``conv2`` frozen (``requires_grad_(False)``) and an input that
needs no gradient, the convolutional backward is skipped altogether.  In ``eval()`` mode it is the inference path of
:class:`B200MyCNN`; optimizer steps edit the parameters in place, so the next inference call re-uploads them.

:func:`mycnn_train_forward` is the same computation as a function of explicit parameters and dropout masks.
"""
from __future__ import annotations

import ctypes
from typing import Optional, Sequence

import torch
import torch.nn as nn
from torch.autograd.function import once_differentiable

from . import capi
from .arch import BLOB_KEYS, ArchConfig
from .model import B200MyCNN

_MODES = {"sequence": capi.MODE_SEQUENCE, "independent": capi.MODE_INDEPENDENT}


def _ptr(t: Optional[torch.Tensor]):
    return ctypes.c_void_p(t.data_ptr()) if t is not None else None


def check_trainable(arch: ArchConfig) -> None:
    """The training kernels cover the reference's tanh layer stack without the affine variant."""
    if arch.affine or arch.act_id != 0:
        raise NotImplementedError("training covers the reference's tanh stack (bin/models.py:23,26) without the affine variant")


def draw_masks(arch: ArchConfig, B: int, p: float, device, generator: Optional[torch.Generator] = None):
    """The two nn.Dropout masks of bin/models.py:25,28 for B windows, scaled by 1/(1-p) like torch's dropout; (None, None)
    for p = 0.  Drawn from ``generator``, or from torch's default generator of the device when None."""
    if not 0.0 <= p < 1.0:
        raise ValueError("dropout p must be in [0, 1)")
    if p == 0.0:
        return None, None
    keep = 1.0 - p
    m1 = torch.bernoulli(torch.full((B, arch.c_mid, arch.p1), keep, device=device), generator=generator).div_(keep)
    m2 = torch.bernoulli(torch.full((B, arch.l_out), keep, device=device), generator=generator).div_(keep)
    return m1, m2


def check_masks(arch: ArchConfig, B: int, device, mask1: Optional[torch.Tensor], mask2: Optional[torch.Tensor]):
    """The two dropout masks as contiguous fp32 tensors on ``device``: each None or of shape [B, c_mid, P1] / [B, L_out]."""
    out = []
    for i, (m, shape) in enumerate(((mask1, (B, arch.c_mid, arch.p1)), (mask2, (B, arch.l_out))), 1):
        if m is not None:
            m = m.detach().to(device, torch.float32).contiguous()
            if tuple(m.shape) != shape:
                raise RuntimeError(f"dropout mask {i} must be {shape}, got {tuple(m.shape)}")
        out.append(m)
    return out


class _TrainForward(torch.autograd.Function):
    """Inputs: a :class:`_Call` (non-tensor), x [B,C,W] fp32, age [B] fp32, then the 14 ``BLOB_KEYS`` tensors."""

    @staticmethod
    def forward(ctx, call, x, age, *params):
        dev = x.device
        blob = torch.cat([p.detach().reshape(-1) for p in params])               # the packed blob (include/b2cnn.h)
        B = x.shape[0]
        ws = torch.empty(call.workspace_bytes(B), dtype=torch.uint8, device=dev)
        z = torch.empty(B, dtype=torch.float32, device=dev)
        st = torch.cuda.current_stream(dev).cuda_stream
        rc = call.lib.b2cnn_train_forward(ctypes.byref(call.cfg), _ptr(blob), _ptr(x), B, _ptr(age), call.mode,
                                          _ptr(call.mask1), _ptr(call.mask2), _ptr(z), _ptr(ws), ws.numel(), ctypes.c_void_p(st))
        capi.check(rc, "b2cnn_train_forward")
        ctx.call, ctx.blob, ctx.ws = call, blob, ws
        ctx.shapes = [p.shape for p in params]
        ctx.save_for_backward(x, age)
        return z

    @staticmethod
    @once_differentiable
    def backward(ctx, dz):
        call, blob, ws = ctx.call, ctx.blob, ctx.ws
        x, age = ctx.saved_tensors
        B = x.shape[0]
        dz = dz.to(torch.float32).contiguous()
        grads = torch.empty_like(blob)
        dx = torch.empty_like(x) if ctx.needs_input_grad[1] else None
        dage = torch.empty_like(age) if ctx.needs_input_grad[2] else None
        # conv1 / conv2 frozen and no input gradient wanted (fine-tuning the head): the library skips the conv backward
        frozen = dx is None and not any(ctx.needs_input_grad[3:7])
        st = torch.cuda.current_stream(x.device).cuda_stream
        rc = call.lib.b2cnn_train_backward_ex(ctypes.byref(call.cfg), _ptr(blob), _ptr(x), B, _ptr(age), call.mode, _ptr(call.mask1),
                                              _ptr(call.mask2), _ptr(dz), _ptr(grads), _ptr(dx), _ptr(dage),
                                              capi.TRAIN_FROZEN_CONV if frozen else 0, _ptr(ws), ws.numel(), ctypes.c_void_p(st))
        capi.check(rc, "b2cnn_train_backward")
        out, at = [], 0
        for shape, need in zip(ctx.shapes, ctx.needs_input_grad[3:]):
            n = shape.numel()
            out.append(grads[at:at + n].view(shape) if need else None)
            at += n
        return (None, dx, dage, *out)


class _Call:
    """What one forward / backward pair shares besides tensors: the library, its configuration, mode and masks."""

    def __init__(self, arch: ArchConfig, device: torch.device, mode: int, mask1, mask2):
        self.lib = capi.load_library()
        self.cfg = capi.make_config(arch, device.index if device.index is not None else torch.cuda.current_device())
        self.mode, self.mask1, self.mask2 = mode, mask1, mask2

    def workspace_bytes(self, B: int) -> int:
        need = int(self.lib.b2cnn_train_workspace_bytes(ctypes.byref(self.cfg), B))
        if need < 0:
            capi.check(capi.EINVAL, "b2cnn_train_workspace_bytes")
        return need


def mycnn_train_forward(x: torch.Tensor, age: torch.Tensor, params: Sequence[torch.Tensor], arch: ArchConfig,
                        mode: str = "sequence", mask1: Optional[torch.Tensor] = None,
                        mask2: Optional[torch.Tensor] = None) -> torch.Tensor:
    """Logits [B] of the model in train() mode (bin/models.py:22-36), differentiable in ``x``, ``age`` and ``params``.

    ``params``: the 14 tensors of ``BLOB_KEYS`` in that order, on one CUDA device.  ``x`` [B,C,W] (fp32 or bf16; cast
    to fp32), ``age`` 1 or B values.  ``mode``: "sequence" (the LSTM scans the batch axis, as ``model(x, age)`` does in
    the reference) or "independent" (every window from the zero state).  ``mask1`` [B, c_mid, P1] / ``mask2``
    [B, L_out]: the two dropout masks, already scaled by 1/(1-p); None = no dropout."""
    check_trainable(arch)
    if mode not in _MODES:
        raise ValueError("mode must be 'sequence' or 'independent'")
    if len(params) != len(BLOB_KEYS):
        raise ValueError(f"expected the {len(BLOB_KEYS)} tensors of BLOB_KEYS, got {len(params)}")
    shapes = arch.param_shapes()
    for k, p in zip(BLOB_KEYS, params):
        if tuple(p.shape) != shapes[k]:
            raise RuntimeError(f"{k}: expected shape {shapes[k]}, got {tuple(p.shape)}")
    dev = params[0].device
    if dev.type != "cuda" or any(p.device != dev for p in params):
        raise RuntimeError("training on the device needs every parameter on one CUDA device (there is no CPU fallback)")
    if any(p.dtype != torch.float32 for p in params):
        raise RuntimeError("training on the device needs float32 parameters")
    if x.dim() != 3 or x.shape[1] != arch.in_channels or x.shape[2] != arch.window:
        raise RuntimeError(f"expected x of shape [B, {arch.in_channels}, {arch.window}], got {tuple(x.shape)}")
    B = x.shape[0]
    if B < 1:
        raise RuntimeError("expected at least one window")
    x = x.to(dev, torch.float32).contiguous()
    age = torch.as_tensor(age).to(dev, torch.float32).reshape(-1)
    if age.numel() == 1:
        age = age.expand(B)
    if age.numel() != B:
        raise RuntimeError(f"age must have 1 or {B} elements, got {age.numel()}")
    age = age.contiguous()
    call = _Call(arch, dev, _MODES[mode], *check_masks(arch, B, dev, mask1, mask2))
    return _TrainForward.apply(call, x, age, *params)


class B200TrainableMyCNN(B200MyCNN):
    """A :class:`B200MyCNN` that trains with torch autograd and any optimizer (bin/utils.py:183-227)::

        model = B200TrainableMyCNN.from_reference(sd).to("cuda")
        criterion = nn.BCEWithLogitsLoss(pos_weight=torch.tensor(13.5, device="cuda"))
        optimizer = torch.optim.Adam(model.parameters(), lr=1e-5)
        model.train()
        optimizer.zero_grad(); loss = criterion(model(x, age), y); loss.backward(); optimizer.step()
        model.eval(); logits = model(x_test, age_test)

    Every parameter of the reference requires grad (5957 for MyCNN5, bin/explore_torch.ipynb:2117); the ones its
    forward never uses (``out1``, ``out2``, ``age_fn``) keep ``.grad is None``.  In train mode the dropout masks are
    drawn on the device with ``p = self.dropout.p`` from torch's default CUDA generator."""

    def __init__(self, arch: ArchConfig = ArchConfig(), *a, **kw):
        check_trainable(arch)
        super().__init__(arch, *a, **kw)
        self.requires_grad_(True)

    def train(self, mode: bool = True):
        return nn.Module.train(self, mode)

    def draw_masks(self, B: int):
        """The two nn.Dropout masks of bin/models.py:25,28 with ``p = self.dropout.p``, from torch's default generator."""
        return draw_masks(self.arch, B, float(self.dropout.p), self._device())

    def forward(self, x: torch.Tensor, age: torch.Tensor) -> torch.Tensor:
        """``model(x, age)`` (bin/models.py:22-36): differentiable in train mode, the inference path in eval mode."""
        if not self.training:
            return super().forward(x, age)
        if self._device().type != "cuda":
            raise RuntimeError("B200TrainableMyCNN needs the model on a CUDA device to train (there is no CPU fallback)")
        B = x.shape[0]
        mode = "sequence" if (self.batch_mode == "sequence" and B > 1) else "independent"
        m1, m2 = self.draw_masks(B)
        named = dict(self.named_parameters())
        return mycnn_train_forward(x, age, [named[k] for k in BLOB_KEYS], self.arch, mode, m1, m2)
