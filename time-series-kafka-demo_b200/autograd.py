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

:func:`mycnn_train_forward` is the same computation as a function of explicit parameters and dropout masks, and
:func:`mycnn_train_record_forward` the same over every sliding window of whole recordings ``[B, C, N]``, each window
feature computed and back-propagated once.
"""
from __future__ import annotations

import ctypes
import operator
from typing import Optional, Sequence

import torch
import torch.nn as nn
from torch.autograd.function import once_differentiable

from . import capi
from .arch import BLOB_KEYS, ArchConfig
from .model import B200MyCNN, check_record_state

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


def check_record_batch(arch: ArchConfig, records: torch.Tensor, stride, age, window_counts):
    """The arguments of a whole-recording training call, refused (ValueError) before anything runs: ``records``
    [B, C, N] float32 / bfloat16, ``stride`` a positive multiple of the feature stride ``pool_s ** 2``, ``age`` a scalar
    or one value per recording, ``window_counts`` as :func:`capi.window_counts_array` takes it.  Returns ``(stride, age,
    counts, M, rarch)``: age flattened (still differentiable), the host counts array, the number of windows and the
    geometry of a window of N samples (the dropout masks' shape)."""
    C = arch.in_channels
    if not torch.is_tensor(records) or records.dim() != 3 or records.shape[1] != C:
        got = tuple(records.shape) if torch.is_tensor(records) else type(records).__name__
        raise ValueError(f"expected records [B, {C}, N], got {got}")
    if records.dtype not in (torch.float32, torch.bfloat16):
        raise ValueError(f"records must be float32 or bfloat16, got {records.dtype}")
    B, N = records.shape[0], records.shape[2]
    if B < 1:
        raise ValueError("records must hold at least one recording")
    if isinstance(stride, bool):
        raise ValueError("stride must be an integer, got bool")
    try:
        stride = operator.index(stride)
    except TypeError:
        raise ValueError(f"stride must be an integer, got {type(stride).__name__}") from None
    F = arch.pool_s ** 2
    if stride < 1 or stride % F:
        raise ValueError(f"stride must be a positive multiple of the feature stride {F}, got {stride}")
    counts, M = capi.window_counts_array(window_counts, B, N, arch.window, stride)
    age = (age if torch.is_tensor(age) else torch.tensor(age, dtype=torch.float32)).reshape(-1)
    if age.numel() not in (1, B):
        raise ValueError(f"age must be a scalar or have {B} elements (one per recording), got {age.numel()}")
    return stride, age, counts, M, arch.with_shape(C, N)


def window_ages(age: torch.Tensor, counts, M: int, device) -> torch.Tensor:
    """One age per window [M] from one per recording (or a scalar): every window of recording b takes age[b]
    (``get_arr``).  Differentiable, so autograd sums d age over each recording's windows."""
    age = age.to(device, torch.float32)
    if age.numel() == 1:
        return age.expand(M).contiguous()
    return age.repeat_interleave(torch.tensor(list(counts), device=device), output_size=M).contiguous()


def cut_record_windows(records: torch.Tensor, window: int, stride: int, counts, pool_s: int, mask1=None, mask2=None):
    """The windows the ``_record`` training calls train on, cut out as copies: ``[M, C, W]`` (recording-major, window
    order, ``counts[b]`` windows of recording b) and the recording's dropout masks cut the same way (window w of
    recording b: ``mask1[b, :, wS/pool_s : wS/pool_s + P1]`` and ``mask2[b, wS/pool_s**2 : wS/pool_s**2 + L]``), or None
    where a mask is None.  ``B200Trainer.step`` on these equals ``step_record`` on the recordings."""
    counts = [int(c) for c in counts]
    sel = [(b, w) for b, n in enumerate(counts) for w in range(n)]
    bi = torch.tensor([b for b, _ in sel], device=records.device)
    wi = torch.tensor([w for _, w in sel], device=records.device)
    x = records.unfold(2, window, stride)[bi, :, wi]
    out = [x.contiguous()]
    for m, unit in ((mask1, pool_s), (mask2, pool_s ** 2)):
        if m is None:
            out.append(None)
            continue
        P = m.shape[-1] - (records.shape[2] - window) // unit          # the window's P1 / L
        cut = m.unfold(-1, P, stride // unit)
        out.append((cut[bi, :, wi] if m.dim() == 3 else cut[bi, wi]).contiguous())
    return tuple(out)


class _TrainForward(torch.autograd.Function):
    """Inputs: a :class:`_Call` (non-tensor), x [B,C,W] fp32 (with a record call the recordings [B,C,N]), age [rows]
    fp32, then the 14 ``BLOB_KEYS`` tensors."""

    @staticmethod
    def forward(ctx, call, x, age, *params):
        dev = x.device
        blob = torch.cat([p.detach().reshape(-1) for p in params])               # the packed blob (include/b2cnn.h)
        B = x.shape[0]
        ws = torch.empty(call.workspace_bytes(B), dtype=torch.uint8, device=dev)
        z = torch.empty(age.numel(), dtype=torch.float32, device=dev)
        st = torch.cuda.current_stream(dev).cuda_stream
        if call.rec is not None:
            N, S, counts, _ = call.rec
            rc = call.lib.b2cnn_train_forward_record(ctypes.byref(call.cfg), _ptr(blob), _ptr(x), B, N, S, counts, call.mode, _ptr(age),
                                                     _ptr(call.mask1), _ptr(call.mask2), _ptr(z), _ptr(ws), ws.numel(), ctypes.c_void_p(st))
        elif call.lens is None:
            rc = call.lib.b2cnn_train_forward(ctypes.byref(call.cfg), _ptr(blob), _ptr(x), B, _ptr(age), call.mode,
                                              _ptr(call.mask1), _ptr(call.mask2), _ptr(z), _ptr(ws), ws.numel(), ctypes.c_void_p(st))
        else:
            rc = call.lib.b2cnn_train_forward_seq(ctypes.byref(call.cfg), _ptr(blob), _ptr(x), B, _ptr(age), call.lens, len(call.lens),
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
        flags = capi.TRAIN_FROZEN_CONV if frozen else 0
        if call.rec is not None:
            N, S, counts, _ = call.rec
            rc = call.lib.b2cnn_train_backward_record(ctypes.byref(call.cfg), _ptr(blob), _ptr(x), B, N, S, counts, call.mode, _ptr(age),
                                                      _ptr(call.mask1), _ptr(call.mask2), _ptr(dz), _ptr(grads), _ptr(dx), _ptr(dage), flags,
                                                      _ptr(ws), ws.numel(), ctypes.c_void_p(st))
        elif call.lens is None:
            rc = call.lib.b2cnn_train_backward_ex(ctypes.byref(call.cfg), _ptr(blob), _ptr(x), B, _ptr(age), call.mode, _ptr(call.mask1),
                                                  _ptr(call.mask2), _ptr(dz), _ptr(grads), _ptr(dx), _ptr(dage), flags, _ptr(ws),
                                                  ws.numel(), ctypes.c_void_p(st))
        else:
            rc = call.lib.b2cnn_train_backward_seq(ctypes.byref(call.cfg), _ptr(blob), _ptr(x), B, _ptr(age), call.lens, len(call.lens),
                                                   _ptr(call.mask1), _ptr(call.mask2), _ptr(dz), _ptr(grads), _ptr(dx), _ptr(dage), flags,
                                                   _ptr(ws), ws.numel(), ctypes.c_void_p(st))
        capi.check(rc, "b2cnn_train_backward")
        return (None, dx, dage, *_param_grads(grads, ctx.shapes, ctx.needs_input_grad[3:]))


def _param_grads(grads, shapes, needs):
    """the packed gradient blob as one tensor per parameter (None where none is needed)"""
    out, at = [], 0
    for shape, need in zip(shapes, needs):
        n = shape.numel()
        out.append(grads[at:at + n].view(shape) if need else None)
        at += n
    return out


class _TrainRecordState(torch.autograd.Function):
    """The sequence-mode ``_record`` call with each recording's LSTM state as an input and an output.  Inputs: a
    :class:`_Call` with ``rec`` set, the recordings [B,C,N] fp32, age [M] fp32, state [B,2,2,16] fp32 or None (zeros),
    then the 14 ``BLOB_KEYS`` tensors.  Outputs: the logits [M] and the state after each recording's last counted window
    [B,2,2,16]; both are differentiable, and so is the input state."""

    @staticmethod
    def forward(ctx, call, x, age, state, *params):
        dev = x.device
        blob = torch.cat([p.detach().reshape(-1) for p in params])
        B = x.shape[0]
        N, S, counts, _ = call.rec
        ws = torch.empty(call.workspace_bytes(B), dtype=torch.uint8, device=dev)
        z = torch.empty(age.numel(), dtype=torch.float32, device=dev)
        state_out = torch.empty(B, 2, 2, 16, dtype=torch.float32, device=dev)
        st = torch.cuda.current_stream(dev).cuda_stream
        rc = call.lib.b2cnn_train_forward_record_state(ctypes.byref(call.cfg), _ptr(blob), _ptr(x), B, N, S, counts, call.mode, _ptr(age),
                                                       _ptr(call.mask1), _ptr(call.mask2), _ptr(state), _ptr(state_out), _ptr(z),
                                                       _ptr(ws), ws.numel(), ctypes.c_void_p(st))
        capi.check(rc, "b2cnn_train_forward_record_state")
        ctx.call, ctx.blob, ctx.ws = call, blob, ws
        ctx.shapes = [p.shape for p in params]
        ctx.save_for_backward(x, age, state)
        return z, state_out

    @staticmethod
    @once_differentiable
    def backward(ctx, dz, dstate):
        call, blob, ws = ctx.call, ctx.blob, ctx.ws
        x, age, state = ctx.saved_tensors
        B = x.shape[0]
        N, S, counts, _ = call.rec
        dz = dz.to(torch.float32).contiguous()
        dstate = dstate.to(torch.float32).contiguous()
        grads = torch.empty_like(blob)
        dx = torch.empty_like(x) if ctx.needs_input_grad[1] else None
        dage = torch.empty_like(age) if ctx.needs_input_grad[2] else None
        dstate_in = torch.empty_like(dstate) if ctx.needs_input_grad[3] else None
        frozen = dx is None and not any(ctx.needs_input_grad[4:8])
        st = torch.cuda.current_stream(x.device).cuda_stream
        rc = call.lib.b2cnn_train_backward_record_state(ctypes.byref(call.cfg), _ptr(blob), _ptr(x), B, N, S, counts, call.mode, _ptr(age),
                                                        _ptr(call.mask1), _ptr(call.mask2), _ptr(state), _ptr(dz), _ptr(dstate),
                                                        _ptr(grads), _ptr(dx), _ptr(dage), _ptr(dstate_in),
                                                        capi.TRAIN_FROZEN_CONV if frozen else 0, _ptr(ws), ws.numel(), ctypes.c_void_p(st))
        capi.check(rc, "b2cnn_train_backward_record_state")
        return (None, dx, dage, dstate_in, *_param_grads(grads, ctx.shapes, ctx.needs_input_grad[4:]))


class _Call:
    """What one forward / backward pair shares besides tensors: the library, its configuration, mode, masks, sequence
    lengths (the host array of the _seq calls, or None) and, for the _record calls, (N, stride, counts array, M)."""

    def __init__(self, arch: ArchConfig, device: torch.device, mode: int, mask1, mask2, lens=None, rec=None):
        self.lib = capi.load_library()
        self.cfg = capi.make_config(arch, device.index if device.index is not None else torch.cuda.current_device())
        self.mode, self.mask1, self.mask2, self.lens, self.rec = mode, mask1, mask2, lens, rec

    def workspace_bytes(self, B: int) -> int:
        if self.rec is not None:
            N, S, counts, _ = self.rec
            need = int(self.lib.b2cnn_train_workspace_bytes_record(ctypes.byref(self.cfg), B, N, S, counts, self.mode))
        elif self.lens is None:
            need = int(self.lib.b2cnn_train_workspace_bytes(ctypes.byref(self.cfg), B))
        else:
            need = int(self.lib.b2cnn_train_workspace_bytes_seq(ctypes.byref(self.cfg), B, self.lens, len(self.lens)))
        if need < 0:
            capi.check(capi.EINVAL, "b2cnn_train_workspace_bytes")
        return need


def _check_params(params: Sequence[torch.Tensor], arch: ArchConfig) -> torch.device:
    """The 14 ``BLOB_KEYS`` tensors of ``arch``: float32, on one CUDA device (returned)."""
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
    return dev


def mycnn_train_forward(x: torch.Tensor, age: torch.Tensor, params: Sequence[torch.Tensor], arch: ArchConfig,
                        mode: str = "sequence", mask1: Optional[torch.Tensor] = None,
                        mask2: Optional[torch.Tensor] = None, seq_lengths=None) -> torch.Tensor:
    """Logits [B] of the model in train() mode (bin/models.py:22-36), differentiable in ``x``, ``age`` and ``params``.

    ``params``: the 14 tensors of ``BLOB_KEYS`` in that order, on one CUDA device.  ``x`` [B,C,W] (fp32 or bf16; cast
    to fp32), ``age`` 1 or B values.  ``mode``: "sequence" (the LSTM scans the batch axis, as ``model(x, age)`` does in
    the reference) or "independent" (every window from the zero state).  ``mask1`` [B, c_mid, P1] / ``mask2``
    [B, L_out]: the two dropout masks, already scaled by 1/(1-p); None = no dropout.  ``seq_lengths`` (mode "sequence"
    only; a list, tuple or integer tensor, each >= 1, adding up to B): the batch is that many consecutive sequences, each
    scanned from the zero LSTM state, as ``torch.cat([model(x[o:o+n], age[o:o+n]) for ...])``."""
    check_trainable(arch)
    if mode not in _MODES:
        raise ValueError("mode must be 'sequence' or 'independent'")
    if seq_lengths is not None and mode != "sequence":
        raise ValueError("seq_lengths is only accepted with mode='sequence'")
    dev = _check_params(params, arch)
    if x.dim() != 3 or x.shape[1] != arch.in_channels or x.shape[2] != arch.window:
        raise RuntimeError(f"expected x of shape [B, {arch.in_channels}, {arch.window}], got {tuple(x.shape)}")
    B = x.shape[0]
    if B < 1:
        raise RuntimeError("expected at least one window")
    lens = None
    if seq_lengths is not None:
        lens = capi.seq_lengths_array(seq_lengths, B)
        if torch.as_tensor(age).dim() > 1:
            raise ValueError(f"with seq_lengths, age must have 1 or {B} elements (one per window), got shape {tuple(torch.as_tensor(age).shape)}")
    x = x.to(dev, torch.float32).contiguous()
    age = torch.as_tensor(age).to(dev, torch.float32).reshape(-1)
    if age.numel() == 1:
        age = age.expand(B)
    if age.numel() != B:
        raise RuntimeError(f"age must have 1 or {B} elements, got {age.numel()}")
    age = age.contiguous()
    call = _Call(arch, dev, _MODES[mode], *check_masks(arch, B, dev, mask1, mask2), lens=lens)
    return _TrainForward.apply(call, x, age, *params)


def mycnn_train_record_forward(records: torch.Tensor, stride: int, age, params: Sequence[torch.Tensor], arch: ArchConfig,
                               mode: str = "sequence", mask1: Optional[torch.Tensor] = None, mask2: Optional[torch.Tensor] = None,
                               window_counts=None, state=None, return_state: bool = False):
    """Logits [M] of every counted window of whole recordings in train() mode, differentiable in ``records``, ``age``
    and ``params``; each window feature is computed, and back-propagated, once however many windows share it.

    ``records`` [B, C, N] (fp32 or bf16; cast to fp32); window w of recording b is ``records[b, :, w*stride :
    w*stride + W]``, for w < ``window_counts[b]`` (default: all n_w = (N - W) // stride + 1 of them; a count may be
    smaller, down to 0, so recordings of different lengths can be padded to one N).  The logits are recording-major, in
    window order.  ``stride``: a positive multiple of the feature stride ``pool_s ** 2``.  ``age``: a scalar or one value
    per recording, every window of recording b taking age[b] (its gradient sums over the recording's windows).
    ``mode``: "sequence" (each recording's windows one sequence, the LSTM from the zero state -- ``seq_lengths`` = the
    non-zero counts) or "independent".  ``mask1`` [B, c_mid, P1(N)] / ``mask2`` [B, L(N)]: the recording's dropout
    masks, the geometry of a window of N samples (``arch.with_shape(C, N)``); window w uses the slices at its own
    positions, so a feature two windows share is dropped in both or in neither (the one difference from cutting the
    windows first and drawing their masks independently).  Samples no counted window reads change nothing, NaN
    included, and get a zero gradient.

    State across calls (mode "sequence" only, else ValueError): ``state`` ``[B, 2, 2, 16]``, [recording][layer][h |
    c][unit] (as ``nn.LSTM``'s tuple: ``h = state[:, :, 0].transpose(0, 1)``, ``c = state[:, :, 1].transpose(0, 1)``), is
    the state recording b's LSTM starts from (None: zeros); it may require grad.  ``return_state=True`` returns ``(z,
    state_out)``, ``state_out[b]`` the state after recording b's last counted window (``state[b]`` itself for a count of
    0), differentiable too: chaining two calls through it and back-propagating once gives the gradients of one call over
    the whole recordings (full back-propagation through time); ``state_out.detach()`` cuts it (truncated)."""
    check_trainable(arch)
    if mode not in _MODES:
        raise ValueError("mode must be 'sequence' or 'independent'")
    dev = _check_params(params, arch)
    stride, age, counts, M, rarch = check_record_batch(arch, records, stride, age, window_counts)
    check_record_state(records, mode, state, return_state)
    B, N = records.shape[0], records.shape[2]
    masks = check_masks(rarch, B, dev, mask1, mask2)
    records = records.to(dev, torch.float32).contiguous()
    call = _Call(arch, dev, _MODES[mode], *masks, rec=(N, stride, counts, M))
    if state is None and not return_state:
        return _TrainForward.apply(call, records, window_ages(age, counts, M, dev), *params)
    if state is not None:
        state = state.to(dev, torch.float32).contiguous()
    z, state_out = _TrainRecordState.apply(call, records, window_ages(age, counts, M, dev), state, *params)
    return (z, state_out) if return_state else z


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

    def draw_masks(self, B: int, n_samples: Optional[int] = None):
        """The two nn.Dropout masks of bin/models.py:25,28 with ``p = self.dropout.p``, from torch's default generator;
        with ``n_samples``, those of B recordings of that many samples (:meth:`forward_record`)."""
        arch = self.arch if n_samples is None else self.arch.with_shape(self.arch.in_channels, n_samples)
        return draw_masks(arch, B, float(self.dropout.p), self._device())

    def forward(self, x: torch.Tensor, age: torch.Tensor, seq_lengths=None) -> torch.Tensor:
        """``model(x, age)`` (bin/models.py:22-36): differentiable in train mode, the inference path in eval mode.
        ``seq_lengths``: the batch is that many consecutive sequences, each from the zero LSTM state, in either mode
        (``batch_mode == "sequence"`` only; see :func:`mycnn_train_forward`)."""
        if seq_lengths is not None and self.batch_mode != "sequence":
            raise ValueError("seq_lengths needs batch_mode == 'sequence'")
        if not self.training:
            return super().forward(x, age, seq_lengths)
        if self._device().type != "cuda":
            raise RuntimeError("B200TrainableMyCNN needs the model on a CUDA device to train (there is no CPU fallback)")
        B = x.shape[0]
        if seq_lengths is not None:
            capi.seq_lengths_array(seq_lengths, B)          # refused before the masks are drawn
        mode = "sequence" if (self.batch_mode == "sequence" and (B > 1 or seq_lengths is not None)) else "independent"
        m1, m2 = self.draw_masks(B)
        named = dict(self.named_parameters())
        return mycnn_train_forward(x, age, [named[k] for k in BLOB_KEYS], self.arch, mode, m1, m2, seq_lengths)

    def forward_record(self, records: torch.Tensor, stride: int, age, window_counts=None, state=None, return_state: bool = False):
        """Logits [M] of every counted window of whole recordings ``[B, C, N]`` (see :func:`mycnn_train_record_forward`),
        recording-major: in train mode differentiable, with the dropout masks drawn at the recording's geometry and the
        LSTM over each recording's windows (``batch_mode == "sequence"``) or every window alone; in eval mode
        ``predict_record(records, stride, age, mode=batch_mode)`` with each row cut to its count.  ``state`` /
        ``return_state``: the LSTM state across calls (``batch_mode == "sequence"``; see
        :func:`mycnn_train_record_forward`); in eval mode ``predict_record``'s, which counts every window."""
        stride, _, counts, M, _ = check_record_batch(self.arch, records, stride, age, window_counts)
        check_record_state(records, self.batch_mode, state, return_state)
        if not self.training and (state is not None or return_state):
            n_w = (records.shape[2] - self.arch.window) // stride + 1 if records.shape[2] >= self.arch.window else 0
            if any(int(c) != n_w for c in counts):
                raise ValueError("in eval mode the LSTM state needs every window counted (window_counts=None)")
            return self.predict_record(records, stride, age, mode=self.batch_mode, state=state, return_state=return_state)
        if not self.training:
            out = self.predict_record(records, stride, age, mode=self.batch_mode)
            keep = torch.arange(out.shape[1], device=out.device) < torch.tensor(list(counts), device=out.device)[:, None]
            return out[keep]
        if self._device().type != "cuda":
            raise RuntimeError("B200TrainableMyCNN needs the model on a CUDA device to train (there is no CPU fallback)")
        m1, m2 = self.draw_masks(records.shape[0], records.shape[2])
        named = dict(self.named_parameters())
        return mycnn_train_record_forward(records, stride, age, [named[k] for k in BLOB_KEYS], self.arch, self.batch_mode, m1, m2,
                                          window_counts, state, return_state)
