"""One training step on the device (SURVEY.md section 8, row f4).

The reference trains with ``utils.train`` (bin/utils.py:183-227): per batch

    optimizer.zero_grad(); output = model(input, age); loss = criterion(output, target)
    loss.backward(); optimizer.step()

with ``criterion = nn.BCEWithLogitsLoss(pos_weight=pos_weight)``, ``pos_weight = num_negatives / num_positives``,
and ``torch.optim.Adam`` (bin/explore_torch.ipynb:3170,3204-3205).  :class:`B200Trainer` is that loop body as ONE
C-ABI call (``b2cnn_train_step``, or ``b2cnn_train_step_weighted`` when ``pos_weight`` is given; csrc/b2cnn_train.cu:
hand-written forward-with-saved-activations, BPTT over the batch axis, pooling/conv backward, Adam) on a
:class:`B200MyCNN`'s parameters::

    trainer = B200Trainer(model, lr=1e-5, pos_weight=13.5)
    for x, age, y in loader:                       # x [B,10,120] or waveform windows [B,3,75000]; age [B], y [B] in {0,1}
        loss = trainer.step(x, age, y)             # == the five reference lines above
    model.predict(...)                             # scores with the updated weights

``mode="sequence"`` (default) is what ``model(input_batch, age)`` computes in the reference: the LSTM scans
the batch axis (bin/models.py:29-30).  Dropout (bin/models.py:15, p = 0.1) uses masks drawn by torch on the
device; torch's own Philox stream cannot be reproduced by another implementation, so parity tests pass the
same explicit masks to both sides.

Any other loss or optimizer: :class:`~tskd_b200.autograd.B200TrainableMyCNN` runs the same kernels under torch autograd.
"""
from __future__ import annotations

import ctypes
import math
from typing import Dict, Optional, Tuple

import torch

from . import capi
from .arch import BLOB_KEYS
from .autograd import check_masks, check_trainable, draw_masks
from .model import B200MyCNN


class B200Trainer:
    def __init__(self, model: B200MyCNN, lr: float = 1e-3, betas: Tuple[float, float] = (0.9, 0.999), eps: float = 1e-8,
                 mode: str = "sequence", dropout: float = 0.1, seed: int = 0, pos_weight: Optional[float] = None):
        """``pos_weight``: the class weight of ``nn.BCEWithLogitsLoss(pos_weight=...)`` (a positive number; None = the
        unweighted loss)."""
        check_trainable(model.arch)
        if mode not in ("sequence", "independent"):
            raise ValueError("mode must be 'sequence' or 'independent'")
        if not 0.0 <= float(dropout) < 1.0:
            raise ValueError("dropout must be in [0, 1)")
        if pos_weight is not None:
            pos_weight = float(pos_weight)
            if not (math.isfinite(pos_weight) and pos_weight > 0.0):
                raise ValueError("pos_weight must be a positive finite number")
        dev = model._device()
        if dev.type != "cuda":
            raise RuntimeError("B200Trainer needs the model on a CUDA device (there is no CPU fallback)")
        self.model, self.mode, self.dropout, self.pos_weight = model, mode, float(dropout), pos_weight
        self._lib = capi.load_library()
        self._cfg = capi.make_config(model.arch, dev.index if dev.index is not None else torch.cuda.current_device())
        self._opt = capi.Adam(lr, betas[0], betas[1], eps)
        self._params = model.packed_weights().to(dev).contiguous()          # master copy, updated in place by the library
        self._m = torch.zeros_like(self._params)
        self._v = torch.zeros_like(self._params)
        self._grads = torch.zeros_like(self._params)
        self._loss = torch.zeros(1, device=dev)
        self._ws: Optional[torch.Tensor] = None
        self._gen = torch.Generator(device=dev)
        self._gen.manual_seed(seed)
        self.steps = 0

    # ------------------------------------------------------------------
    def _views(self, flat: torch.Tensor) -> Dict[str, torch.Tensor]:
        sd, out, at = self.model.state_dict(), {}, 0
        for k in BLOB_KEYS:
            n = sd[k].numel()
            out[k] = flat[at:at + n].view(sd[k].shape)
            at += n
        return out

    def grads(self) -> Dict[str, torch.Tensor]:
        """d loss / d parameter of the most recent step, keyed like the reference's state_dict."""
        return self._views(self._grads)

    def draw_masks(self, B: int) -> Tuple[Optional[torch.Tensor], Optional[torch.Tensor]]:
        """The two nn.Dropout masks of bin/models.py:25,28, scaled by 1/(1-p) like torch's dropout, from the trainer's
        seeded generator."""
        return draw_masks(self.model.arch, B, self.dropout, self._params.device, self._gen)

    def step(self, x: torch.Tensor, age: torch.Tensor, target: torch.Tensor,
             masks: Optional[Tuple[Optional[torch.Tensor], Optional[torch.Tensor]]] = None, update: bool = True,
             seq_lengths=None) -> torch.Tensor:
        """zero_grad + forward + BCEWithLogitsLoss(pos_weight) + backward + Adam step; returns the batch loss (a 0-d device
        tensor).

        ``seq_lengths`` [n_0, ..., n_{N-1}] (sequence mode only; a list, tuple or integer tensor, each >= 1, adding up to
        B): the batch is N consecutive sequences -- one patient's windows each -- and the LSTM starts every one from the
        zero state, as ``torch.cat([model(x[o:o+n], age[o:o+n]) for ...])`` would; the loss is still the mean over all B
        windows and one Adam step updates the parameters."""
        dev = self._params.device
        a = self.model.arch
        if x.dim() != 3 or x.shape[1] != a.in_channels or x.shape[2] != a.window:
            raise RuntimeError(f"expected x of shape [B, {a.in_channels}, {a.window}], got {tuple(x.shape)}")
        B = x.shape[0]
        lens = None
        if seq_lengths is not None:
            if self.mode != "sequence":
                raise ValueError("seq_lengths needs a trainer in mode='sequence'")
            lens = capi.seq_lengths_array(seq_lengths, B)
        x = x.to(dev, torch.float32).contiguous()
        age = age.to(dev, torch.float32).reshape(-1).contiguous()
        target = target.to(dev, torch.float32).reshape(-1).contiguous()
        if age.numel() != B or target.numel() != B:
            raise RuntimeError("age and target must have one entry per window")
        m1, m2 = check_masks(a, B, dev, *(masks if masks is not None else self.draw_masks(B)))
        if lens is None:
            need = self._lib.b2cnn_train_workspace_bytes(ctypes.byref(self._cfg), B)
        else:
            need = self._lib.b2cnn_train_workspace_bytes_seq(ctypes.byref(self._cfg), B, lens, len(lens))
        if need < 0:
            capi.check(capi.EINVAL, "b2cnn_train_workspace_bytes")
        if self._ws is None or self._ws.numel() < need:
            self._ws = torch.empty(need, dtype=torch.uint8, device=dev)
        ptr = lambda t: ctypes.c_void_p(t.data_ptr()) if t is not None else None
        st = torch.cuda.current_stream(dev).cuda_stream
        head = (ctypes.byref(self._cfg), ptr(self._params), ptr(self._m), ptr(self._v), ptr(self._grads), self.steps + 1,
                ctypes.byref(self._opt), 1 if update else 0, ptr(x), B, ptr(age), ptr(target))
        tail = (capi.MODE_SEQUENCE if self.mode == "sequence" else capi.MODE_INDEPENDENT, ptr(m1), ptr(m2), ptr(self._loss),
                ptr(self._ws), need, ctypes.c_void_p(st))
        if lens is not None:
            pw = None if self.pos_weight is None else ctypes.byref(ctypes.c_float(self.pos_weight))
            capi.check(self._lib.b2cnn_train_step_seq(*head, pw, lens, len(lens), *tail[1:]), "b2cnn_train_step_seq")
        elif self.pos_weight is None:
            capi.check(self._lib.b2cnn_train_step(*head, *tail), "b2cnn_train_step")
        else:
            capi.check(self._lib.b2cnn_train_step_weighted(*head, self.pos_weight, *tail), "b2cnn_train_step_weighted")
        if update:
            self.steps += 1
            with torch.no_grad():                        # the inference kernels read the module's parameters
                sd = self.model.state_dict()
                for k, v in self._views(self._params).items():
                    sd[k].copy_(v)
            self.model.sync_weights()
        return self._loss[0].clone()
