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
from typing import Dict, List, Optional, Tuple

import torch

from . import capi
from .arch import BLOB_KEYS
from .autograd import check_masks, check_record_batch, check_trainable, draw_masks, window_ages
from .model import B200MyCNN, check_head_models, check_record_state


def _check_options(arch, mode: str, dropout: float, pos_weight: Optional[float]) -> Optional[float]:
    """The options both trainers take, refused before anything runs; returns pos_weight as a float (None: unweighted)."""
    check_trainable(arch)
    if mode not in ("sequence", "independent"):
        raise ValueError("mode must be 'sequence' or 'independent'")
    if not 0.0 <= float(dropout) < 1.0:
        raise ValueError("dropout must be in [0, 1)")
    if pos_weight is not None:
        pos_weight = float(pos_weight)
        if not (math.isfinite(pos_weight) and pos_weight > 0.0):
            raise ValueError("pos_weight must be a positive finite number")
    return pos_weight


class _FusedTrainer:
    """What :class:`B200Trainer` and :class:`B200HeadTrainer` share: the checks of their options and batches, the
    library's configuration and Adam arguments, the dropout generator and the workspace."""

    def _setup(self, who: str, model: B200MyCNN, dev: torch.device, lr: float, betas: Tuple[float, float], eps: float, mode: str,
               dropout: float, seed: int, pos_weight: Optional[float], heads=None) -> None:
        """After the checks of :func:`_check_options`: refuses a model off the GPU, then binds the library to its device
        and takes the blob of ``model`` (or with ``heads`` one row per head), its Adam state and gradients."""
        if dev.type != "cuda":
            raise RuntimeError(f"{who} needs the model on a CUDA device (there is no CPU fallback)")
        self.model, self.mode, self.dropout, self.pos_weight = model, mode, float(dropout), pos_weight
        self._mode = capi.MODE_SEQUENCE if mode == "sequence" else capi.MODE_INDEPENDENT
        self._lib = capi.load_library()
        self._cfg = capi.make_config(model.arch, dev.index if dev.index is not None else torch.cuda.current_device())
        self._opt = capi.Adam(lr, betas[0], betas[1], eps)
        if heads is None:
            self._params = model.packed_weights().to(dev).contiguous()     # master copy, updated in place by the library
        else:
            self._params = torch.stack([h.packed_weights().to(dev) for h in heads]).contiguous()   # [K, n]: one blob per head
        self._m = torch.zeros_like(self._params)
        self._v = torch.zeros_like(self._params)
        self._grads = torch.zeros_like(self._params)
        self._loss = torch.zeros(1 if heads is None else len(heads), device=dev)
        self._ws: Optional[torch.Tensor] = None
        self._gen = torch.Generator(device=dev)
        self._gen.manual_seed(seed)
        self.steps = 0

    def _views(self, flat: torch.Tensor) -> Dict[str, torch.Tensor]:
        sd, out, at = self.model.state_dict(), {}, 0
        for k in BLOB_KEYS:
            n = sd[k].numel()
            out[k] = flat[at:at + n].view(sd[k].shape)
            at += n
        return out

    def draw_masks(self, B: int, n_samples: Optional[int] = None) -> Tuple[Optional[torch.Tensor], Optional[torch.Tensor]]:
        """The two nn.Dropout masks of bin/models.py:25,28, scaled by 1/(1-p) like torch's dropout, from the trainer's
        seeded generator: of B windows, or with ``n_samples`` of B recordings of that many samples (:meth:`step_record`).
        A :class:`B200HeadTrainer` shares one draw between all its heads."""
        arch = self.model.arch if n_samples is None else self.model.arch.with_shape(self.model.arch.in_channels, n_samples)
        return draw_masks(arch, B, self.dropout, self._params.device, self._gen)

    @staticmethod
    def _ptr(t):
        return ctypes.c_void_p(t.data_ptr()) if t is not None else None

    def _pos_weight(self):
        """pos_weight as the ``const float *`` of the C calls (NULL: the unweighted loss)."""
        return None if self.pos_weight is None else ctypes.byref(ctypes.c_float(self.pos_weight))

    def _stream(self):
        return ctypes.c_void_p(torch.cuda.current_stream(self._params.device).cuda_stream)

    def _workspace(self, need: int, what: str) -> torch.Tensor:
        if need < 0:
            capi.check(capi.EINVAL, what)
        if self._ws is None or self._ws.numel() < need:
            self._ws = torch.empty(need, dtype=torch.uint8, device=self._params.device)
        return self._ws

    def _window_batch(self, x: torch.Tensor, age: torch.Tensor, target: torch.Tensor, masks, seq_lengths):
        """A batch of :meth:`step` on the device: ``(x, age, target, B, lens, mask1, mask2)``, ``lens`` the host array of
        ``seq_lengths`` (None without)."""
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
        return x, age, target, B, lens, m1, m2

    def _record_batch(self, records: torch.Tensor, stride, age, target, window_counts, masks, state, return_state):
        """A batch of :meth:`step_record` on the device: ``(records, B, N, stride, counts, age, target, mask1, mask2)``,
        one age per window."""
        dev = self._params.device
        stride, age, counts, M, rarch = check_record_batch(self.model.arch, records, stride, age, window_counts)
        check_record_state(records, self.mode, state, return_state)
        B, N = records.shape[0], records.shape[2]
        target = torch.as_tensor(target).detach().to(dev, torch.float32).reshape(-1).contiguous()
        if target.numel() != M:
            raise ValueError(f"target must have one entry per window ({M}), got {target.numel()}")
        m1, m2 = check_masks(rarch, B, dev, *(masks if masks is not None else self.draw_masks(B, N)))
        records = records.to(dev, torch.float32).contiguous()
        return records, B, N, stride, counts, window_ages(age.detach(), counts, M, dev), target, m1, m2


class B200Trainer(_FusedTrainer):
    def __init__(self, model: B200MyCNN, lr: float = 1e-3, betas: Tuple[float, float] = (0.9, 0.999), eps: float = 1e-8,
                 mode: str = "sequence", dropout: float = 0.1, seed: int = 0, pos_weight: Optional[float] = None):
        """``pos_weight``: the class weight of ``nn.BCEWithLogitsLoss(pos_weight=...)`` (a positive number; None = the
        unweighted loss)."""
        pos_weight = _check_options(model.arch, mode, dropout, pos_weight)
        self._setup("B200Trainer", model, model._device(), lr, betas, eps, mode, dropout, seed, pos_weight)

    # ------------------------------------------------------------------
    def grads(self) -> Dict[str, torch.Tensor]:
        """d loss / d parameter of the most recent step, keyed like the reference's state_dict."""
        return self._views(self._grads)

    def step(self, x: torch.Tensor, age: torch.Tensor, target: torch.Tensor,
             masks: Optional[Tuple[Optional[torch.Tensor], Optional[torch.Tensor]]] = None, update: bool = True,
             seq_lengths=None) -> torch.Tensor:
        """zero_grad + forward + BCEWithLogitsLoss(pos_weight) + backward + Adam step; returns the batch loss (a 0-d device
        tensor).

        ``seq_lengths`` [n_0, ..., n_{N-1}] (sequence mode only; a list, tuple or integer tensor, each >= 1, adding up to
        B): the batch is N consecutive sequences -- one patient's windows each -- and the LSTM starts every one from the
        zero state, as ``torch.cat([model(x[o:o+n], age[o:o+n]) for ...])`` would; the loss is still the mean over all B
        windows and one Adam step updates the parameters."""
        x, age, target, B, lens, m1, m2 = self._window_batch(x, age, target, masks, seq_lengths)
        if lens is None:
            need = self._lib.b2cnn_train_workspace_bytes(ctypes.byref(self._cfg), B)
        else:
            need = self._lib.b2cnn_train_workspace_bytes_seq(ctypes.byref(self._cfg), B, lens, len(lens))
        ws = self._workspace(need, "b2cnn_train_workspace_bytes")
        p = self._ptr
        head = (ctypes.byref(self._cfg), p(self._params), p(self._m), p(self._v), p(self._grads), self.steps + 1,
                ctypes.byref(self._opt), 1 if update else 0, p(x), B, p(age), p(target))
        tail = (p(m1), p(m2), p(self._loss), p(ws), need, self._stream())
        if lens is not None:
            capi.check(self._lib.b2cnn_train_step_seq(*head, self._pos_weight(), lens, len(lens), *tail), "b2cnn_train_step_seq")
        elif self.pos_weight is None:
            capi.check(self._lib.b2cnn_train_step(*head, self._mode, *tail), "b2cnn_train_step")
        else:
            capi.check(self._lib.b2cnn_train_step_weighted(*head, self.pos_weight, self._mode, *tail), "b2cnn_train_step_weighted")
        return self._finish(update)

    def step_record(self, records: torch.Tensor, stride: int, age, target: torch.Tensor, window_counts=None,
                    masks: Optional[Tuple[Optional[torch.Tensor], Optional[torch.Tensor]]] = None, update: bool = True,
                    state=None, return_state: bool = False):
        """:meth:`step` over every counted window of whole recordings ``[B, C, N]`` (fp32 or bf16), each window feature
        computed and back-propagated once: window w of recording b is ``records[b, :, w*stride : w*stride + W]`` for
        w < ``window_counts[b]`` (default: all n_w = (N - W) // stride + 1; fewer, down to 0, pads a ragged batch to one
        N).  ``stride``: a positive multiple of ``pool_s ** 2``.  ``age``: a scalar or one per recording; ``target``: one
        per window, recording-major [M].  In sequence mode each recording's windows are one sequence, the LSTM starting
        from zero (``step(windows, ..., seq_lengths=`` the non-zero counts ``)``); in independent mode every window is
        alone.  The loss is the mean over the M windows.  ``masks``: the recording's dropout masks [B, c_mid, P1(N)] /
        [B, L(N)] (default :meth:`draw_masks` ``(B, N)``); window w uses the slices at its own positions, so a feature
        two windows share is dropped in both or in neither.  Samples no counted window reads (tails, gaps when stride >
        W, recordings with count 0) change nothing, NaN included.

        Truncated back-propagation through time (sequence mode only, else ValueError): ``state`` ``[B, 2, 2, 16]``
        ([recording][layer][h | c][unit]; None: zeros) is the LSTM state each recording starts from, and with
        ``return_state=True`` the call returns ``(loss, state_out)``, ``state_out`` detached: the state after each
        recording's last counted window (``state[b]`` for a count of 0), to pass to the step on the next chunk."""
        records, B, N, stride, counts, age, target, m1, m2 = self._record_batch(records, stride, age, target, window_counts, masks,
                                                                                state, return_state)
        need = self._lib.b2cnn_train_workspace_bytes_record(ctypes.byref(self._cfg), B, N, stride, counts, self._mode)
        ws = self._workspace(need, "b2cnn_train_workspace_bytes_record")
        p = self._ptr
        head = (ctypes.byref(self._cfg), p(self._params), p(self._m), p(self._v), p(self._grads), self.steps + 1, ctypes.byref(self._opt),
                1 if update else 0, p(records), B, N, stride, counts, self._mode, p(age), p(target), self._pos_weight(), p(m1), p(m2))
        tail = (p(self._loss), p(ws), need, self._stream())
        if state is None and not return_state:
            capi.check(self._lib.b2cnn_train_step_record(*head, *tail), "b2cnn_train_step_record")
            return self._finish(update)
        if state is not None:
            state = state.detach().to(self._params.device, torch.float32).contiguous()
        state_out = torch.empty(B, 2, 2, 16, dtype=torch.float32, device=self._params.device)
        capi.check(self._lib.b2cnn_train_step_record_state(*head, p(state), p(state_out), *tail), "b2cnn_train_step_record_state")
        loss = self._finish(update)
        return (loss, state_out) if return_state else loss

    def _finish(self, update: bool) -> torch.Tensor:
        if update:
            self.steps += 1
            with torch.no_grad():                        # the inference kernels read the module's parameters
                sd = self.model.state_dict()
                for k, v in self._views(self._params).items():
                    sd[k].copy_(v)
            self.model.sync_weights()
        return self._loss[0].clone()


class B200HeadTrainer(_FusedTrainer):
    """Train up to 8 candidate heads on one frozen front end in one fused step per batch.

    ``model``'s conv1 / conv2 are the front end: the conv forward runs once per step on them and nothing
    back-propagates into them.  Each of ``heads`` (1 to 8 distinct :class:`B200MyCNN` with the model's architecture,
    device and conv weights; ``model`` itself may be one of them) trains its own LSTM and ``out`` parameters with its own
    Adam state::

        trainer = B200HeadTrainer(model, [cand_a, cand_b, model], lr=[1e-3, 3e-4, 1e-4])
        for x, age, y in loader:
            losses = trainer.step(x, age, y)        # Tensor[K]: head i's loss
        model.predict_record(records, stride, ages, heads=trainer.heads)   # backtest them, then SlidingScorer.set_heads

    Every head sees the same features and the same dropout masks (one draw per step, :meth:`draw_masks`); row i is
    what :class:`B200Trainer` on a copy of head i gives for its LSTM / Linear entries with those masks.  ``lr`` is one
    float or one per head; betas, eps, ``pos_weight``, ``mode`` and ``dropout`` are shared.  After an update each head's
    state dict holds its new weights and :meth:`B200MyCNN.sync_weights` has run."""

    def __init__(self, model: B200MyCNN, heads, lr=1e-3, betas: Tuple[float, float] = (0.9, 0.999), eps: float = 1e-8,
                 mode: str = "sequence", dropout: float = 0.1, seed: int = 0, pos_weight: Optional[float] = None):
        if not isinstance(model, B200MyCNN):
            raise TypeError(f"model must be a B200MyCNN, got {type(model).__name__}")
        pos_weight = _check_options(model.arch, mode, dropout, pos_weight)
        dev = model._device()
        sd = model.state_dict()
        front = {k: sd[k] for k in BLOB_KEYS[:BLOB_KEYS.index("lstm.weight_ih_l0")]}

        def same_front_end(i, m):
            if m._device() != dev:
                return                                   # check_head_models refuses it next
            hsd = m.state_dict()
            bad = [k for k, v in front.items() if not torch.equal(hsd[k], v)]
            if bad:
                raise ValueError(f"heads[{i}] differs from the model's front end in {', '.join(bad)}")

        heads = check_head_models(heads, model.arch, dev, "B200HeadTrainer", "the model", "the model", extra=same_front_end)
        if not heads:
            raise ValueError("B200HeadTrainer needs at least one head")
        if len({id(h) for h in heads}) != len(heads):
            raise ValueError("heads must be distinct models")
        K = len(heads)
        if isinstance(lr, (int, float)) and not isinstance(lr, bool):
            lrs = [float(lr)] * K
        else:
            lrs = [float(v) for v in lr]
            if len(lrs) != K:
                raise ValueError(f"lr must be one float or {K} floats (one per head), got {len(lrs)}")
        if not all(math.isfinite(v) and v >= 0.0 for v in lrs):
            raise ValueError("every lr must be a finite number >= 0")
        self._setup("B200HeadTrainer", model, dev, 0.0, betas, eps, mode, dropout, seed, pos_weight, heads=heads)
        self.heads = heads
        self._lr = (ctypes.c_float * K)(*lrs)
        self._front = model.packed_weights().to(dev).contiguous()         # read for its conv entries only
        ptrs = lambda t: (ctypes.c_void_p * K)(*[t[i].data_ptr() for i in range(K)])
        self._pp, self._pm, self._pv, self._pg = ptrs(self._params), ptrs(self._m), ptrs(self._v), ptrs(self._grads)

    def grads(self) -> List[Dict[str, torch.Tensor]]:
        """d loss / d parameter of the most recent step, one dict per head, keyed like the reference's state_dict from
        ``lstm.weight_ih_l0`` on (the front end gets no gradient)."""
        first = BLOB_KEYS.index("lstm.weight_ih_l0")
        return [{k: v for k, v in self._views(self._grads[i]).items() if k in BLOB_KEYS[first:]} for i in range(len(self.heads))]

    def step(self, x: torch.Tensor, age: torch.Tensor, target: torch.Tensor,
             masks: Optional[Tuple[Optional[torch.Tensor], Optional[torch.Tensor]]] = None, update: bool = True,
             seq_lengths=None) -> torch.Tensor:
        """:meth:`B200Trainer.step` for every head at once, with its rules; returns the K heads' batch losses, a device
        tensor [K]."""
        x, age, target, B, lens, m1, m2 = self._window_batch(x, age, target, masks, seq_lengths)
        K, n_seq = len(self.heads), len(lens) if lens is not None else 0
        need = self._lib.b2cnn_train_heads_workspace_bytes(ctypes.byref(self._cfg), K, B, lens, n_seq)
        ws = self._workspace(need, "b2cnn_train_heads_workspace_bytes")
        p = self._ptr
        capi.check(self._lib.b2cnn_train_heads_step(ctypes.byref(self._cfg), p(self._front), K, self._pp, self._pm, self._pv, self._pg,
                                                    self._lr, self.steps + 1, ctypes.byref(self._opt), 1 if update else 0, p(x), B,
                                                    p(age), p(target), self._pos_weight(), self._mode, lens, n_seq, p(m1), p(m2),
                                                    p(self._loss), p(ws), need, self._stream()), "b2cnn_train_heads_step")
        return self._finish(update)

    def step_record(self, records: torch.Tensor, stride: int, age, target: torch.Tensor, window_counts=None,
                    masks: Optional[Tuple[Optional[torch.Tensor], Optional[torch.Tensor]]] = None, update: bool = True,
                    state=None, return_state: bool = False) -> torch.Tensor:
        """:meth:`B200Trainer.step_record` for every head at once, in both modes; returns the K heads' losses [K].
        Carrying an LSTM state across chunks (``state`` / ``return_state``) is not supported (ValueError)."""
        if state is not None or return_state:
            raise ValueError("B200HeadTrainer.step_record carries no LSTM state across calls (state / return_state)")
        records, B, N, stride, counts, age, target, m1, m2 = self._record_batch(records, stride, age, target, window_counts, masks,
                                                                                None, False)
        K = len(self.heads)
        need = self._lib.b2cnn_train_heads_workspace_bytes_record(ctypes.byref(self._cfg), K, B, N, stride, counts, self._mode)
        ws = self._workspace(need, "b2cnn_train_heads_workspace_bytes_record")
        p = self._ptr
        capi.check(self._lib.b2cnn_train_heads_step_record(ctypes.byref(self._cfg), p(self._front), K, self._pp, self._pm, self._pv,
                                                           self._pg, self._lr, self.steps + 1, ctypes.byref(self._opt), 1 if update else 0,
                                                           p(records), B, N, stride, counts, self._mode, p(age), p(target), self._pos_weight(),
                                                           p(m1), p(m2), p(self._loss), p(ws), need, self._stream()), "b2cnn_train_heads_step_record")
        return self._finish(update)

    def _finish(self, update: bool) -> torch.Tensor:
        if update:
            self.steps += 1
            with torch.no_grad():                        # the inference kernels read the module's parameters
                for i, h in enumerate(self.heads):
                    sd = h.state_dict()
                    for k, v in self._views(self._params[i]).items():
                        sd[k].copy_(v)
                    h.sync_weights()
        return self._loss.clone()
