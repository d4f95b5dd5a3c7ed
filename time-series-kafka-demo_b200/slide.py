"""``SlidingScorer`` -- long waveform windows scored incrementally (libb2cnn's b2cnn_slide_*, csrc/b2cnn_slide.cu).

The reference scores every patient with a window of the last W samples that slides by S samples
(bin/predictStream.py:248-252: 600 s every 60 s).  Instead of keeping a ``[P, C, W]`` buffer, shifting it and calling
``predict()`` on whole windows, a scorer keeps every patient's window features on the device; each ``push`` brings the
S new samples of all patients, computes only the features they complete and scores the P windows::

    scorer = SlidingScorer(model, n_patients=P, stride=7500)         # 60 s at 125 Hz
    for samples in triggers:                                         # [P, C, 7500] on the device
        logits = scorer.push(samples, age=ages)                      # None until the first W samples arrived

Patients come and go one at a time: ``admit(patients, history)`` restarts their streams (optionally from the samples a
monitor already holds), ``discharge(patients)`` stops scoring them; the others are not disturbed.

``export(patients)`` takes the listed patients' state out of a scorer (their window features, last samples and counts,
as plain tensors ``torch.save`` can write) and ``restore(patients, state)`` puts it into this or another scorer of
the same model front end, path and dtype, which then continues those streams bit for bit::

    torch.save(scorer.export(range(P)), "ward.pt")                   # before a restart
    scorer.restore(range(P), torch.load("ward.pt"))                  # in the new process: no window is lost

``set_heads(models)`` attaches up to 8 extra heads -- models with the scorer's architecture and conv weights whose
LSTM, Linear or age coefficient differ (a retrained candidate, an ensemble) -- scored at every push from the same
stored features, with no cold start and no second front end::

    scorer.set_heads([candidate])
    out = scorer.push(samples, age=ages, heads=True)                 # [2, P]: production row 0, candidate row 1

With ``shorter_windows=True`` a head may have a shorter window than the scorer's (risk over the last 60 s, 300 s and
600 s of one stream), scored from the tail of the same stored window instead of by a scorer of its own::

    scorer = SlidingScorer(m600, n_patients=P, stride=7500)          # W = 75000: 600 s at 125 Hz
    scorer.set_heads([m60, m300], shorter_windows=True)              # W_k = 7500 and 37500, the same conv weights
    out = scorer.push(samples, age=ages, heads=True)                 # [3, P] once the 60 s window is complete

``mode="sequence"`` scores every patient as ``utils.run_model`` scores a recording, live: the LSTM runs along the
patient's windows, its state (h and c of both layers, 256 bytes per patient) carried on the device from one scored
window to the next, so each push costs one LSTM step per patient however long the stay::

    scorer = SlidingScorer(model, n_patients=P, stride=7500, mode="sequence")
    for samples in triggers:
        logits = scorer.push(samples, age=ages)                      # model(windows since admission, age)[-1] per patient

For a patient whose stream is ``s`` (history first), with ``s0`` its ``samples_seen`` at the first push with
``samples_seen >= W`` and ``o = s0 - W``, the push at ``samples_seen == s0 + j * stride`` returns
``predict_record(s[:, :, o : s0 + j * stride], stride, age, mode="sequence")[:, j]`` -- bit for bit on the generic
path.  The state starts at zero at ``reset()``, ``admit()`` and ``discharge()``; a NaN sample poisons its patient's
state (NaN at every later push, as in ``run_model``) until ``admit()`` starts it again.
"""
from __future__ import annotations

import ctypes
import operator

import torch

from . import capi
from .model import HEAD_ARCH_FIELDS, check_head_models, check_lstm_state


class SlidingScorer:
    """P independent patient streams scored with the model's window ``W = model.arch.window`` every ``stride``
    samples.  After push n (from 1) a patient's window is the last W samples of its stream; ``push`` returns the
    ``Tensor[P]`` of ``predict(window, age, mode="independent")`` from the first push with ``n * stride >= W`` on,
    ``None`` before.  ``dtype`` is the dtype of the pushed samples (``torch.bfloat16`` or ``torch.float32``).

    Each patient has its own count of samples, ``samples_seen``: ``reset()`` starts all at 0, a push adds ``stride``,
    ``admit`` restarts listed patients (at the length of the history given), ``discharge`` sets -1.  Once ``admit`` or
    ``discharge`` was called, a patient's score is NaN until its count reaches W.

    ``path``: ``"tensorcore"`` (the default) runs the tensor-core kernels, which hold tanh models without affine of the
    MyCNN5 or MyCNN2/3/4 conv/pool geometry with 1 to 3 channels; ``"generic"`` runs exact fp32 CUDA-core kernels for
    any model the library accepts (its logits are ``predict()``'s with ``path="generic"`` and ``small_kernel=0``), with
    ``stride`` a multiple of the feature stride ``pool_s ** 2``; ``"auto"`` takes the tensor-core path where it holds
    the model and the generic one otherwise.  ``scorer.path`` tells which one runs.

    Extra heads: ``set_heads(models)`` attaches models of the same architecture and front-end (conv / affine) weights,
    ``push(..., heads=True)`` returns ``Tensor[1 + K, P]``, row 0 what ``push`` returns and row i ``heads[i - 1]``'s
    logits of the same windows.  ``heads`` is the tuple attached.  ``set_heads(models, shorter_windows=True)`` also
    takes heads whose window ``W_k <= W`` ends where the scorer's does (``W - W_k`` a multiple of the feature stride);
    ``head_windows`` lists each row's window.

    ``mode``: ``"independent"`` (the default) scores every window from the zero LSTM state, the reference's per-window
    call (bin/predictStream.py:157).  ``"sequence"`` carries each patient's LSTM state from its previous scored window,
    as ``model(windows, age)`` with the windows as the batch (bin/models.py:29-30, ``utils.run_model``) and as
    ``B200Trainer`` trains by default: ``push`` returns, for patient p, the output ``model(windows_p, age)`` gives for
    its last row, ``windows_p`` all of p's windows scored since its admission (or ``reset()``), in order.  The state
    is zeroed at ``reset()``, ``admit()`` and ``discharge()`` and does not advance while p's score is NaN for an
    incomplete window; the age scales the output only.  A sequence scorer takes no extra heads.  ``scorer.mode``
    tells which one runs."""

    ARCH_FIELDS = HEAD_ARCH_FIELDS

    PATHS = {"tensorcore": capi.PATH_TENSORCORE, "generic": capi.PATH_GENERIC, "auto": capi.PATH_AUTO}
    MODES = {"independent": capi.MODE_INDEPENDENT, "sequence": capi.MODE_SEQUENCE}
    LSTM_STATE = (2, 2, 16)                                             # [layer][h | c][unit] per patient
    mode = "independent"                                                # the instance's, set at construction
    STATE_HEADER = tuple(n for n, _ in capi.SlideStateHeader._fields_)

    def __init__(self, model, n_patients: int, stride: int, dtype=torch.bfloat16, path: str = "tensorcore",
                 mode: str = "independent"):
        if dtype not in (torch.bfloat16, torch.float32):
            raise ValueError("dtype must be torch.bfloat16 or torch.float32")
        if path not in self.PATHS:
            raise ValueError(f"path must be one of {sorted(self.PATHS)}, got {path!r}")
        if not isinstance(mode, str) or mode not in self.MODES:
            raise ValueError(f"mode must be one of {sorted(self.MODES)}, got {mode!r}")
        n_patients, stride = int(n_patients), int(stride)
        if n_patients < 1:
            raise ValueError(f"n_patients must be >= 1, got {n_patients}")
        W = model.arch.window
        F = 4 if path == "tensorcore" else model.arch.pool_s ** 2           # the feature stride in samples
        if stride < 1 or stride > W or stride % F:
            raise ValueError(f"stride must be a multiple of {F} in [{F}, {W}] (the window), got {stride}")
        self.model, self.n_patients, self.stride, self.dtype = model, n_patients, stride, dtype
        self.channels, self.window = model.arch.in_channels, W
        self._lib, h = model._ensure_handle()
        self._hv = h.value
        self.device = model._handle_device
        s = ctypes.c_void_p()
        with torch.cuda.device(self.device):
            if mode == "sequence":
                capi.check(self._lib.b2cnn_slide_create_ex(h, n_patients, stride, self._dt(), self.PATHS[path], capi.MODE_SEQUENCE,
                                                           ctypes.byref(s)), "b2cnn_slide_create_ex")
            elif path == "tensorcore":
                capi.check(self._lib.b2cnn_slide_create(h, n_patients, stride, self._dt(), ctypes.byref(s)), "b2cnn_slide_create")
            else:
                capi.check(self._lib.b2cnn_slide_create_path(h, n_patients, stride, self._dt(), self.PATHS[path], ctypes.byref(s)),
                           "b2cnn_slide_create_path")
        self._s = s
        self.mode = mode
        self._heads = ()
        self.path = "generic" if self._lib.b2cnn_slide_path(s) == capi.PATH_GENERIC else "tensorcore"
        self.window_index = -1
        hdr = capi.SlideStateHeader()
        capi.check(self._lib.b2cnn_slide_describe_state(s, ctypes.byref(hdr)), "b2cnn_slide_describe_state")
        # what an imported state must match here (its digest is checked by the library against the current weights)
        self._state_fields = {n: int(getattr(hdr, n)) for n in self.STATE_HEADER if n != "frontend_digest"}

    def _dt(self) -> int:
        return capi.DTYPE_BF16 if self.dtype == torch.bfloat16 else capi.DTYPE_F32

    def close(self):
        s, self._s = getattr(self, "_s", None), None
        if s is not None:
            self._lib.b2cnn_slide_destroy(s)

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def _handle(self):
        # weight changes made through the model reach the library here; the library then refuses pushes until reset()
        _, h = self.model._ensure_handle()
        if h.value != self._hv:
            raise RuntimeError("the model's library handle was replaced (device change); create a new SlidingScorer")
        if self._s is None:
            raise RuntimeError("SlidingScorer is closed")

    def reset(self):
        """Forget all streams (the next push is push 1 again; every patient admitted with an empty stream, so the
        per-patient masking of admit / discharge is off again) and take the model's current weights."""
        self._handle()
        with torch.cuda.device(self.device):
            capi.check(self._lib.b2cnn_slide_reset(self._s, torch.cuda.current_stream().cuda_stream), "b2cnn_slide_reset")
        self.window_index = -1

    def check_samples(self, samples: torch.Tensor) -> int:
        """Validates a push's ``[P, C, stride]`` tensor; returns its row pitch in elements."""
        if not torch.is_tensor(samples) or samples.dim() != 3:
            raise RuntimeError(f"expected samples [{self.n_patients}, {self.channels}, {self.stride}], got "
                               f"{tuple(samples.shape) if torch.is_tensor(samples) else type(samples).__name__}")
        if tuple(samples.shape) != (self.n_patients, self.channels, self.stride):
            raise RuntimeError(f"expected samples [{self.n_patients}, {self.channels}, {self.stride}], got {tuple(samples.shape)}")
        if samples.dtype != self.dtype:
            raise RuntimeError(f"expected {self.dtype} samples (the scorer's dtype), got {samples.dtype}")
        return self._pitch(samples)

    def _pitch(self, x: torch.Tensor) -> int:
        """row pitch of a validated [k, C, n] tensor in elements, 0: needs a contiguous copy"""
        if x.is_contiguous():
            return x.shape[2]
        # a row-padded view ([P, C, Sp][:, :, :S]) is read in place whatever its alignment: the library copies unaligned
        # rows into its staging rows itself, so a contiguous copy here would copy the segment twice
        if x.device.type == "cuda" and x.stride(2) == 1 and x.stride(1) >= x.shape[2] \
                and (x.shape[0] == 1 or x.stride(0) == self.channels * x.stride(1)):
            return x.stride(1)
        return 0

    def check_patients(self, patients) -> list:
        """Validates patient indices (a sequence or an integer tensor): distinct, in [0, P); returns them as a list."""
        if torch.is_tensor(patients):
            if patients.is_floating_point() or patients.is_complex() or patients.dtype == torch.bool:
                raise ValueError(f"patient indices must be integers, got {patients.dtype}")
            idx = [int(v) for v in patients.reshape(-1).tolist()]
        else:
            try:
                idx = [operator.index(v) for v in patients]
            except TypeError:
                raise ValueError("patient indices must be a sequence of integers") from None
        bad = [v for v in idx if not 0 <= v < self.n_patients]
        if bad:
            raise ValueError(f"patient indices must be in [0, {self.n_patients}), got {bad[:4]}")
        if len(set(idx)) != len(idx):
            raise ValueError("patient indices must be distinct")
        return idx

    def check_history(self, history: torch.Tensor, k: int) -> int:
        """Validates an admission's ``[k, C, H]`` history (0 <= H <= W); returns its row pitch in elements."""
        if not torch.is_tensor(history) or history.dim() != 3 or tuple(history.shape[:2]) != (k, self.channels):
            got = tuple(history.shape) if torch.is_tensor(history) else type(history).__name__
            raise ValueError(f"expected history [{k}, {self.channels}, H], got {got}")
        if history.shape[2] > self.window:
            raise ValueError(f"a history holds at most the window, {self.window} samples, got {history.shape[2]}")
        if history.dtype != self.dtype:
            raise ValueError(f"expected a {self.dtype} history (the scorer's dtype), got {history.dtype}")
        return self._pitch(history)

    @property
    def heads(self) -> tuple:
        """The models attached by ``set_heads`` (read-only)."""
        return self._heads

    @property
    def head_windows(self) -> tuple:
        """The window of each row of ``push(heads=True)`` in samples, row 0 (the scorer's own, W) first (read-only)."""
        return (self.window,) + tuple(m.arch.window for m in self._heads)

    def check_heads(self, models, shorter_windows: bool = False) -> tuple:
        """Validates ``set_heads``' argument without touching the library; returns the models as a tuple."""
        if not isinstance(shorter_windows, bool):
            raise TypeError(f"shorter_windows must be True or False, got {type(shorter_windows).__name__}")
        fields = [f for f in self.ARCH_FIELDS if not (shorter_windows and f in ("window", "l_out"))]
        return check_head_models(models, self.model.arch, self.device, "set_heads", "the scorer's model", "the scorer", fields,
                                 (lambda i, m: self._check_head_window(i, m.arch)) if shorter_windows else None)

    def _check_head_window(self, i: int, arch):
        """a head window W_k ends where the scorer's does: W_k <= W, W - W_k a multiple of the feature stride F, and
        the head's LSTM input size the feature count of W_k"""
        a = self.model.arch
        F = a.pool_s ** 2                                         # 4 on the tensor-core path's geometries too
        R = a.receptive_field
        Wk = arch.window
        if Wk > self.window:
            raise ValueError(f"heads[{i}]'s window {Wk} is longer than the scorer's, {self.window}")
        if (self.window - Wk) % F:
            raise ValueError(f"heads[{i}]'s window {Wk} is not the scorer's window {self.window} minus a multiple of the "
                             f"feature stride {F}")
        if Wk < R or arch.l_out != (Wk - R) // F + 1:
            raise ValueError(f"heads[{i}]'s l_out {arch.l_out} is not the feature count of its window {Wk}")

    def set_heads(self, models, shorter_windows: bool = False):
        """Replace the extra heads with ``models`` (a list of ``B200MyCNN``, possibly empty, at most 8): each with the
        scorer model's architecture (``age_coef`` may differ), its conv / affine weights and its device.  Takes a
        SNAPSHOT of each head's LSTM / Linear weights and ``age_coef``: a later change to a head model's weights has no
        effect until ``set_heads`` is called again.  A head attached at push n is scored from push n on, as a scorer of
        that model running since the start would score it.  Atomic: a failed call leaves the previous heads.

        ``shorter_windows=True``: a head's ``window`` (and with it its LSTM input size) may also be shorter than the
        scorer's W, as long as ``W - window`` is a multiple of the feature stride (4 on the tensor-core path,
        ``pool_s ** 2`` on the generic path).  Its window ends where the scorer's does, so its features are the last
        ones of the stored window, and its row equals what a scorer of that model at its own window and the same
        stride computes from the same pushes, NaN for a patient whose ``samples_seen`` is below its window."""
        models = self.check_heads(models, shorter_windows)
        if models and self.mode == "sequence":
            raise ValueError("a sequence-mode SlidingScorer takes no extra heads")
        self._handle()
        hs = [m._ensure_handle()[1].value for m in models]
        arr = (ctypes.c_void_p * max(len(hs), 1))(*hs)
        with torch.cuda.device(self.device):
            st = torch.cuda.current_stream().cuda_stream
            if shorter_windows:
                capi.check(self._lib.b2cnn_slide_set_heads_ex(self._s, arr, len(hs), capi.SLIDE_HEADS_SHORTER_WINDOWS, st),
                           "b2cnn_slide_set_heads_ex")
            else:
                capi.check(self._lib.b2cnn_slide_set_heads(self._s, arr, len(hs), st), "b2cnn_slide_set_heads")
        self._heads = models

    @torch.no_grad()
    def push(self, samples: torch.Tensor, age=65.0, return_prob: bool = False, heads: bool = False):
        """``samples`` [P, C, stride] of the scorer's dtype (a row-padded view is read in place, like ``predict``);
        ``age`` scalar or [P].  Returns the logits (or probabilities) of the P current windows, or ``None`` while the
        first window fills.  After ``admit`` / ``discharge``: NaN for every patient whose window is not complete
        (``samples_seen < W``; a discharged patient's samples are ignored), ``None`` when no patient's window is.
        ``heads=True``: ``Tensor[1 + K, P]`` (or ``None`` as above), row 0 exactly what ``heads=False`` returns, row i
        the scores of ``heads[i - 1]`` on the same windows and ages, NaN where row 0 is.  In sequence mode each
        patient's row is ``model(windows, age)``'s last row over its windows since admission (the class docstring
        states the identity with ``predict_record(mode="sequence")``), and its state advances only where the result
        is not NaN for an incomplete window.  With heads of shorter windows
        (``set_heads(..., shorter_windows=True)``) row i is NaN where that row's own window ``head_windows[i]`` is
        incomplete, and the result is returned as soon as any row has a complete window for one patient (row 0 may
        then be all NaN)."""
        if not isinstance(heads, bool):
            raise TypeError(f"heads must be True or False, got {type(heads).__name__}")
        pitch = self.check_samples(samples)
        self._handle()
        if samples.device != self.device:
            samples = samples.to(self.device)
            pitch = self.stride if samples.is_contiguous() else pitch
        if not pitch:
            samples, pitch = samples.contiguous(), self.stride
        if not torch.is_tensor(age):
            age = torch.tensor(float(age), dtype=torch.float32)
        age = age.detach().reshape(-1).to(device=self.device, dtype=torch.float32).contiguous()
        if age.numel() not in (1, self.n_patients):
            raise RuntimeError(f"age must be a scalar or have {self.n_patients} elements")
        em, widx = ctypes.c_int32(0), ctypes.c_int64(-1)
        shape = (1 + len(self._heads), self.n_patients) if heads else (self.n_patients,)
        out = torch.empty(shape, dtype=torch.float32, device=self.device)
        fn = "b2cnn_slide_push_heads" if heads else "b2cnn_slide_push"
        with torch.cuda.device(self.device):
            st = torch.cuda.current_stream().cuda_stream
            capi.check(getattr(self._lib, fn)(self._s, samples.data_ptr(), pitch, age.data_ptr(), age.numel(), int(return_prob),
                                              out.data_ptr(), ctypes.byref(em), ctypes.byref(widx), st), fn)
        if not em.value:
            return None
        self.window_index = int(widx.value)
        return out

    @torch.no_grad()
    def features(self) -> torch.Tensor:
        """[P, L] fp32: the stored features of the current windows in window order (== ``model.features(window)``);
        after ``admit`` / ``discharge``, NaN rows for patients without a complete window (an error when no patient has
        one)."""
        self._handle()
        feats = torch.empty(self.n_patients, self.model.arch.l_out, dtype=torch.float32, device=self.device)
        with torch.cuda.device(self.device):
            capi.check(self._lib.b2cnn_slide_features(self._s, feats.data_ptr(), torch.cuda.current_stream().cuda_stream),
                       "b2cnn_slide_features")
        return feats

    def check_lstm(self, lstm, k: int):
        """Validates ``admit``'s ``lstm`` for k patients: None, or a float tensor ``[k, 2, 2, 16]`` on a sequence-mode
        scorer."""
        if lstm is None:
            return None
        if self.mode != "sequence":
            raise ValueError("lstm is only accepted by a sequence-mode scorer: independent windows carry no LSTM state")
        check_lstm_state(lstm, k, "lstm", "patient")
        return lstm

    @torch.no_grad()
    def admit(self, patients, history=None, lstm=None):
        """Restart the streams of ``patients`` (distinct indices in [0, P)).  ``history``: None, or ``[k, C, H]`` in
        the scorer's dtype with 0 <= H <= W, the samples just before the next push's (a row-padded or unaligned view is
        read in place).  A patient's window after a later push is the last W samples of (history | pushes since
        admission); it is scored from the push at which ``samples_seen`` reaches W -- with H = W, the next one.

        ``lstm`` (sequence mode only, else ``ValueError``): ``[k, 2, 2, 16]``, the LSTM state each patient's next step
        starts from instead of zeros, in ``export()["lstm"]``'s layout (converted to float32 on the scorer's device).
        The handoff from a backtest of a stay of T >= W samples: ``admit([p], stay[:, :, T - W:T], lstm=st)`` with ``st
        = model.predict_record(stay[:, :, (T - W) % S:T], S, age, mode="sequence", return_state=True)[1]``; every later
        push then scores what ``predict_record(mode="sequence")`` gives over the stay and the pushes."""
        idx = self.check_patients(patients)
        k = len(idx)
        lstm = self.check_lstm(lstm, k)
        H, pitch = 0, 0
        if history is not None:
            pitch = self.check_history(history, k)
            H = int(history.shape[2])
        self._handle()
        if lstm is not None:
            lstm = lstm.detach().to(device=self.device, dtype=torch.float32).contiguous()
        if H:
            if history.device != self.device:
                history = history.to(self.device)
                pitch = H if history.is_contiguous() else pitch
            if not pitch:
                history, pitch = history.contiguous(), H
        arr = (ctypes.c_int32 * max(k, 1))(*idx)
        with torch.cuda.device(self.device):
            nbytes = int(self._lib.b2cnn_slide_admit_workspace_bytes(self._s, k, H))
            if nbytes < 0:
                raise RuntimeError(f"b2cnn_slide_admit_workspace_bytes: invalid arguments (k={k}, H={H})")
            ws = torch.empty(max(nbytes, 1), dtype=torch.uint8, device=self.device)
            st = torch.cuda.current_stream().cuda_stream
            if lstm is None:
                capi.check(self._lib.b2cnn_slide_admit(self._s, arr, k, history.data_ptr() if H else None, H, pitch, self._dt(),
                                                       ws.data_ptr(), nbytes, st), "b2cnn_slide_admit")
            else:
                capi.check(self._lib.b2cnn_slide_admit_ex(self._s, arr, k, history.data_ptr() if H else None, H, pitch, self._dt(),
                                                          lstm.data_ptr(), ws.data_ptr(), nbytes, st), "b2cnn_slide_admit_ex")

    def discharge(self, patients):
        """Stop scoring ``patients``: their scores and features are NaN, their samples in later pushes ignored, until
        they are admitted again."""
        idx = self.check_patients(patients)
        self._handle()
        arr = (ctypes.c_int32 * max(len(idx), 1))(*idx)
        with torch.cuda.device(self.device):
            capi.check(self._lib.b2cnn_slide_discharge(self._s, arr, len(idx), torch.cuda.current_stream().cuda_stream),
                       "b2cnn_slide_discharge")

    @property
    def samples_seen(self) -> torch.Tensor:
        """int64 [P] on the device: each patient's stream samples since its admission (since ``reset()`` for patients
        never admitted), -1 for a discharged patient.  A score is defined once it is >= W."""
        self._handle()
        out = torch.empty(self.n_patients, dtype=torch.int64, device=self.device)
        with torch.cuda.device(self.device):
            capi.check(self._lib.b2cnn_slide_samples_seen(self._s, out.data_ptr(), torch.cuda.current_stream().cuda_stream),
                       "b2cnn_slide_samples_seen")
        return out

    @torch.no_grad()
    def export(self, patients) -> dict:
        """The state of ``patients`` (distinct indices in [0, P)), row j for ``patients[j]``, as plain tensors and ints
        ``torch.save`` can write: ``features`` [k, L] fp32 (each current window in window order, raw: a patient without
        a complete window has no NaN mask here), ``tail`` [k, C, T] fp32 (the stream's last T samples per channel),
        both on the scorer's device, ``seen`` [k] CPU int64 (``samples_seen``), and the header fields (path, dtype,
        C, W, L, feature stride F, T and a digest of the conv weights).  Changes nothing in the scorer.
        ``window_index`` is not part of it: it counts this scorer's own pushes.  A sequence-mode scorer adds ``lstm``
        [k, 2, 2, 16] fp32 on its device, each patient's LSTM state as [layer][h | c][unit]."""
        idx = self.check_patients(patients)
        k = len(idx)
        self._handle()
        f = self._state_fields
        feats = torch.empty(k, f["lstm_input"], dtype=torch.float32, device=self.device)
        tail = torch.empty(k, self.channels, f["tail_len"], dtype=torch.float32, device=self.device)
        seen = torch.empty(k, dtype=torch.int64)
        hdr = capi.SlideStateHeader()
        arr = (ctypes.c_int32 * max(k, 1))(*idx)
        with torch.cuda.device(self.device):
            nbytes = int(self._lib.b2cnn_slide_state_workspace_bytes(self._s, k))
            ws = torch.empty(max(nbytes, 1), dtype=torch.uint8, device=self.device)
            st = torch.cuda.current_stream().cuda_stream
            if self.mode == "sequence":
                lstm = torch.empty((k,) + self.LSTM_STATE, dtype=torch.float32, device=self.device)
                capi.check(self._lib.b2cnn_slide_export_ex(self._s, arr, k, feats.data_ptr(), tail.data_ptr(), seen.data_ptr(),
                                                           lstm.data_ptr(), ctypes.byref(hdr), ws.data_ptr(), nbytes, st),
                           "b2cnn_slide_export_ex")
            else:
                capi.check(self._lib.b2cnn_slide_export(self._s, arr, k, feats.data_ptr(), tail.data_ptr(), seen.data_ptr(), ctypes.byref(hdr),
                                                        ws.data_ptr(), nbytes, st), "b2cnn_slide_export")
        state = {"features": feats, "tail": tail, "seen": seen}
        if self.mode == "sequence":
            state["lstm"] = lstm
        state.update({n: int(getattr(hdr, n)) for n in self.STATE_HEADER})
        return state

    def check_state(self, state, k: int):
        """Validates a state of k patients (``export``'s dict) against this scorer; returns (features, tail, seen).  The
        state holds ``lstm`` exactly when the scorer is in sequence mode."""
        if not isinstance(state, dict):
            raise ValueError(f"expected the dict of SlidingScorer.export(), got {type(state).__name__}")
        if ("lstm" in state) != (self.mode == "sequence"):
            raise ValueError(f"the state was exported in another mode than this scorer's ({self.mode}): it "
                             + ("lacks" if self.mode == "sequence" else "holds") + " 'lstm'")
        missing = [n for n in ("features", "tail", "seen") + self.STATE_HEADER if n not in state]
        if missing:
            raise ValueError(f"the state lacks {missing}")
        for n in self.STATE_HEADER:
            try:
                operator.index(state[n])
            except TypeError:
                raise ValueError(f"state[{n!r}] must be an integer, got {type(state[n]).__name__}") from None
        if not 0 <= int(state["frontend_digest"]) < 1 << 64:
            raise ValueError("state['frontend_digest'] must be a 64-bit unsigned integer")
        bad = {n: (int(state[n]), v) for n, v in self._state_fields.items() if int(state[n]) != v}
        if bad:
            raise ValueError("the state does not fit this scorer (field: (state, scorer)): "
                             + ", ".join(f"{n}: {a}" for n, a in bad.items()))
        L, T = self._state_fields["lstm_input"], self._state_fields["tail_len"]
        want = {"features": ((k, L), torch.float32), "tail": ((k, self.channels, T), torch.float32), "seen": ((k,), torch.int64)}
        if self.mode == "sequence":
            want["lstm"] = ((k,) + self.LSTM_STATE, torch.float32)
        for n, (shape, dtype) in want.items():
            t = state[n]
            if not torch.is_tensor(t) or tuple(t.shape) != shape or t.dtype != dtype:
                got = (tuple(t.shape), t.dtype) if torch.is_tensor(t) else type(t).__name__
                raise ValueError(f"state[{n!r}]: expected {dtype} {list(shape)}, got {got}")
        seen = state["seen"].cpu()
        if k and int(seen.min()) < -1:
            raise ValueError("state['seen'] holds a count below -1")
        return state["features"], state["tail"], seen

    @torch.no_grad()
    def restore(self, patients, state: dict):
        """Put ``export``'s ``state`` into the streams of ``patients`` (row j into ``patients[j]``; any slots, any P and
        stride, on any device: the tensors are moved to this scorer's).  As ``admit`` with the full exported window:
        a patient with ``samples_seen >= W`` is in ``features()`` at once and scored from the next push on, exactly as
        the exporting scorer would have scored it on the same samples; one exported discharged stays discharged.  The
        state must come from a scorer of the same path, dtype, C, W and conv weights (the LSTM and head weights may
        differ: change them, ``reset()``, then restore).  A sequence-mode scorer takes only a sequence-mode state (with
        ``lstm``), from which the patients' LSTM continues; an independent one only an independent state.  Errors
        leave the scorer unchanged."""
        idx = self.check_patients(patients)
        k = len(idx)
        feats, tail, seen = self.check_state(state, k)
        lstm = state.get("lstm")
        self._handle()
        feats = feats.to(self.device).contiguous()
        tail = tail.to(self.device).contiguous()
        seen = seen.contiguous()
        hdr = capi.SlideStateHeader(**{n: int(state[n]) for n in self.STATE_HEADER})
        arr = (ctypes.c_int32 * max(k, 1))(*idx)
        with torch.cuda.device(self.device):
            nbytes = int(self._lib.b2cnn_slide_state_workspace_bytes(self._s, k))
            ws = torch.empty(max(nbytes, 1), dtype=torch.uint8, device=self.device)
            st = torch.cuda.current_stream().cuda_stream
            if lstm is not None:
                lstm = lstm.to(self.device).contiguous()
                capi.check(self._lib.b2cnn_slide_import_ex(self._s, arr, k, ctypes.byref(hdr), feats.data_ptr(), tail.data_ptr(),
                                                           seen.data_ptr(), lstm.data_ptr(), ws.data_ptr(), nbytes, st),
                           "b2cnn_slide_import_ex")
            else:
                capi.check(self._lib.b2cnn_slide_import(self._s, arr, k, ctypes.byref(hdr), feats.data_ptr(), tail.data_ptr(), seen.data_ptr(),
                                                        ws.data_ptr(), nbytes, st), "b2cnn_slide_import")
