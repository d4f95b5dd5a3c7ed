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
"""
from __future__ import annotations

import ctypes
import operator

import torch

from . import capi


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
    the model and the generic one otherwise.  ``scorer.path`` tells which one runs."""

    PATHS = {"tensorcore": capi.PATH_TENSORCORE, "generic": capi.PATH_GENERIC, "auto": capi.PATH_AUTO}

    def __init__(self, model, n_patients: int, stride: int, dtype=torch.bfloat16, path: str = "tensorcore"):
        if dtype not in (torch.bfloat16, torch.float32):
            raise ValueError("dtype must be torch.bfloat16 or torch.float32")
        if path not in self.PATHS:
            raise ValueError(f"path must be one of {sorted(self.PATHS)}, got {path!r}")
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
            if path == "tensorcore":
                capi.check(self._lib.b2cnn_slide_create(h, n_patients, stride, self._dt(), ctypes.byref(s)), "b2cnn_slide_create")
            else:
                capi.check(self._lib.b2cnn_slide_create_path(h, n_patients, stride, self._dt(), self.PATHS[path], ctypes.byref(s)),
                           "b2cnn_slide_create_path")
        self._s = s
        self.path = "generic" if self._lib.b2cnn_slide_path(s) == capi.PATH_GENERIC else "tensorcore"
        self.window_index = -1

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

    @torch.no_grad()
    def push(self, samples: torch.Tensor, age=65.0, return_prob: bool = False):
        """``samples`` [P, C, stride] of the scorer's dtype (a row-padded view is read in place, like ``predict``);
        ``age`` scalar or [P].  Returns the logits (or probabilities) of the P current windows, or ``None`` while the
        first window fills.  After ``admit`` / ``discharge``: NaN for every patient whose window is not complete
        (``samples_seen < W``; a discharged patient's samples are ignored), ``None`` when no patient's window is."""
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
        out = torch.empty(self.n_patients, dtype=torch.float32, device=self.device)
        with torch.cuda.device(self.device):
            st = torch.cuda.current_stream().cuda_stream
            capi.check(self._lib.b2cnn_slide_push(self._s, samples.data_ptr(), pitch, age.data_ptr(), age.numel(), int(return_prob),
                                                  out.data_ptr(), ctypes.byref(em), ctypes.byref(widx), st), "b2cnn_slide_push")
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

    @torch.no_grad()
    def admit(self, patients, history=None):
        """Restart the streams of ``patients`` (distinct indices in [0, P)).  ``history``: None, or ``[k, C, H]`` in
        the scorer's dtype with 0 <= H <= W, the samples just before the next push's (a row-padded or unaligned view is
        read in place).  A patient's window after a later push is the last W samples of (history | pushes since
        admission); it is scored from the push at which ``samples_seen`` reaches W -- with H = W, the next one."""
        idx = self.check_patients(patients)
        k = len(idx)
        H, pitch = 0, 0
        if history is not None:
            pitch = self.check_history(history, k)
            H = int(history.shape[2])
        self._handle()
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
            capi.check(self._lib.b2cnn_slide_admit(self._s, arr, k, history.data_ptr() if H else None, H, pitch, self._dt(),
                                                   ws.data_ptr(), nbytes, st), "b2cnn_slide_admit")

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
