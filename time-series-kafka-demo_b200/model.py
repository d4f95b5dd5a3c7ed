"""``B200MyCNN`` -- the Python face of the drop-in.

Mirrors the reference's operator interface for the hot path:

* construction / loading:  ``model = torch.load(path); model.eval()`` (bin/predictStream.py:36-37)
  -> ``B200MyCNN.from_reference(load_reference_checkpoint(path)).eval()``; ``state_dict()`` /
  ``load_state_dict()`` use the reference's key names and shapes (bin/models.py:10-20), the
  never-used ``out1`` / ``out2`` / ``age_fn`` included as inert parameters;
* the call:  ``output = model(x, age)`` (bin/predictStream.py:157; utils.py:204,249,682) with the
  reference's semantics -- for B > 1 the LSTM scans the batch axis (bin/models.py:29-30);
* ``predict(windows, age)``: the batched dispatch predictStream's per-row loop turns into --
  every row an independent window from the zero LSTM state (what looping ``model(x[i:i+1])`` gives).

The sub-modules (``conv1``, ``lstm`` ...) are parameter containers only; the arithmetic runs in
libb2cnn.so (hand-written sm_90a kernels) through ctypes.  No CUDA device -> RuntimeError.
"""
from __future__ import annotations

import ctypes
import operator
from typing import Optional

import torch
import torch.nn as nn

from . import capi
from .arch import BLOB_KEYS, ArchConfig, arch_from_state_dict
from .checkpoint import arch_of_module

_PATHS = {"auto": capi.PATH_AUTO, "generic": capi.PATH_GENERIC, "tensorcore": capi.PATH_TENSORCORE}
_PATH_NAMES = {v: k for k, v in _PATHS.items()}
_PATH_NAMES[3] = "stream"            # B2CNN_PATH_STREAM: fp32 windows through the streaming kernel


class B200MyCNN(nn.Module):
    def __init__(self, arch: ArchConfig = ArchConfig(), has_out12: bool = True,
                 device: Optional[torch.device | str] = None, path: str = "auto", tc_splits: int = 3):
        super().__init__()
        self.arch = arch
        self.MAGICNUM = arch.l_out                                         # bin/models.py:8
        if arch.l1 < arch.pool_k or arch.l2 < arch.pool_k or arch.l_out < 1:
            raise RuntimeError(f"window={arch.window} is too short for this conv/pool stack")
        # same construction order as bin/models.py:10-20 (=> same default-init RNG stream)
        self.conv1 = nn.Conv1d(arch.in_channels, arch.c_mid, arch.k1)
        self.conv2 = nn.Conv1d(arch.c_mid, 1, arch.k2)
        self.pool = nn.MaxPool1d(arch.pool_k, arch.pool_s)
        if has_out12:
            self.out1 = nn.Linear(567, 1)
        self.dropout = nn.Dropout(0.1)
        self.lstm = nn.LSTM(arch.l_out, arch.hidden, arch.layers)
        self.out = nn.Linear(arch.hidden, 1)
        if has_out12:
            self.out2 = nn.Linear(arch.hidden, 1)
        self.age_fn = nn.Linear(1, 1)
        if arch.affine:   # folded eval-BatchNorm: y = conv(x) * scale + shift, per channel
            self.affine1_scale = nn.Parameter(torch.ones(arch.c_mid))
            self.affine1_shift = nn.Parameter(torch.zeros(arch.c_mid))
            self.affine2_scale = nn.Parameter(torch.ones(1))
            self.affine2_shift = nn.Parameter(torch.zeros(1))
        self.requires_grad_(False)
        self.training = False              # inference only (predictStream.py:37 calls eval())
        self.batch_mode = "sequence"       # semantics of forward() for B > 1 (== the reference)
        self._path = path
        self._tc_splits = tc_splits
        self._handle = None
        self._handle_device = None
        self._synced_version = None
        self._ws = None
        if device is not None:
            self.to(device)

    # ------------------------------------------------------------------ construction
    @classmethod
    def from_reference(cls, ref, window: int = 120, age_coef: Optional[float] = None, **kw) -> "B200MyCNN":
        """``ref``: the object ``torch.load`` returns for a reference checkpoint (a full module,
        see checkpoint.py) or a plain state_dict."""
        if isinstance(ref, nn.Module):
            arch = arch_of_module(ref, window=window, age_coef=age_coef)
            sd = ref.state_dict()
        else:
            sd = dict(ref)
            arch = arch_from_state_dict(sd, window=window, age_coef=age_coef)
        m = cls(arch, has_out12=("out1.weight" in sd), **kw)
        m.load_state_dict(sd)
        return m

    def train(self, mode: bool = True):
        if mode:
            raise NotImplementedError("B200MyCNN.forward is the inference path (no dropout); the reference's training-loop "
                                      "body (bin/utils.py:200-208) is B200Trainer(model).step(x, age, target)")
        return super().train(False)

    # ------------------------------------------------------------------ library plumbing
    def _device(self) -> torch.device:
        return self.conv1.weight.device

    def _weights_version(self):
        # in-place edits (p.copy_(), p.mul_(), p.data.fill_() ...) bump Tensor._version; swapping a
        # parameter object or moving the module changes the id / device entries
        ps = self.__dict__.get("_vparams")
        if ps is None:
            ps = self.__dict__["_vparams"] = tuple(self.parameters())
        return tuple(p._version for p in ps) + (id(ps[0]), ps[0].device)

    def packed_weights(self) -> torch.Tensor:
        """The blob b2cnn_set_weights() takes (include/b2cnn.h), on the parameters' device."""
        sd = self.state_dict()
        parts = [sd[k].detach().reshape(-1).float() for k in BLOB_KEYS]
        if self.arch.affine:
            parts += [self.affine1_scale.detach().float(), self.affine1_shift.detach().float(),
                      self.affine2_scale.detach().float(), self.affine2_shift.detach().float()]
        return torch.cat(parts).contiguous()

    # Weight changes reach the library lazily.  load_state_dict() and .to()/.cuda() mark the
    # model dirty; after in-place edits of a parameter call sync_weights() (or any of the two).
    def load_state_dict(self, *a, **k):
        r = super().load_state_dict(*a, **k)
        self.__dict__["_dirty"] = True
        return r

    def _apply(self, fn, *a, **k):
        r = super()._apply(fn, *a, **k)
        self.__dict__["_dirty"] = True
        self.__dict__["_vparams"] = None          # .to() may replace the Parameter objects
        return r

    # The native handle, the CDLL and the workspace tensor never travel with a copy or a pickle
    # (the reference saves whole-module pickles, bin/explore_torch.ipynb:3234): a restored / copied
    # module rebuilds its own handle lazily on its first forward.
    _NATIVE_STATE = ("_handle", "_handle_device", "_lib", "_ws", "_ws_need", "_synced_version", "_vparams", "_dirty")

    def __getstate__(self):
        st = dict(self.__dict__)
        for k in self._NATIVE_STATE:
            st.pop(k, None)
        return st

    def __setstate__(self, st):
        self.__dict__.update(st)
        self.__dict__.update(_handle=None, _handle_device=None, _ws=None, _synced_version=None, _dirty=True)

    def __deepcopy__(self, memo):
        import copy
        new = self.__class__.__new__(self.__class__)
        memo[id(self)] = new
        new.__setstate__(copy.deepcopy(self.__getstate__(), memo))
        return new

    def sync_weights(self):
        self.__dict__["_dirty"] = True
        self._ensure_handle()

    def _ensure_handle(self):
        if not self.__dict__.get("_dirty", True) and self._handle is not None \
                and self._synced_version == self._weights_version():
            return self._lib, self._handle                      # fast path of the hot call
        dev = self._device()
        if dev.type != "cuda":
            if not torch.cuda.is_available():
                raise RuntimeError("B200MyCNN needs a CUDA device: the forward pass is sm_100a CUDA "
                                   "and there is no CPU fallback")
            self.to("cuda")
            dev = self._device()
        lib = capi.load_library()
        self.__dict__["_lib"] = lib
        if self._handle is None or self._handle_device != dev:
            self._release()
            cfg = capi.make_config(self.arch, dev.index if dev.index is not None else torch.cuda.current_device())
            h = ctypes.c_void_p()
            capi.check(lib.b2cnn_create(ctypes.byref(cfg), ctypes.byref(h)), "b2cnn_create")
            self._handle, self._handle_device = h, dev
            capi.check(lib.b2cnn_set_option(h, b"tc_splits", int(self._tc_splits)), "b2cnn_set_option")
            capi.check(lib.b2cnn_set_option(h, b"path", _PATHS[self._path]), "b2cnn_set_option")
            self._synced_version = None
            self.__dict__["_ws_need"] = {}
        if self._synced_version != self._weights_version():
            blob = self.packed_weights()
            with torch.cuda.device(dev):
                st = torch.cuda.current_stream().cuda_stream
                capi.check(lib.b2cnn_set_weights(self._handle, blob.data_ptr(), blob.numel(), 1, st),
                           "b2cnn_set_weights")
                torch.cuda.current_stream().synchronize()
            self._synced_version = self._weights_version()
        self.__dict__["_dirty"] = False
        return lib, self._handle

    def _release(self):
        h = self.__dict__.get("_handle")
        if h is not None:
            self.__dict__["_handle"] = None      # plain dict write: safe during interpreter shutdown
            try:
                capi.load_library().b2cnn_destroy(h)
            except Exception:
                pass

    def __del__(self):
        try:
            self._release()
        except Exception:
            pass

    def set_path(self, path: str):
        """'auto' | 'generic' (exact fp32 CUDA cores) | 'tensorcore' (wgmma conv1)."""
        self._path = path
        self.__dict__["_ws_need"] = {}                     # the scratch size depends on the path a call takes
        if self._handle is not None:
            capi.check(capi.load_library().b2cnn_set_option(self._handle, b"path", _PATHS[path]), "b2cnn_set_option")

    def set_option(self, key: str, value: int):
        """Library options (include/b2cnn.h): e.g. "tc_fused" = 0 keeps the tensor-core front
        end and the projection as separate kernels."""
        lib, h = self._ensure_handle()
        capi.check(lib.b2cnn_set_option(h, key.encode(), int(value)), "b2cnn_set_option")
        self.__dict__["_ws_need"] = {}

    def set_profile(self, on: bool = True):
        """Record CUDA events around the stages of every forward (bench.py's roofline figure)."""
        lib, h = self._ensure_handle()
        capi.check(lib.b2cnn_set_option(h, b"profile", int(on)), "b2cnn_set_option")

    def last_stage_ms(self, stage: int = 0) -> float:
        """Device time of stage 0 (front end, the dominant kernel) / 1 (projection + head)."""
        return float(capi.load_library().b2cnn_last_stage_ms(self._handle, stage)) if self._handle else -1.0

    @property
    def gpu_launches(self) -> int:
        return int(capi.load_library().b2cnn_last_launch_count(self._handle)) if self._handle else 0

    @property
    def last_path(self) -> str:
        if not self._handle:
            return "none"
        return _PATH_NAMES.get(int(capi.load_library().b2cnn_last_path(self._handle)), "none")

    def _workspace(self, lib, h, B: int, mode: int, dtype: int, dev) -> torch.Tensor:
        cache = self.__dict__.setdefault("_ws_need", {})
        need = cache.get((B, mode, dtype))
        if need is None:
            need = cache[(B, mode, dtype)] = int(lib.b2cnn_workspace_bytes_for(h, B, mode, dtype))
        ws = self._ws
        if ws is None or ws.numel() < need or ws.device != dev:
            ws = self._ws = torch.empty(need, dtype=torch.uint8, device=dev)
        return ws

    # ------------------------------------------------------------------ the hot call
    def _check_x(self, x: torch.Tensor) -> torch.Tensor:
        if x.dim() != 3 or x.shape[1] != self.arch.in_channels or x.shape[2] != self.arch.window:
            raise RuntimeError(f"expected input [B, {self.arch.in_channels}, {self.arch.window}], got {tuple(x.shape)}")
        if x.dtype not in (torch.float32, torch.bfloat16):
            x = x.float()                      # predictStream.py:155 casts float64 -> float32
        return x if self._row_pitch(x) else x.contiguous()

    def _row_pitch(self, x: torch.Tensor) -> int:
        """Row pitch (elements) of a CUDA tensor whose rows are padded by its producer -- a [B, C, W] view of a
        [B, C, Wp] buffer (see :meth:`empty_windows`) -- or 0 when the tensor has to be taken as contiguous."""
        if x.device.type != "cuda" or x.dim() != 3 or x.stride(2) != 1 or x.is_contiguous():
            return 0
        pitch = x.stride(1)
        unit = 16 // x.element_size()
        if pitch < x.shape[2] or pitch % unit or (x.shape[0] > 1 and x.stride(0) != x.shape[1] * pitch) \
                or (x.data_ptr() % 16):
            return 0
        return pitch

    def empty_windows(self, B: int, dtype=torch.bfloat16, device=None) -> torch.Tensor:
        """A ``[B, C, W]`` window batch whose rows start on 16-byte boundaries whatever W is: a view of a
        ``[B, C, Wp]`` buffer, ``Wp`` = W rounded up to 8 bf16 / 4 fp32 samples.  A producer that fills THIS tensor
        (instead of a contiguous one) lets the TMA kernels stream windows with W % 8 != 0 (7500, 37500 ...)
        straight from it -- no re-pitching copy; the pad is never read."""
        unit = 16 // torch.empty((), dtype=dtype).element_size()
        W = self.arch.window
        Wp = (W + unit - 1) // unit * unit
        dev = device if device is not None else self._device()
        return torch.empty(B, self.arch.in_channels, Wp, dtype=dtype, device=dev)[:, :, :W]

    def _run(self, x: torch.Tensor, age: torch.Tensor, mode: int, sigmoid: bool) -> torch.Tensor:
        lib, h = self._ensure_handle()
        dev = self._handle_device
        x = self._check_x(x)
        B = x.shape[0]
        if not (age.dtype == torch.float32 and age.dim() == 1 and age.is_contiguous()):
            age = age.detach().reshape(-1).float().contiguous()
        n_age = age.numel()
        if n_age != 1 and n_age != B:
            raise RuntimeError(f"age must have 1 or {B} elements, got {n_age}")
        dtype = capi.DTYPE_BF16 if x.dtype == torch.bfloat16 else capi.DTYPE_F32
        if x.device.type == "cpu":
            # host buffers in, host buffers out: chunked H2D inside the library
            out = torch.empty(B, dtype=torch.float32)
            age_h = age.cpu()
            with torch.cuda.device(dev):
                capi.check(lib.b2cnn_forward_host(h, x.data_ptr(), dtype, B, age_h.data_ptr(), n_age,
                                                  mode, int(sigmoid), out.data_ptr()), "b2cnn_forward_host")
            return out
        if x.device != dev:
            x = x.to(dev)
        if age.device != dev:
            age = age.to(dev)
        out = torch.empty(B, dtype=torch.float32, device=dev)
        ws = self._workspace(lib, h, B, mode, dtype, dev)
        pitch = 0 if x.is_contiguous() else self._row_pitch(x)
        if pitch:                                               # rows padded by the producer: no re-pitching copy
            with torch.cuda.device(dev):
                rc = lib.b2cnn_forward_pitched(h, x.data_ptr(), dtype, B, pitch, age.data_ptr(), n_age, mode, int(sigmoid),
                                               out.data_ptr(), ws.data_ptr(), ws.numel(), torch.cuda.current_stream().cuda_stream)
        elif torch.cuda.current_device() == dev.index:          # the usual case: no device switch needed
            rc = lib.b2cnn_forward(h, x.data_ptr(), dtype, B, age.data_ptr(), n_age, mode, int(sigmoid),
                                   out.data_ptr(), ws.data_ptr(), ws.numel(), torch.cuda.current_stream().cuda_stream)
        else:
            with torch.cuda.device(dev):
                rc = lib.b2cnn_forward(h, x.data_ptr(), dtype, B, age.data_ptr(), n_age, mode, int(sigmoid),
                                       out.data_ptr(), ws.data_ptr(), ws.numel(), torch.cuda.current_stream().cuda_stream)
        if rc:
            capi.check(rc, "b2cnn_forward")
        return out

    def _seq_args(self, x: torch.Tensor, age, seq_lengths):
        """Validates a many-sequence call before anything runs: (x, age as 1 or B float32 values, the host length array)."""
        x = self._check_x(x)
        B = x.shape[0]
        age = (age if torch.is_tensor(age) else torch.tensor(age, dtype=torch.float32)).detach()
        if age.dim() > 1 or age.numel() not in (1, B):
            raise ValueError(f"with seq_lengths, age must have 1 or {B} elements (one per window), got shape {tuple(age.shape)}")
        return x, age.reshape(-1).float().contiguous(), capi.seq_lengths_array(seq_lengths, B)

    def _run_seq(self, x: torch.Tensor, age, seq_lengths, sigmoid: bool) -> torch.Tensor:
        """Sequence mode over the consecutive sequences ``seq_lengths`` of the batch (b2cnn_forward_seq)."""
        x, age, lens = self._seq_args(x, age, seq_lengths)
        lib, h = self._ensure_handle()
        dev = self._handle_device
        x, age = x.to(dev), age.to(dev)
        B = x.shape[0]
        pitch = 0 if x.is_contiguous() else self._row_pitch(x)
        if not x.is_contiguous() and not pitch:
            x = x.contiguous()
        dtype = capi.DTYPE_BF16 if x.dtype == torch.bfloat16 else capi.DTYPE_F32
        out = torch.empty(B, dtype=torch.float32, device=dev)
        with torch.cuda.device(dev):
            need = int(lib.b2cnn_workspace_bytes_seq(h, B, lens, len(lens)))
            if need < 0:
                capi.check(capi.EINVAL, "b2cnn_workspace_bytes_seq")
            ws = self._ws
            if ws is None or ws.numel() < need or ws.device != dev:
                ws = self._ws = torch.empty(need, dtype=torch.uint8, device=dev)
            capi.check(lib.b2cnn_forward_seq(h, x.data_ptr(), dtype, B, pitch or self.arch.window, age.data_ptr(), age.numel(), lens,
                                             len(lens), int(sigmoid), out.data_ptr(), ws.data_ptr(), ws.numel(),
                                             torch.cuda.current_stream().cuda_stream), "b2cnn_forward_seq")
        return out

    @torch.no_grad()
    def forward(self, x: torch.Tensor, age: torch.Tensor, seq_lengths=None) -> torch.Tensor:
        """``model(x, age)`` with the reference's semantics (bin/models.py:22-36).

        ``seq_lengths`` [n_0, ..., n_{N-1}] (a list, tuple or integer tensor; each >= 1, adding up to B): the batch is N
        consecutive sequences, each scanned from the zero LSTM state -- ``torch.cat([model(x[o:o+n], age[o:o+n]) for
        ...])`` in one call.  Sequence mode only (``batch_mode == "sequence"``); age then has 1 or B elements."""
        if seq_lengths is not None:
            if self.batch_mode != "sequence":
                raise ValueError("seq_lengths needs batch_mode == 'sequence'")
            return self._run_seq(x, age, seq_lengths, False)
        mode = capi.MODE_SEQUENCE if (self.batch_mode == "sequence" and x.shape[0] > 1) else capi.MODE_INDEPENDENT
        B = x.shape[0]
        if age.dim() == 1 and age.numel() in (1, B):
            return self._run(x, age, mode, False)
        # Unusual age shapes (e.g. utils.run_model's (1, n), bin/utils.py:681): reproduce the
        # reference's broadcasting of `x * relu(age.unsqueeze(1)*coef + 1)` around the kernel
        # result computed with a unit age factor (age = 0 -> relu(0*coef + 1) == 1 exactly).
        y = self._run(x, torch.zeros(1), mode, False)
        age = age.to(y.device).float()
        age_scale = torch.relu(age.unsqueeze(1) * self.arch.age_coef + 1)
        return (y.unsqueeze(1) * age_scale).squeeze(1)

    @torch.no_grad()
    def predict(self, window_tensor: torch.Tensor, age=None, mode: str = "independent", seq_lengths=None,
                return_prob: bool = False) -> torch.Tensor:
        """Batched dispatch for predictStream's per-row loop (bin/predictStream.py:70-162):
        ``window_tensor`` [B, C, W]; ``age`` scalar / [B] (default 65.0, predictStream.py:149);
        returns logits [B] or, with ``return_prob``, ``sigmoid(logit)`` (predictStream.py:160).

        ``mode="sequence", seq_lengths=[n_0, ...]``: the batch is consecutive sequences (each >= 1 window, adding up to
        B), each scored like ``predict(x_s, age_s, mode="sequence")`` in one call (see :meth:`forward`)."""
        if window_tensor.dim() == 2:
            window_tensor = window_tensor.unsqueeze(0)
        B = window_tensor.shape[0]
        if seq_lengths is not None:
            if mode != "sequence":
                raise ValueError("seq_lengths is only accepted with mode='sequence'")
            return self._run_seq(window_tensor, 65.0 if age is None else age, seq_lengths, return_prob)
        if age is None:
            age = 65.0
        if not torch.is_tensor(age):
            age = torch.tensor(age, dtype=torch.float32)
        age = age.reshape(-1)
        m = capi.MODE_INDEPENDENT if mode == "independent" else capi.MODE_SEQUENCE
        if mode not in ("independent", "sequence"):
            raise ValueError("mode must be 'independent' or 'sequence'")
        if B == 0 and mode == "independent":
            # the per-row loop over zero rows scores nothing (bin/predictStream.py:70); model(x, a) itself raises on an
            # empty batch (nn.LSTM rejects a zero-length sequence) and so does forward() / mode="sequence"
            self._check_x(window_tensor)
            return torch.empty(0, dtype=torch.float32, device=window_tensor.device)
        if age.numel() not in (1, B):
            raise RuntimeError(f"age must be a scalar or have {B} elements")
        return self._run(window_tensor, age, m, return_prob)

    def check_record_args(self, records, stride, age=None, path: str = "auto", mode: str = "independent"):
        """Validates ``predict_record``'s arguments without touching the library; returns ``(stride, age)`` with age a
        float32 vector of 1 or B elements."""
        if not isinstance(mode, str) or mode not in ("independent", "sequence"):
            raise ValueError(f"mode must be 'independent' or 'sequence', got {mode!r}")
        C = self.arch.in_channels
        if not torch.is_tensor(records) or records.dim() != 3 or records.shape[1] != C:
            got = tuple(records.shape) if torch.is_tensor(records) else type(records).__name__
            raise ValueError(f"expected records [B, {C}, N], got {got}")
        if records.dtype not in (torch.float32, torch.bfloat16):
            raise ValueError(f"records must be float32 or bfloat16, got {records.dtype}")
        if records.shape[0] < 1:
            raise ValueError("records must hold at least one recording")
        if path not in _PATHS:
            raise ValueError(f"path must be one of {sorted(_PATHS)}, got {path!r}")
        if isinstance(stride, bool) or not isinstance(stride, int):
            try:
                stride = operator.index(stride)
            except TypeError:
                raise ValueError(f"stride must be an integer, got {type(stride).__name__}") from None
        F = 4 if path == "tensorcore" else self.arch.pool_s ** 2          # the feature stride in samples
        if stride < 1 or stride % F:
            raise ValueError(f"stride must be a positive multiple of the feature stride {F}, got {stride}")
        if age is None:
            age = 65.0
        age = (age if torch.is_tensor(age) else torch.tensor(age, dtype=torch.float32)).detach().reshape(-1).float()
        if age.numel() not in (1, records.shape[0]):
            raise ValueError(f"age must be a scalar or have {records.shape[0]} elements (one per recording), got {age.numel()}")
        return stride, age

    @torch.no_grad()
    def predict_record(self, records: torch.Tensor, stride: int, age=None, return_prob: bool = False,
                       path: str = "auto", mode: str = "independent") -> torch.Tensor:
        """Every window of whole recordings in one call: ``records`` ``[B, C, N]`` (float32 or bfloat16; contiguous or
        a row-padded view), windows of the model's W samples starting every ``stride`` samples.  Returns ``[B, n_w]``,
        ``n_w = (N - W) // stride + 1`` (0 when N < W): element ``[b, w]`` is ``predict(records[b, :, w*stride :
        w*stride + W], age[b])`` (the probability with ``return_prob``).  ``age``: a scalar or one per recording
        (default 65.0).  Each window feature is computed once, however many windows share it.

        ``mode="sequence"``: row ``b`` is instead ``model(windows_b, age_b)``, ``windows_b`` the recording's ``n_w``
        windows in order -- the LSTM carried across one recording's windows, as ``bin/utils.py``'s ``run_model`` scores
        a recording; the state starts at zero for every recording and never passes from one to the next.  The scan is
        causal (the first k outputs do not depend on later windows), and a NaN window makes its own and every later
        output of its recording NaN.

        ``path``: ``"tensorcore"`` (the models a tensor-core ``SlidingScorer`` holds), ``"generic"`` (every model; its
        logits are bit-identical to ``predict()`` with ``path="generic"`` and ``small_kernel=0``, per recording with
        ``mode="sequence"`` in sequence mode) or ``"auto"``.  ``stride`` must be a multiple of the feature stride
        ``pool_s ** 2`` (4 on the tensor-core path); it may exceed W.  ``bin/utils.py``'s ``create_batch`` drops the
        last window when ``(N - W) % stride == 0``: ``out[:, :-1]`` is its set then, in either mode."""
        stride, age = self.check_record_args(records, stride, age, path, mode)
        B, N, W = records.shape[0], records.shape[2], self.arch.window
        lib, h = self._ensure_handle()
        dev = self._handle_device
        n_w = (N - W) // stride + 1 if N >= W else 0
        if n_w == 0:
            return torch.empty(B, 0, dtype=torch.float32, device=dev)
        if records.device != dev:
            records = records.to(dev)
        age = age.to(dev).contiguous()
        C = self.arch.in_channels
        if records.is_contiguous():
            pitch = N
        elif records.stride(2) == 1 and records.stride(1) >= N and (B == 1 or records.stride(0) == C * records.stride(1)):
            pitch = records.stride(1)                            # a row-padded view, read in place
        else:
            records, pitch = records.contiguous(), N
        dtype = capi.DTYPE_BF16 if records.dtype == torch.bfloat16 else capi.DTYPE_F32
        out = torch.empty(B, n_w, dtype=torch.float32, device=dev)
        m = capi.MODE_SEQUENCE if mode == "sequence" else capi.MODE_INDEPENDENT
        with torch.cuda.device(dev):
            need = int(lib.b2cnn_record_workspace_bytes_ex(h, B, N, pitch, stride, dtype, _PATHS[path], m))
            if need < 0:
                raise RuntimeError(capi.last_error())
            ws = torch.empty(max(need, 256), dtype=torch.uint8, device=dev)
            capi.check(lib.b2cnn_score_record_ex(h, records.data_ptr(), dtype, B, N, pitch, stride, _PATHS[path], m, age.data_ptr(),
                                                 age.numel(), int(return_prob), out.data_ptr(), ws.data_ptr(), ws.numel(),
                                                 torch.cuda.current_stream().cuda_stream), "b2cnn_score_record_ex")
        return out

    def call_plan(self, window_tensor: torch.Tensor, age: torch.Tensor, mode: str = "independent",
                  return_prob: bool = False):
        """A pre-resolved ``predict()`` for a FIXED pair of device tensors -- the streaming scorer's case: every
        trigger the ring buffer rewrites the same ``[P, 10, 120]`` tensor and the same ages apply (bin/predictStream.py
        rebuilds and re-validates everything per row).  Shapes, dtypes, pointers, workspace and the output tensor are
        resolved once; each call of the returned function is ONE ctypes call (one kernel launch for the production
        shape) on the then-current CUDA stream and returns the same output tensor.  Re-plan after changing weights,
        options or tensors."""
        lib, h = self._ensure_handle()
        dev = self._handle_device
        x = self._check_x(window_tensor)
        if x.device != dev or x.data_ptr() != window_tensor.data_ptr():
            raise RuntimeError("call_plan needs a float32 / bfloat16 tensor already on the model's device (it is captured by address)")
        age = age.reshape(-1)
        if age.device != dev or age.dtype != torch.float32 or not age.is_contiguous() or age.numel() not in (1, x.shape[0]):
            raise RuntimeError("call_plan needs a contiguous float32 age tensor on the model's device with 1 or B elements")
        if mode not in ("independent", "sequence"):
            raise ValueError("mode must be 'independent' or 'sequence'")
        B = x.shape[0]
        md = capi.MODE_INDEPENDENT if mode == "independent" else capi.MODE_SEQUENCE
        dtype = capi.DTYPE_BF16 if x.dtype == torch.bfloat16 else capi.DTYPE_F32
        out = torch.empty(B, dtype=torch.float32, device=dev)
        ws = torch.empty(max(int(lib.b2cnn_workspace_bytes_for(h, B, md, dtype)), 256), dtype=torch.uint8, device=dev)
        pitch = 0 if x.is_contiguous() else self._row_pitch(x)
        pitch = pitch or self.arch.window
        args = (h, x.data_ptr(), dtype, B, pitch, age.data_ptr(), age.numel(), md, int(return_prob), out.data_ptr(),
                ws.data_ptr(), ws.numel())
        fwd, cur, index, keep = lib.b2cnn_forward_pitched, torch.cuda.current_stream, dev.index, (x, age, ws, self)

        def run():
            rc = fwd(*args, cur(index).cuda_stream)
            if rc:
                capi.check(rc, "b2cnn_forward_pitched")
            return out

        run.keepalive = keep
        return run

    @torch.no_grad()
    def features(self, x: torch.Tensor) -> torch.Tensor:
        """The tensor after ``x.view(-1, MAGICNUM)`` (bin/models.py:29): [B, L_out] fp32."""
        lib, h = self._ensure_handle()
        dev = self._device()
        x = self._check_x(x).to(dev).contiguous()
        B = x.shape[0]
        dtype = capi.DTYPE_BF16 if x.dtype == torch.bfloat16 else capi.DTYPE_F32
        feats = torch.empty(B, self.arch.l_out, dtype=torch.float32, device=dev)
        with torch.cuda.device(dev):
            st = torch.cuda.current_stream().cuda_stream
            capi.check(lib.b2cnn_features(h, x.data_ptr(), dtype, B, feats.data_ptr(), st), "b2cnn_features")
        return feats
