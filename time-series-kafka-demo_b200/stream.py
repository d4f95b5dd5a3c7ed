"""Streaming replay at the model boundary (BASELINE.json configs[4], SURVEY.md section 8 f1-lite).

The reference's live path is Kafka -> Spark -> ``write_to_mysql`` (bin/predictStream.py:53-192),
which calls ``model(x_arr, a_arr)`` once per patient row with B=1.  None of that plumbing exists
here (no Kafka / Spark / MySQL in this image, and it is out of scope); this module replays WFDB
numerics records through the window logic ON THE DEVICE (csrc/b2cnn_prep.cu) and hands whole micro-batches of
windows to ONE ``predict()`` call -- the "batched GPU dispatch" the north-star asks for -- either a complete record at
once (``replay``) or trigger by trigger for many patients through device ring buffers (``replay_stream``):

  sendStream.py:39-72      one message per (sample, signal): value = [signal_index, sample];
                           the index is the position in the record's selected signal list
  processStream.py:196-208 per (patient, signal): mean over a 180 s window sliding by 5 s
  processStream.py:62-123  forward-fill, back-fill, then 0-fill of the 5-second grid
  predictStream.py:245-259 600 s windows sliding by 60 s  ->  120 points per signal
  predictStream.py:105-139 x_arr[0, signal_index, :] = the 120 points; absent signals = zeros
  predictStream.py:146-151 age from the patients table, 65.0 when unknown
  predictStream.py:160-162,172-181  sigmoid -> RISK_SCORE row (SUBJECT_ID, PRED_TIME, RISK_SCORE)

The reference's ``x_arr = np.empty(...)`` + stale ``signal_index`` quirk (SURVEY.md section 5)
makes its live MySQL rows non-deterministic, so parity is asserted where it is defined: on
identical ``x_arr`` at the ``model(x, a)`` boundary.
"""
from __future__ import annotations

from dataclasses import dataclass
from typing import List, Sequence, Tuple

import numpy as np

# config.cfg:23 -- the names wfdb.rdrecord(channel_names=...) selects by (sendStream.py:46)
CHANNEL_NAMES = ("HR", "RESP", "PULSE", "PVC Rate per Minute", "SpO2", "CVP", "ST V",
                 "NBP Mean", "NBP Dias", "NBP Sys")
N_CHANNELS = 10          # predictStream.py:105
WINDOW_POINTS = 120      # config.cfg:23 WINDOWSIZE
GRID_S = 5               # processStream.py: 5-second slide
SMOOTH_S = 180           # processStream.py: 180-second window
STRIDE_S = 60            # predictStream.py: 60-second slide


@dataclass
class NumericsRecord:
    """A WFDB format-16 numerics record (little-endian int16, interleaved signals)."""
    names: Tuple[str, ...]
    gains: np.ndarray          # ADC units per physical unit
    baselines: np.ndarray
    fs: float                  # samples per second (1/60 for MIMIC numerics)
    raw: np.ndarray            # [n_samples, n_signals] int16; -32768 == missing

    @property
    def physical(self) -> np.ndarray:
        p = (self.raw.astype(np.float64) - self.baselines) / self.gains
        p[self.raw == -32768] = np.nan
        return p

    @classmethod
    def from_wfdb_files(cls, hea_path: str, dat_path: str) -> "NumericsRecord":
        with open(hea_path) as f:
            lines = [l.split() for l in f.read().strip().splitlines() if l.strip() and not l.startswith("#")]
        n_sig = int(lines[0][1])
        fs = float(lines[0][2].split("/")[0])
        names, gains, bases = [], [], []
        for l in lines[1:1 + n_sig]:
            g = l[2].split("/")[0]
            gain = float(g.split("(")[0]) if g else 200.0
            base = float(g.split("(")[1].rstrip(")")) if "(" in g else float(l[4])
            names.append(" ".join(l[8:])); gains.append(gain or 200.0); bases.append(base)
        raw = np.fromfile(dat_path, dtype="<i2").reshape(-1, n_sig)
        return cls(tuple(names), np.array(gains), np.array(bases), fs, raw)


def selected_signals(record: NumericsRecord) -> List[int]:
    """Indices of the record's signals whose names are in CHANNEL_NAMES, in record order
    (wfdb.rdrecord(channel_names=...), sendStream.py:46).  Message index i == position here."""
    return [i for i, n in enumerate(record.names) if n in CHANNEL_NAMES]


def assemble_windows_gpu(record: NumericsRecord, device="cuda", dtype=None):
    """The same model inputs built ON THE DEVICE by libb2cnn's b2cnn_prep_windows (csrc/b2cnn_prep.cu): the raw
    int16 record goes up once (a few KB), smoothing / filling / window assembly run as four small kernels and the
    [n_windows, 10, 120] batch is written straight into the tensor predict() reads.  oracle/stream_np.py (pinned
    against pandas) is the checker of this path.  Returns (x [n_windows, 10, 120] f32|bf16 on `device`, t0 [n_windows] f64 seconds)."""
    import ctypes

    import torch

    from . import capi
    lib = capi.load_library()
    dev = torch.device(device)
    if dev.type != "cuda":
        raise RuntimeError("assemble_windows_gpu needs a CUDA device; there is no CPU fallback")
    dtype = dtype or torch.float32
    if dtype not in (torch.float32, torch.bfloat16):
        raise RuntimeError("dtype must be torch.float32 or torch.bfloat16")
    sel = np.ascontiguousarray(selected_signals(record), dtype=np.int32)
    gains = np.ascontiguousarray(record.gains, dtype=np.float64)
    bases = np.ascontiguousarray(record.baselines, dtype=np.float64)
    raw_h = np.ascontiguousarray(record.raw, dtype=np.int16)
    n, n_sig = raw_h.shape
    cfg = capi.PrepConfig(N_CHANNELS, WINDOW_POINTS, GRID_S, SMOOTH_S, STRIDE_S)
    n_win = lib.b2cnn_prep_window_count(n, float(record.fs), ctypes.byref(cfg))
    ws_bytes = lib.b2cnn_prep_workspace_bytes(n, float(record.fs), len(sel), ctypes.byref(cfg))
    if n_win < 0 or ws_bytes < 0:
        raise RuntimeError(f"b2cnn_prep: {capi.last_error()}")
    if n_win == 0 or len(sel) == 0:                                # record shorter than one 600 s window / nothing selected
        return (torch.zeros((n_win if len(sel) == 0 else 0, N_CHANNELS, WINDOW_POINTS), dtype=dtype, device=dev),
                torch.arange(n_win if len(sel) == 0 else 0, dtype=torch.float64, device=dev) * float(STRIDE_S))
    with torch.cuda.device(dev):
        raw_d = torch.from_numpy(raw_h).to(dev)
        x = torch.empty((n_win, N_CHANNELS, WINDOW_POINTS), dtype=dtype, device=dev)
        t0 = torch.empty((n_win,), dtype=torch.float64, device=dev)
        ws = torch.empty((max(int(ws_bytes), 256),), dtype=torch.uint8, device=dev)
        stream = torch.cuda.current_stream(dev).cuda_stream
        rc = lib.b2cnn_prep_windows(raw_d.data_ptr(), n, n_sig, sel.ctypes.data, len(sel), gains.ctypes.data, bases.ctypes.data,
                                    float(record.fs), ctypes.byref(cfg), x.data_ptr(), 0 if dtype == torch.float32 else 1,
                                    t0.data_ptr(), ws.data_ptr(), int(ws.numel()), stream)
        capi.check(rc, "b2cnn_prep_windows")
        ws.record_stream(torch.cuda.current_stream(dev)); raw_d.record_stream(torch.cuda.current_stream(dev))
    return x, t0


def _model_device(model):
    """The CUDA device a (possibly not yet migrated) B200MyCNN lives on: a model built the documented way
    (``B200MyCNN.from_reference(...).eval()``, no ``.to('cuda')``) migrates on its first forward."""
    ensure = getattr(model, "_ensure_handle", None)
    if ensure is not None:
        ensure()
    return next(model.parameters()).device


def _rows(rows, subject_id, t0, prob):
    for tt, p in zip(t0, prob):
        if not np.isnan(p):                                      # predictStream.py:171 drops NaN results
            rows.append((int(subject_id), float(tt), float(p)))


def replay(model, record: NumericsRecord, subject_id: int, age: float = 65.0,
           micro_batch: int = 0) -> List[Tuple[int, float, float]]:
    """Score every window of the record and return the rows the reference INSERTs into
    ``predictions`` (db/init.sql:24-28): (SUBJECT_ID, PRED_TIME [s since record start], RISK_SCORE).
    The raw record goes to the device once; smoothing, filling, window assembly (b2cnn_prep_windows) and scoring
    never leave it.  ``micro_batch`` = windows per predict() call (0 = all at once)."""
    rows: List[Tuple[int, float, float]] = []
    xg, t0g = assemble_windows_gpu(record, device=_model_device(model))
    if len(xg) == 0:
        return rows
    mb = micro_batch or len(xg)
    t0 = t0g.cpu().numpy()
    for b0 in range(0, len(xg), mb):
        prob = model.predict(xg[b0:b0 + mb], age, return_prob=True).cpu().numpy()
        _rows(rows, subject_id, t0[b0:b0 + mb], prob)
    return rows


class PatientRing:
    """Device-resident streaming state for P patients (libb2cnn's b2cnn_ring_*, csrc/b2cnn_prep.cu): what
    bin/predictStream.py:70-156 rebuilds on the host for every patient row of every trigger.  ``push`` appends one
    trigger's samples for all patients and returns the ``[P, 10, 120]`` batch of the window that just completed
    (``None`` while the first 600 s fill) -- the input of ONE ``predict()`` call per trigger."""

    def __init__(self, n_patients: int, n_sig: int, fs: float, device="cuda", dtype=None):
        import ctypes

        import torch

        from . import capi
        self._lib = capi.load_library()
        self.device = torch.device(device)
        if self.device.type != "cuda":
            raise RuntimeError("PatientRing needs a CUDA device; there is no CPU fallback")
        if self.device.index is None:
            self.device = torch.device("cuda", torch.cuda.current_device())
        self.dtype = dtype or torch.float32
        if self.dtype not in (torch.float32, torch.bfloat16):
            raise RuntimeError("dtype must be torch.float32 or torch.bfloat16")
        self.n_patients, self.n_sig, self.fs = int(n_patients), int(n_sig), float(fs)
        cfg = capi.PrepConfig(N_CHANNELS, WINDOW_POINTS, GRID_S, SMOOTH_S, STRIDE_S)
        h = ctypes.c_void_p()
        capi.check(self._lib.b2cnn_ring_create(ctypes.byref(cfg), self.n_patients, self.n_sig, self.fs, self.device.index,
                                               ctypes.byref(h)), "b2cnn_ring_create")
        self._h = h
        self.x = torch.empty((self.n_patients, N_CHANNELS, WINDOW_POINTS), dtype=self.dtype, device=self.device)

    def close(self):
        h, self._h = getattr(self, "_h", None), None
        if h is not None:
            self._lib.b2cnn_ring_destroy(h)

    __del__ = close

    def set_signals(self, patient: int, sel, gains=None, baselines=None):
        """``sel``: frame columns of the model's signals for this patient (position i -> model channel i, the
        message index of bin/sendStream.py:59-64); ``gains`` / ``baselines`` [n_sig] for ADC input."""
        from . import capi
        sel = np.ascontiguousarray(sel, dtype=np.int32)
        g = None if gains is None else np.ascontiguousarray(gains, dtype=np.float64)
        b = None if baselines is None else np.ascontiguousarray(baselines, dtype=np.float64)
        capi.check(self._lib.b2cnn_ring_set_signals(self._h, int(patient), sel.ctypes.data, len(sel),
                                                    None if g is None else g.ctypes.data,
                                                    None if b is None else b.ctypes.data, None), "b2cnn_ring_set_signals")

    def set_record_signals(self, patient: int, record: NumericsRecord):
        self.set_signals(patient, selected_signals(record), record.gains, record.baselines)

    def reset(self):
        from . import capi
        capi.check(self._lib.b2cnn_ring_reset(self._h, None), "b2cnn_ring_reset")

    def push(self, new_samples, grid_points: bool = False):
        """``new_samples`` [P, n_new, n_sig]: int16 ADC units (WFDB format 16, -32768 = missing) or float64 physical
        values (NaN = missing), host or device; with ``grid_points`` the rows are 5-second grid points that
        bin/processStream.py already smoothed and filled (the ``call-stream`` payload).  Returns ``(x [P,10,120] on the device, window_index, t0_seconds)`` or
        ``None`` while the first window is still filling.  The returned tensor is reused by the next push.
        One push carries at most one stride (60 s) of samples or 12 grid points and emits at most one window: a push
        after which the next window would be complete too raises RuntimeError and leaves the ring as it was.  Cutting
        the stream at cumulative stride boundaries (push n = the samples with time < n * 60 s) never does."""
        import ctypes

        import torch

        from . import capi
        t = torch.as_tensor(new_samples)
        if t.dim() == 2:
            t = t.unsqueeze(0)
        if grid_points:
            kind, t = capi.SAMPLES_GRID, t.to(torch.float64)
        elif t.dtype == torch.int16:
            kind = capi.SAMPLES_ADC16
        else:
            kind, t = capi.SAMPLES_F64, t.to(torch.float64)
        if t.shape[0] != self.n_patients or t.shape[2] != self.n_sig:
            raise RuntimeError(f"expected samples [{self.n_patients}, n_new, {self.n_sig}], got {tuple(t.shape)}")
        t = t.to(self.device).contiguous()
        em, widx, t0 = ctypes.c_int32(0), ctypes.c_int64(-1), ctypes.c_double(0.0)
        with torch.cuda.device(self.device):
            st = torch.cuda.current_stream().cuda_stream
            capi.check(self._lib.b2cnn_ring_push(self._h, t.data_ptr(), kind, t.shape[1], self.x.data_ptr(),
                                                 0 if self.dtype == torch.float32 else 1, ctypes.byref(em), ctypes.byref(widx),
                                                 ctypes.byref(t0), st), "b2cnn_ring_push")
            t.record_stream(torch.cuda.current_stream())
        return (self.x, int(widx.value), float(t0.value)) if em.value else None


def trigger_cuts(n_samples: int, fs: float) -> List[int]:
    """Where the triggers of a record sampled at ``fs`` begin and end: trigger n (n = 1, 2, ...) holds the samples with
    time < n * STRIDE_S on the ring's integer-nanosecond time base (sample i at i * round(1e9 / fs) ns).  Returns
    ``[0, c_1, c_2, ..., n_samples]``; trigger n = samples ``c_{n-1} .. c_n - 1``."""
    period_ns, stride_ns = int(round(1e9 / fs)), STRIDE_S * 1_000_000_000
    cuts, k = [0], 1
    while cuts[-1] < n_samples:
        cuts.append(min(n_samples, -(-k * stride_ns // period_ns)))     # number of samples with i * period < k * stride
        k += 1
    return cuts


def replay_stream(model, records: Sequence[NumericsRecord], subject_ids: Sequence[int], ages=65.0,
                  samples_per_trigger: int = 0) -> List[Tuple[int, float, float]]:
    """The live path's shape (bin/predictStream.py:263: one foreachBatch per 60 s trigger) with the B = 1 per-row loop
    turned into the batched dispatch: all records (same sampling rate and length, one per patient) are fed trigger by
    trigger into a PatientRing and every trigger costs ONE ``predict()`` over ``[P, 10, 120]``.  Trigger n carries the
    samples with time < n * 60 s, so every trigger from the 10th on emits exactly the window that just completed, at
    any sampling rate; ``samples_per_trigger`` > 0 cuts fixed-size triggers instead (each must keep to one window per
    push, see ``PatientRing.push``).  Returns the ``predictions`` rows (db/init.sql:24-28) of all patients, trigger-major."""
    P = len(records)
    if P == 0:
        return []
    if len(subject_ids) != P:
        raise RuntimeError(f"replay_stream: {P} records but {len(subject_ids)} subject ids")
    fs, n, n_sig = records[0].fs, records[0].raw.shape[0], records[0].raw.shape[1]
    if any(r.fs != fs or r.raw.shape != (n, n_sig) for r in records):
        raise RuntimeError("replay_stream: the records of one ring share sampling rate, length and signal count")
    dev = _model_device(model)
    ring = PatientRing(P, n_sig, fs, device=dev)
    try:
        return _replay_ring(model, ring, records, subject_ids, ages, samples_per_trigger, dev)
    finally:
        ring.close()                                  # the native ring is freed on error paths too


def _replay_ring(model, ring, records, subject_ids, ages, samples_per_trigger, dev):
    import torch
    P, fs, n = len(records), records[0].fs, records[0].raw.shape[0]
    for p, r in enumerate(records):
        ring.set_record_signals(p, r)
    cuts = list(range(0, n, samples_per_trigger)) + [n] if samples_per_trigger else trigger_cuts(n, fs)
    raw = torch.from_numpy(np.stack([np.ascontiguousarray(r.raw, dtype=np.int16) for r in records])).to(dev)
    age_t = torch.as_tensor(ages, dtype=torch.float32).reshape(-1)
    if age_t.numel() not in (1, P):
        raise RuntimeError(f"ages must be a scalar or have {P} elements")
    rows: List[Tuple[int, float, float]] = []
    # the ring rewrites ONE [P, 10, 120] tensor per trigger: shapes, pointers and the output buffer are resolved once
    score = model.call_plan(ring.x, age_t.to(dev), return_prob=True) if hasattr(model, "call_plan") else None
    for i0, i1 in zip(cuts[:-1], cuts[1:]):
        out = ring.push(raw[:, i0:i1])
        if out is None:
            continue
        x, _, t0 = out
        prob = (score() if score else model.predict(x, age_t, return_prob=True)).cpu().numpy()    # one batched call per trigger
        for p in range(P):
            if not np.isnan(prob[p]):                                     # predictStream.py:171 drops NaN results
                rows.append((int(subject_ids[p]), t0, float(prob[p])))
    return rows


# ---------------------------------------------------------------------------------------------- wire formats (row f3)
def _message_buffer(values, device):
    """A trigger's message values (a sequence of bytes objects, or one bytes buffer + offsets) as device tensors."""
    import torch
    if isinstance(values, tuple):
        buf, offs = values
        offs = np.ascontiguousarray(offs, dtype=np.int64)
    else:
        lens = np.fromiter((len(v) for v in values), dtype=np.int64, count=len(values))
        offs = np.concatenate([[0], np.cumsum(lens)]).astype(np.int64)
        buf = b"".join(values)
    b = torch.frombuffer(bytearray(buf) if len(buf) else bytearray(1), dtype=torch.uint8).to(device)
    return b, torch.from_numpy(offs).to(device), len(offs) - 1


def decode_sample_messages(values, rows, n_rows: int, n_sig: int, device="cuda"):
    """The ``[i, val]`` messages of bin/sendStream.py:59-64, decoded on the device and scattered into the fp64 frame
    ``[n_rows, n_sig]`` (NaN = no message / missing) that ``PatientRing.push`` takes.  ``rows[t]`` = frame row of message t
    (patient * n_new + sample, from the message key and arrival order).  Returns (frame, number of malformed messages)."""
    import torch

    from . import capi
    lib = capi.load_library()
    dev = torch.device(device)
    b, offs, n = _message_buffer(values, dev)
    rows_t = torch.as_tensor(np.ascontiguousarray(rows, dtype=np.int64)).to(dev)
    frame = torch.empty((n_rows, n_sig), dtype=torch.float64, device=dev)
    bad = torch.zeros(1, dtype=torch.int32, device=dev)
    with torch.cuda.device(dev):
        capi.check(lib.b2cnn_decode_sample_messages(b.data_ptr(), offs.data_ptr(), n, None, None, rows_t.data_ptr(), frame.data_ptr(),
                                                    n_rows, n_sig, bad.data_ptr(), torch.cuda.current_stream().cuda_stream),
                   "b2cnn_decode_sample_messages")
        for t in (b, offs, rows_t):
            t.record_stream(torch.cuda.current_stream())
    return frame, int(bad.item())


def decode_array_messages(values, max_vals: int = 12, device="cuda"):
    """The ``[v0,v1,...]`` messages of bin/processStream.py:126-131 (12 grid points per patient, channel and trigger),
    decoded on the device.  Returns (vals [n_msgs, max_vals] fp64 NaN-padded, counts [n_msgs], malformed)."""
    import torch

    from . import capi
    lib = capi.load_library()
    dev = torch.device(device)
    b, offs, n = _message_buffer(values, dev)
    vals = torch.empty((n, max_vals), dtype=torch.float64, device=dev)
    counts = torch.empty((n,), dtype=torch.int32, device=dev)
    bad = torch.zeros(1, dtype=torch.int32, device=dev)
    with torch.cuda.device(dev):
        capi.check(lib.b2cnn_decode_array_messages(b.data_ptr(), offs.data_ptr(), n, max_vals, vals.data_ptr(), counts.data_ptr(),
                                                   bad.data_ptr(), torch.cuda.current_stream().cuda_stream), "b2cnn_decode_array_messages")
        for t in (b, offs):
            t.record_stream(torch.cuda.current_stream())
    return vals, counts, int(bad.item())


def pack_frame(subject_ids, samples: np.ndarray, first_index: int = 0, grid_points: bool = False) -> bytes:
    """One binary frame per trigger for all patients (include/b2cnn.h b2cnn_frame_header): ``samples`` [P, n_new, n_sig]
    int16 ADC units or float64 -- the array ``PatientRing.push`` takes, so decoding is one copy."""
    import struct

    from . import capi
    samples = np.ascontiguousarray(samples)
    if samples.ndim != 3 or samples.dtype not in (np.int16, np.float64):
        raise ValueError("samples must be [P, n_new, n_sig] int16 or float64")
    kind = capi.SAMPLES_GRID if grid_points else (capi.SAMPLES_ADC16 if samples.dtype == np.int16 else capi.SAMPLES_F64)
    P, n_new, n_sig = samples.shape
    ids = np.ascontiguousarray(subject_ids, dtype="<i4")
    if ids.shape != (P,):
        raise ValueError("one subject id per patient")
    head = struct.pack("<IHHIIIIQ", capi.FRAME_MAGIC, 1, kind, P, n_new, n_sig, 0, int(first_index))
    pad = b"\0" * ((-(len(head) + ids.nbytes)) % 8)
    return head + ids.tobytes() + pad + samples.astype(samples.dtype.newbyteorder("<")).tobytes()


def unpack_frame(frame: bytes):
    """Validates a frame with the library (b2cnn_frame_check) and returns (subject_ids, samples, first_index, grid_points)
    as zero-copy numpy views of the buffer."""
    import ctypes

    from . import capi
    lib = capi.load_library()
    hd, o_ids, o_smp = capi.FrameHeader(), ctypes.c_int64(0), ctypes.c_int64(0)
    buf = (ctypes.c_char * len(frame)).from_buffer_copy(frame)
    capi.check(lib.b2cnn_frame_check(ctypes.addressof(buf), len(frame), ctypes.byref(hd), ctypes.byref(o_ids), ctypes.byref(o_smp)),
               "b2cnn_frame_check")
    ids = np.frombuffer(frame, dtype="<i4", count=hd.n_patients, offset=o_ids.value)
    dt = "<i2" if hd.kind == capi.SAMPLES_ADC16 else "<f8"
    smp = np.frombuffer(frame, dtype=dt, count=hd.n_patients * hd.n_new * hd.n_sig, offset=o_smp.value)
    return ids, smp.reshape(hd.n_patients, hd.n_new, hd.n_sig), int(hd.first_index), hd.kind == capi.SAMPLES_GRID
