"""TEST INFRASTRUCTURE ONLY -- numpy restatement of the two steps in front of the model call.

  bin/processStream.py:196-208  per (patient, signal): ``avg(value)`` over Spark's
                                ``window(timestamp, "180 seconds", "5 seconds")``, nulls skipped
  bin/processStream.py:62-123   forward-fill, back-fill (ordered by windowStart), then ``fillna(0)``
  bin/predictStream.py:245-259  600 s windows sliding by 60 s -> 120 points per signal
  bin/predictStream.py:105-139  x_arr[0, signal_index, :] = the 120 points; absent signals = zeros

Window-edge convention (pinned by tests/test_stream_oracle.py against pandas, see oracle/stream_pandas.py):
Spark's sliding windows are half-open ``[windowStart, windowStart + 180)`` with starts on the 5-second lattice.
Grid point k of this restatement is the Spark window with ``windowStart = 5k - 175``, labelled by
``tau_k = 5k`` (its last 5-second bin): it averages the valid samples with time in ``[tau - 175, tau + 5)``.
For sample times ON the 5-second lattice (every MIMIC numerics record: fs = 1/60 Hz) that is the same sample set
as pandas' ``rolling('3min')`` window ``(tau - 180, tau]`` over the ``resample('5S').first()`` grid
(bin/explore_torch.ipynb:402,405) -- a sample exactly at ``tau - 180`` is OUT, one exactly at ``tau`` is IN, under
both.  The sequence runs over tau = 0 .. floor(t_last / 5) * 5 (pandas' resample range); Spark would emit 35 more
trailing partial windows (starts up to t_last), which predictStream never assembles into a full 600 s window.

This module is the checker of csrc/b2cnn_prep.cu / b2cnn_ring.cu; the product never imports it.
"""
from __future__ import annotations

from typing import Tuple

import numpy as np

N_CHANNELS = 10          # predictStream.py:105
WINDOW_POINTS = 120      # config.cfg:23 WINDOWSIZE
GRID_S = 5               # processStream.py:199  5-second slide
SMOOTH_S = 180           # processStream.py:199  180-second window
STRIDE_S = 60            # predictStream.py:252  60-second slide


NS = 1_000_000_000


def sample_period_ns(fs: float) -> int:
    """Sample i sits at i * round(1e9 / fs) ns (the time base of pandas' DatetimeIndex and of the device kernels)."""
    return int(round(1e9 / fs))


def smooth_to_grid(samples: np.ndarray, fs: float, fill: bool = True, n_grid: int | None = None) -> np.ndarray:
    """One signal: value at grid label tau (multiples of 5 s) = mean of the valid samples with time in
    [tau - 175, tau + 5); NaN samples are skipped (Spark avg ignores nulls); then ffill, bfill, 0-fill.
    ``n_grid`` overrides the number of grid points (default: labels up to the last sample's time)."""
    period_ns = sample_period_ns(fs)
    t = np.arange(samples.shape[0], dtype=np.int64) * period_ns       # integer nanoseconds: edges compare exactly
    if n_grid is None:
        n_grid = int(t[-1] // (GRID_S * NS)) + 1
    tau = np.arange(n_grid, dtype=np.int64) * (GRID_S * NS)
    lo = np.searchsorted(t, tau - (SMOOTH_S - GRID_S) * NS, side="left")   # first sample with t >= tau - 175
    hi = np.searchsorted(t, tau + GRID_S * NS, side="left")                # first sample with t >= tau + 5
    ok = ~np.isnan(samples)
    g = np.full(n_grid, np.nan)
    for k in range(n_grid):                                            # direct sums in time order, like Spark's avg
        sl = slice(lo[k], hi[k])
        m = ok[sl]
        if m.any():
            g[k] = samples[sl][m].sum() / m.sum() if m.sum() > 1 else samples[sl][m][0]
    if not fill:
        return g
    return fill_grid(g)


def fill_grid(g: np.ndarray) -> np.ndarray:
    """processStream.py:62-123: last(ignorenulls) over rows up to the current one, first(ignorenulls) over the rows
    from the current one on, then fillna(0)."""
    g = g.copy()
    n_grid = g.shape[0]
    idx = np.where(~np.isnan(g), np.arange(n_grid), -1)               # forward fill
    np.maximum.accumulate(idx, out=idx)
    g = np.where(idx >= 0, g[np.maximum(idx, 0)], np.nan)
    if np.isnan(g).any():                                              # back fill, then zeros
        good = np.where(~np.isnan(g))[0]
        if good.size:
            g[:good[0]] = g[good[0]]
        g = np.nan_to_num(g, nan=0.0)
    return g


def grids_of_record(record, sel) -> np.ndarray:
    """[n_sel][n_grid] filled 5-second grids of the selected signals of a NumericsRecord-like object."""
    phys = record.physical
    return np.stack([smooth_to_grid(phys[:, s], record.fs) for s in sel]) if len(sel) else np.zeros((0, 0))


def windows_from_grids(grids: np.ndarray) -> Tuple[np.ndarray, np.ndarray]:
    """x_arr [n_windows, 10, 120] float64 (as predictStream.py:105 builds it) and window start times [s]."""
    n_grid = grids.shape[1] if grids.size else 0
    step = STRIDE_S // GRID_S
    starts = np.arange(0, n_grid - WINDOW_POINTS + 1, step)
    x = np.zeros((len(starts), N_CHANNELS, WINDOW_POINTS), dtype=np.float64)    # absent signals: zeros (:131)
    for ch in range(grids.shape[0]):                                            # message index == ch
        x[:, ch, :] = np.lib.stride_tricks.sliding_window_view(grids[ch], WINDOW_POINTS)[starts]
    return x, starts * float(GRID_S)


def assemble_windows(record, sel) -> Tuple[np.ndarray, np.ndarray]:
    """All model inputs of a whole-record replay."""
    if not len(sel):
        return np.zeros((0, N_CHANNELS, WINDOW_POINTS)), np.zeros((0,))
    return windows_from_grids(grids_of_record(record, sel))


def ring_schedule(fs: float, sizes, grid_points: bool = False):
    """The bookkeeping of a per-patient ring (b2cnn_ring_push) restated: one push of sizes[i] samples (grid points with
    ``grid_points``) finalises grid points 0 .. k_end-1 (k_end = floor(t_next / 5 s), t_next = time of the first sample
    not yet received) and emits the next window once its last point is final.  A push after which the window after that
    one would be complete too is refused and changes nothing.  Returns [(k_end, emitted window or -1, refused)]."""
    period_ns, grid_ns, step = sample_period_ns(fs), GRID_S * NS, STRIDE_S // GRID_S
    n, k_done, w_next, out = 0, 0, 0, []
    for s in sizes:
        k_end = k_done + s if grid_points else (n + s) * period_ns // grid_ns
        if step * (w_next + 1) + WINDOW_POINTS <= k_end:
            out.append((k_end, -1, True))
            continue
        emit = step * w_next + WINDOW_POINTS <= k_end
        out.append((k_end, w_next if emit else -1, False))
        w_next += emit
        n, k_done = n + (0 if grid_points else s), k_end
    return out


def causal_windows(unfilled: np.ndarray, k_ends) -> np.ndarray:
    """The windows a stream can emit: window w is cut when grid points 0 .. k_ends[w]-1 are final (its emitting push
    has finalised them; k_ends[w] >= 12 w + 120).  ``unfilled`` [n_sel][>= max(k_ends)] are the smoothed grid points
    before any fill (``smooth_to_grid(..., fill=False)``).  Forward fill is causal already; the leading gap is
    back-filled from the first valid point among the final ones, else 0 -- where the whole-record form back-fills from
    the future.  Returns x [len(k_ends), 10, 120] float64."""
    step = STRIDE_S // GRID_S
    n_sel = unfilled.shape[0]
    x = np.zeros((len(k_ends), N_CHANNELS, WINDOW_POINTS), dtype=np.float64)
    for ch in range(n_sel):
        g = unfilled[ch]
        idx = np.where(~np.isnan(g), np.arange(g.shape[0]), -1)       # forward fill
        np.maximum.accumulate(idx, out=idx)
        ff = np.where(idx >= 0, g[np.maximum(idx, 0)], np.nan)
        valid = np.nonzero(~np.isnan(g))[0]
        for w, k_end in enumerate(k_ends):
            k_end = int(k_end)
            if k_end < step * w + WINDOW_POINTS or k_end > g.shape[0]:
                raise ValueError(f"window {w} is not complete at k_end {k_end} / beyond the grid")
            v = ff[step * w:step * w + WINDOW_POINTS].copy()
            first = valid[0] if valid.size and valid[0] < k_end else -1
            v[np.isnan(v)] = g[first] if first >= 0 else 0.0
            x[w, ch] = v
    return x
