"""GPU: the sliding-window scorer (SlidingScorer / b2cnn_slide_*, csrc/b2cnn_slide.cu) against predict() and the
PyTorch-CPU oracle on the explicit windows of the same streams."""
import ctypes
from dataclasses import replace

import numpy as np
import pytest
import torch

import tskd_b200
from conftest import rel_err
from oracle import mycnn_torch as O
from tskd_b200 import capi

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
TOL = 1e-4          # against the oracle, as tests/test_gpu_tc.py
TOL_PREDICT = 2e-5  # against predict() on the explicit window


def _pair(kind, W, C=3, seed=0):
    oarch = O.stretched(O.ARCHS[kind], C, W)
    ref = O.make_ref(oarch, seed=seed)
    arch = replace(tskd_b200.ARCH_PRESETS[kind].with_shape(C, W), age_coef=oarch.age_coef)
    m = tskd_b200.B200MyCNN(arch, has_out12=oarch.has_out12).to(DEV)
    m.load_state_dict(ref.state_dict())
    return ref, m


def _stream(P, n_push, S, dtype, seed, dist="normal"):
    return tskd_b200.synth.make_windows(P, 3, n_push * S, dist, seed=seed, dtype=dtype).to(DEV)


def _replay(scorer, stream, S, ages, n_push):
    """Push the stream segment by segment (views into the stream: row-padded, sometimes unaligned); yields
    (n, logits or None)."""
    for n in range(1, n_push + 1):
        yield n, scorer.push(stream[:, :, (n - 1) * S:n * S], ages)


# (200, 100): fewer than 32 new features per push, all computed exactly; (200, 8): S < R, so a seam feature reaches
# back over several pushes and the 24-sample tail is assembled from the old tail and the segment
@pytest.mark.parametrize("W,S", [(7504, 1876), (7500, 740), (7502, 1876), (200, 100), (200, 8)])
@pytest.mark.parametrize("kind", ["mycnn5", "mycnn3"])
@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float32])
def test_slide_matches_predict_and_oracle(kind, dtype, W, S):
    P = 130
    ref, m = _pair(kind, W)
    n0 = -(-W // S)
    n_push = n0 + 2
    stream = _stream(P, n_push, S, dtype, seed=11)
    ages = tskd_b200.synth.make_ages(P, seed=11).to(DEV)
    sc = tskd_b200.SlidingScorer(m, P, S, dtype)
    emitted = 0
    for n, got in _replay(sc, stream, S, ages, n_push):
        if n * S < W:
            assert got is None
            continue
        assert got is not None and sc.window_index == n - n0
        win = stream[:, :, n * S - W:n * S]
        want = m.predict(win, ages).cpu().numpy()
        g = got.cpu().numpy()
        assert rel_err(g, want) <= TOL_PREDICT, (n, rel_err(g, want))
        fw = m.features(win).cpu().numpy()
        fs = sc.features().cpu().numpy()
        assert np.abs(fs - fw).max() < 2e-5, (n, np.abs(fs - fw).max())
        wo = O.ref_independent(ref, win.float().cpu(), ages.cpu()).numpy()
        assert rel_err(g, wo) <= TOL, (n, rel_err(g, wo))
        emitted += 1
    assert emitted == n_push - n0 + 1
    sc.close()


def test_slide_full_size_headline_geometry():
    W, S, P = 75000, 7500, 300
    ref, m = _pair("mycnn5", W)
    stream = _stream(P, 12, S, torch.bfloat16, seed=5)
    ages = tskd_b200.synth.make_ages(P, seed=5).to(DEV)
    sc = tskd_b200.SlidingScorer(m, P, S)
    for n, got in _replay(sc, stream, S, ages, 12):
        if n < 10:
            assert got is None
            continue
        win = stream[:, :, n * S - W:n * S]
        assert rel_err(got.cpu().numpy(), m.predict(win, ages).cpu().numpy()) <= TOL_PREDICT
        if n == 12:
            idx = torch.arange(0, P, P // 32)[:32]
            wo = O.ref_independent(ref, win[idx].float().cpu(), ages[idx].cpu()).numpy()
            assert rel_err(got[idx].cpu().numpy(), wo) <= TOL


def test_slide_determinism_prefix_replay_and_age():
    W, S = 7504, 1876
    _, m = _pair("mycnn5", W)
    stream = _stream(1000, 6, S, torch.bfloat16, seed=3)
    big = tskd_b200.SlidingScorer(m, 1000, S)
    small = tskd_b200.SlidingScorer(m, 300, S)
    age_vec = torch.full((1000,), 50.0, device=DEV)
    first = []
    for n in range(1, 7):
        seg = stream[:, :, (n - 1) * S:n * S]
        a = big.push(seg, age=50.0)
        b = small.push(seg[:300].contiguous(), age=age_vec[:300])
        if a is not None:
            assert torch.equal(a[:300], b), n            # prefix of patients; scalar vs [P] age
            first.append(a.clone())
    big.reset()
    again = [o.clone() for _, o in _replay(big, stream, S, age_vec, 6) if o is not None]
    assert len(again) == len(first) and all(torch.equal(x, y) for x, y in zip(first, again))


@pytest.mark.parametrize("kind,dtype", [("mycnn5", torch.bfloat16), ("mycnn5", torch.float32), ("mycnn3", torch.bfloat16)])
def test_slide_nan_inf_pattern(kind, dtype):
    W, S, n_push = 7502, 1876, 8                # W % 4 == 2: the last 2 samples of a window are not covered
    ref, m = _pair(kind, W)
    R = 24 if kind == "mycnn5" else 16
    stream = _stream(6, n_push, S, dtype, seed=9).clone()
    stream[1, 0, S + 900] = float("nan")        # mid-segment of push 2: windows 4, 5 NaN, then finite again
    stream[2, 1, 2 * S + 3] = float("inf")      # first R samples of push 3 (seam)
    stream[3, 2, 3 * S - 2] = float("-inf")     # last R samples of push 3
    stream[4, 0, 3 * S + R // 2] = float("nan")  # seam of push 4
    stream[5, 1, 5 * S - 2] = float("nan")      # uncovered tail of window 5, covered by window 6
    ages = tskd_b200.synth.make_ages(6, seed=9).to(DEV)
    sc = tskd_b200.SlidingScorer(m, 6, S, dtype)
    nan_rows = {}
    for n, got in _replay(sc, stream, S, ages, n_push):
        if got is None:
            continue
        win = stream[:, :, n * S - W:n * S]
        want = O.ref_independent(ref, win.float().cpu(), ages.cpu()).numpy()
        g = got.cpu().numpy()
        assert np.array_equal(np.isnan(g), np.isnan(want)), (n, g, want)
        fin = ~np.isnan(want)
        assert rel_err(g[fin], want[fin]) <= TOL, (n, rel_err(g[fin], want[fin]))
        nan_rows[n] = set(np.flatnonzero(np.isnan(g)).tolist())
    assert 1 in nan_rows[4] and 1 in nan_rows[5] and 1 not in nan_rows[6]
    assert 5 not in nan_rows[5] and 5 in nan_rows[6]
    assert 2 not in nan_rows[5] and 3 not in nan_rows[5]   # +-inf samples give finite logits


def _rc_create(m, P, S, dtype=capi.DTYPE_BF16):
    lib, h = m._ensure_handle()
    s = ctypes.c_void_p()
    rc = lib.b2cnn_slide_create(h, P, S, dtype, ctypes.byref(s))
    if rc == capi.OK:
        lib.b2cnn_slide_destroy(s)
    return rc


def test_slide_errors():
    W, S = 7504, 1876
    _, m = _pair("mycnn5", W)
    assert _rc_create(m, 4, 1874) == capi.EINVAL        # not a multiple of the feature stride
    assert _rc_create(m, 4, 0) == capi.EINVAL
    assert _rc_create(m, 4, W + 4) == capi.EINVAL       # S > W
    assert _rc_create(m, 4, S) == capi.OK
    with pytest.raises(ValueError):
        tskd_b200.SlidingScorer(m, 4, 1874)
    _, m10 = _pair("mycnn5", 1200, C=10)                # the 10-channel numerics geometry: no tensor-core kernel
    assert _rc_create(m10, 4, 120) == capi.EARCH
    with pytest.raises(RuntimeError, match="error 2"):
        tskd_b200.SlidingScorer(m10, 4, 120)
    sc = tskd_b200.SlidingScorer(m, 4, S)
    stream = _stream(4, 5, S, torch.bfloat16, seed=2)
    with pytest.raises(RuntimeError):
        sc.push(stream[:3, :, :S])
    with pytest.raises(RuntimeError):
        sc.push(stream[:, :, :S - 4])
    with pytest.raises(RuntimeError):
        sc.push(stream[:, :, :S].float())
    for n in range(1, 5):
        sc.push(stream[:, :, (n - 1) * S:n * S])
    # new weights make the stored features stale: refused until reset
    ref2 = O.make_ref(O.stretched(O.ARCHS["mycnn5"], 3, W), seed=1)
    m.load_state_dict(ref2.state_dict())
    with pytest.raises(RuntimeError, match="error 5"):
        sc.push(stream[:, :, 4 * S:5 * S])
    with pytest.raises(RuntimeError, match="error 5"):
        sc.features()
    sc.reset()
    out = None
    for n in range(1, 6):
        out = sc.push(stream[:, :, (n - 1) * S:n * S])
    win = stream[:, :, 5 * S - W:5 * S]
    assert rel_err(out.cpu().numpy(), m.predict(win).cpu().numpy()) <= TOL_PREDICT
