"""GPU: the sequence-mode LSTM state as an input and an output -- predict_record(mode="sequence", state=...,
return_state=True), b2cnn_score_record_state, SlidingScorer.admit(..., lstm=...) and b2cnn_slide_admit_ex.

The state of one recording or patient is [2, 2, 16] = [layer][h | c][unit] (export()["lstm"]'s layout); the float64
truth is oracle/record_state_ref.py, nn.LSTM called with (h0, c0).

- split identity: a recording cut at window k into x[..., :(k-1)S + W] and x[..., kS:], chained through the state, gives
  the outputs and final state of one call: bit for bit (NaN for NaN) on the generic path and on the tensor cores, 24
  chained hourly chunks of a 24 h recording included;
- a random non-zero state against float64 on both paths, outputs and state_out;
- state=None and state=zeros are today's call; n_w = 0 passes the state through; a NaN state poisons its own recording
  only; refusals before any launch, in Python and in the C ABI; the launch list of the state call;
- the warm-start recipe: a patient admitted at T from its backtest is scored as predict_record over the whole stream;
  an admission with a short history starts its first step from the given state; the other patients and an independent
  scorer are untouched."""
import collections
import ctypes
import json
import os
import subprocess
import sys

import pytest
import torch

import tskd_b200
from oracle.record_state_ref import sequence_with_state
from oracle.train_ref import BETA
from test_gpu_record import _records, _tc_pair, _wins
from test_gpu_record_sequence import BETA_TC_SEQ, _check
from test_gpu_slide_generic import _golden, _pair as _generic_pair, _same
from tskd_b200 import capi

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
BF, F32 = torch.bfloat16, torch.float32


def _n_w(N, W, S):
    return (N - W) // S + 1 if N >= W else 0


def _state(B, seed, scale=0.5):
    g = torch.Generator().manual_seed(seed)
    return (scale * torch.randn(B, 2, 2, 16, generator=g)).to(DEV)


def _chain(m, x, S, age, k, path, state=None):
    """x cut at window k, chained through the state: (outputs [B, n_w], final state)"""
    W = m.arch.window
    a, sa = m.predict_record(x[:, :, :(k - 1) * S + W], S, age, path=path, mode="sequence", state=state, return_state=True)
    b, sb = m.predict_record(x[:, :, k * S:], S, age, path=path, mode="sequence", state=sa, return_state=True)
    assert a.shape[1] == k
    return torch.cat([a, b], dim=1), sb


def _truth(ref, x, S, age, state=None, act="tanh", affine=None):
    """float64 and float32 references: (z [B, n_w], state [B, 2, 2, 16]) each"""
    W = ref.arch.window
    res = {}
    for dt in (torch.float64, torch.float32):
        zs, ss = [], []
        for b in range(x.shape[0]):
            r = sequence_with_state(ref, _wins(x[b:b + 1].cpu(), W, S), age.reshape(-1)[0 if age.numel() == 1 else b],
                                    None if state is None else state[b], dtype=dt, act=act, affine=affine)
            zs.append(r["z"])
            ss.append(r["state"])
        res[dt] = (torch.stack(zs), torch.stack(ss))
    return res[torch.float64], res[torch.float32]


# ------------------------------------------------------------------ 1. split identity
@pytest.mark.parametrize("B", [1, 3, 130])
@pytest.mark.parametrize("S", [12, 120])
@pytest.mark.parametrize("dtype", [F32, BF], ids=["f32", "bf16"])
def test_generic_split_identity(dtype, S, B):
    _, m = _golden(5)
    n_w = 9
    x = _records(B, 10, 120 + (n_w - 1) * S + 5, dtype, seed=S + B).to(DEV)
    age = tskd_b200.synth.make_ages(B, seed=S).to(DEV)
    for state in (None, _state(B, seed=B)):
        full, sf = m.predict_record(x, S, age, path="generic", mode="sequence", state=state, return_state=True)
        assert full.shape == (B, n_w) and sf.shape == (B, 2, 2, 16) and m.last_path == "generic"
        for k in (1, n_w // 2, n_w - 1):
            out, s = _chain(m, x, S, age, k, "generic", state)
            assert _same(out, full) and _same(s, sf), (k, state is None)


def test_generic_split_identity_relu_affine():
    """C = 10, relu, a folded affine whose second scale is negative"""
    _, m, _ = _generic_pair((10, 10, 5, 3, 2, 200), act="relu", aff_seed=7, seed=11)
    S, n_w = 24, 8
    for dtype in (F32, BF):
        x = _records(3, 10, 200 + (n_w - 1) * S + 3, dtype, seed=5).to(DEV)
        age = tskd_b200.synth.make_ages(3, seed=5).to(DEV)
        full, sf = m.predict_record(x, S, age, path="generic", mode="sequence", return_state=True)
        for k in (1, n_w // 2, n_w - 1):
            out, s = _chain(m, x, S, age, k, "generic")
            assert _same(out, full) and _same(s, sf), (dtype, k)


def test_tensorcore_split_identity():
    W, S, n_w = 7504, 752, 12
    ref, m = _tc_pair("mycnn5", 3, W, 31)
    x = _records(3, 3, W + (n_w - 1) * S + 5, BF, seed=31).to(DEV)
    age = tskd_b200.synth.make_ages(3, seed=31).to(DEV)
    full, sf = m.predict_record(x, S, age, path="tensorcore", mode="sequence", return_state=True)
    assert m.last_path == "tensorcore"
    for k in (1, n_w // 2, n_w - 1):
        out, s = _chain(m, x, S, age, k, "tensorcore")
        assert torch.equal(out, full) and torch.equal(s, sf), k
    (t, ts), (t32, ts32) = _truth(ref, x, S, age)
    _check([("z", full, t, t32, BETA_TC_SEQ), ("state", sf, ts, ts32, BETA_TC_SEQ)])


@torch.no_grad()
def test_24h_in_hourly_chunks():
    """[1, 3, 10.8M] bf16 at W = 75000, S = 7500 (125 Hz): 24 chained calls of one hour of windows each against one call"""
    W, S, N = 75000, 7500, 10_800_000
    _, m = _tc_pair("mycnn5", 3, W, 41)
    x = _records(1, 3, N, BF, seed=41).to(DEV)
    age = torch.tensor([63.0], device=DEV)
    full, sf = m.predict_record(x, S, age, mode="sequence", return_state=True)
    assert full.shape == (1, 1431) and m.last_path == "tensorcore"
    per = 3600 * 125 // S                                                # 60 windows an hour
    outs, s = [], None
    for j in range(24):
        w0, w1 = j * per, min((j + 1) * per, full.shape[1])
        o, s = m.predict_record(x[:, :, w0 * S:(w1 - 1) * S + W], S, age, mode="sequence", state=s, return_state=True)
        assert o.shape == (1, w1 - w0)
        outs.append(o)
    assert torch.equal(torch.cat(outs, dim=1), full) and torch.equal(s, sf)


# ------------------------------------------------------------------ 2. a random state against float64
@pytest.mark.parametrize("path", ["generic", "tensorcore"])
def test_random_state_against_float64(path):
    if path == "generic":
        ref, m = _golden(5)
        C, W, S, dtype, beta = 10, 120, 12, F32, BETA
    else:
        ref, m = _tc_pair("mycnn5", 3, 7504, 51)
        C, W, S, dtype, beta = 3, 7504, 752, BF, BETA_TC_SEQ
    B = 5
    x = _records(B, C, W + 9 * S + 3, dtype, seed=51).to(DEV)
    age = tskd_b200.synth.make_ages(B, seed=51).to(DEV)
    state = _state(B, seed=51)
    out, so = m.predict_record(x, S, age, path=path, mode="sequence", state=state, return_state=True)
    (t, ts), (t32, ts32) = _truth(ref, x, S, age, state.cpu())
    _check([("z", out, t, t32, beta), ("state", so, ts, ts32, beta)])
    assert not torch.equal(out, m.predict_record(x, S, age, path=path, mode="sequence"))      # the state mattered


# ------------------------------------------------------------------ 3. today's call, n_w = 0, NaN, conversions
@pytest.mark.parametrize("path", ["generic", "tensorcore"])
def test_zero_state_is_todays_call(path):
    W = 7504
    _, m = _tc_pair("mycnn5", 3, W, 61)
    S, B = 1876, 4
    x = _records(B, 3, W + 6 * S, BF, seed=61).to(DEV)
    age = tskd_b200.synth.make_ages(B, seed=61).to(DEV)
    today = m.predict_record(x, S, age, path=path, mode="sequence")
    a, sa = m.predict_record(x, S, age, path=path, mode="sequence", return_state=True)
    b = m.predict_record(x, S, age, path=path, mode="sequence", state=torch.zeros(B, 2, 2, 16, device=DEV))
    c, sc = m.predict_record(x, S, age, path=path, mode="sequence", state=torch.zeros(B, 2, 2, 16, device=DEV), return_state=True)
    assert torch.equal(a, today) and torch.equal(b, today) and torch.equal(c, today) and torch.equal(sa, sc)
    assert torch.equal(m.predict_record(x, S, age, path=path, mode="sequence", return_prob=True),
                       m.predict_record(x, S, age, path=path, mode="sequence", return_prob=True, return_state=True)[0])
    # other float dtypes and devices are converted to float32 on the model's device
    st = _state(B, seed=62)
    want = m.predict_record(x, S, age, path=path, mode="sequence", state=st, return_state=True)
    for other in (st.double().cpu(), st.cpu(), st.double()):
        got = m.predict_record(x, S, age, path=path, mode="sequence", state=other, return_state=True)
        assert torch.equal(got[0], want[0]) and torch.equal(got[1], want[1])


def test_no_windows_pass_the_state_through():
    _, m = _golden(5)
    x = _records(3, 10, 119, F32, seed=7).to(DEV)
    st = _state(3, seed=7)
    st[1, 0, 1, 3] = float("nan")
    out, so = m.predict_record(x, 12, None, mode="sequence", state=st, return_state=True)
    assert out.shape == (3, 0) and _same(so, st) and so.data_ptr() != st.data_ptr()
    out, so = m.predict_record(x, 12, None, mode="sequence", return_state=True)
    assert out.shape == (3, 0) and torch.equal(so, torch.zeros(3, 2, 2, 16, device=DEV))
    # the C ABI: state_out = state_in, or zeros
    lib, h = m._ensure_handle()
    sink = torch.full((3, 2, 2, 16), 7.0, device=DEV)
    stream = torch.cuda.current_stream().cuda_stream
    age = torch.tensor([60.0], device=DEV)
    for src, want in ((st, st), (None, torch.zeros_like(st))):
        rc = lib.b2cnn_score_record_state(h, x.data_ptr(), capi.DTYPE_F32, 3, 119, 119, 12, capi.PATH_GENERIC, capi.MODE_SEQUENCE,
                                          age.data_ptr(), 1, 0, sink.data_ptr(), None if src is None else src.data_ptr(),
                                          sink.data_ptr(), None, 0, stream)
        assert rc == 0, capi.last_error()
        torch.cuda.synchronize()
        assert _same(sink, want)


@pytest.mark.parametrize("path", ["generic", "tensorcore"])
def test_nan_state_poisons_its_recording_only(path):
    W = 7504
    _, m = _tc_pair("mycnn5", 3, W, 71)
    S, B = 1876, 5
    x = _records(B, 3, W + 5 * S, BF, seed=71).to(DEV)
    age = tskd_b200.synth.make_ages(B, seed=71).to(DEV)
    st = _state(B, seed=71)
    clean, sclean = m.predict_record(x, S, age, path=path, mode="sequence", state=st, return_state=True)
    bad = st.clone()
    bad[2, 1, 0, 5] = float("nan")                                       # c of layer 1, one unit
    out, so = m.predict_record(x, S, age, path=path, mode="sequence", state=bad, return_state=True)
    assert torch.isnan(out[2]).all() and torch.isnan(so[2]).any()
    keep = [0, 1, 3, 4]
    assert torch.equal(out[keep], clean[keep]) and torch.equal(so[keep], sclean[keep])


# ------------------------------------------------------------------ 4. refusals before any launch
def test_refusals():
    W, S = 7504, 752
    _, m = _tc_pair("mycnn5", 3, W, 95)
    x = _records(2, 3, W + 2 * S, BF, seed=95).to(DEV)
    age = tskd_b200.synth.make_ages(2, seed=95).to(DEV)
    good, sgood = m.predict_record(x, S, age, mode="sequence", state=_state(2, 95), return_state=True)
    with pytest.raises(ValueError, match="sequence"):
        m.predict_record(x, S, age, state=_state(2, 95))
    with pytest.raises(ValueError, match="sequence"):
        m.predict_record(x, S, age, mode="independent", return_state=True)
    for bad in (torch.zeros(3, 2, 2, 16), torch.zeros(2, 64), torch.zeros(2, 2, 2, 16, dtype=torch.int32), [0.0] * 128):
        with pytest.raises(ValueError, match="state"):
            m.predict_record(x, S, age, mode="sequence", state=bad)
    lib, h = m._ensure_handle()
    N = x.shape[2]
    st = torch.cuda.current_stream().cuda_stream
    need = int(lib.b2cnn_record_workspace_bytes_ex(h, 2, N, N, S, capi.DTYPE_BF16, capi.PATH_TENSORCORE, capi.MODE_SEQUENCE))
    ws = torch.empty(need, dtype=torch.uint8, device=DEV)
    out = torch.full((2, 3), 7.0, device=DEV)
    sin, sout = _state(2, 95), torch.full((2, 2, 2, 16), 7.0, device=DEV)

    def call(mode, n=need, dtype=capi.DTYPE_BF16, s_out=None):
        return lib.b2cnn_score_record_state(h, x.data_ptr(), dtype, 2, N, N, S, capi.PATH_TENSORCORE, mode, age.data_ptr(), 2, 0,
                                            out.data_ptr(), sin.data_ptr(), (sout if s_out is None else s_out).data_ptr(),
                                            ws.data_ptr(), n, st)
    for bad in (capi.MODE_INDEPENDENT, 2, -1):
        assert call(bad) == capi.EINVAL and "mode" in capi.last_error()
    for alias in (sin, sin[1:]):                                        # one buffer for both, or overlapping rows
        assert call(capi.MODE_SEQUENCE, s_out=alias) == capi.EINVAL and "overlap" in capi.last_error()
    assert call(capi.MODE_SEQUENCE, n=need - 256) == capi.ESTATE
    assert call(capi.MODE_SEQUENCE, dtype=7) == capi.EINVAL
    torch.cuda.synchronize()
    assert (out == 7.0).all() and (sout == 7.0).all() and torch.equal(sin, _state(2, 95))   # nothing ran
    assert call(capi.MODE_SEQUENCE) == 0
    torch.cuda.synchronize()
    assert torch.equal(out, good) and torch.equal(sout, sgood)


# ------------------------------------------------------------------ 5. launch lists
# One process per call, each with a session of torch kernels alone before the session it reports, as
# tests/test_gpu_record_sequence.py profiles.  A profiler session can come back incomplete -- that file's own check has
# returned an empty session for a call that launches six kernels -- so the reported session brackets the call with torch
# kernels (two before, two after) and counts only when all four were recorded; an incomplete session is the
# instrument failing, not the library, and is taken again (at most five times).
_LAUNCH_LIST = r"""
import collections, json, sys
import torch
import tskd_b200
from oracle import mycnn_torch as O
from torch.profiler import ProfilerActivity, profile

def session(fn):
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        torch.ones(1, device=dev).add_(1)
        torch.cuda.synchronize()
        fn()
        torch.cuda.synchronize()
        torch.full((1,), 2.0, device=dev).mul_(3)
        torch.cuda.synchronize()
    ev = [e.name for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA]
    lib = collections.Counter(n for n in ev if "b2cnn::" in n or n.startswith("Memset"))
    markers = sum(1 for n in ev if "b2cnn::" not in n and not n.startswith("Memset") and not n.startswith("Memcpy"))
    return lib, markers

def kernels(fn):
    for _ in range(5):
        lib, markers = session(fn)
        if markers >= 4:
            return lib
    raise SystemExit("the profiler recorded no complete session in five")

path, which, W, S = sys.argv[1], sys.argv[2], 7504, 752
dev = torch.device("cuda", 0)
ref = O.make_ref(O.stretched(O.ARCH_MYCNN5, 3, W), seed=91)
m = tskd_b200.B200MyCNN(tskd_b200.ARCH_PRESETS["mycnn5"].with_shape(3, W), has_out12=ref.arch.has_out12).to(dev)
m.load_state_dict(ref.state_dict())
x = tskd_b200.synth.make_windows(3, 3, W + 9 * S, "normal", seed=91, dtype=torch.bfloat16).to(dev)
age = torch.tensor([60.0], device=dev)
st = torch.zeros(3, 2, 2, 16, device=dev)
call = {"ex": lambda: m.predict_record(x, S, age, path=path, mode="sequence"),
        "state": lambda: m.predict_record(x, S, age, path=path, mode="sequence", state=st, return_state=True),
        "empty": lambda: m.predict_record(x[:, :, :W - 4], S, age, path=path, mode="sequence", state=st, return_state=True)}[which]
call()                                                                 # warm-up: attributes, lazy module loads
session(lambda: None)                                                 # profiler warm-up, torch kernels only
print(json.dumps(kernels(call)))
"""


def _kernels(path, which):
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    env = dict(os.environ, PYTHONPATH=os.pathsep.join([root] + [p for p in [os.environ.get("PYTHONPATH")] if p]))
    cmd = [sys.executable] + (["-s"] if sys.flags.no_user_site else []) + ["-c", _LAUNCH_LIST, path, which]
    r = subprocess.run(cmd, capture_output=True, text=True, env=env, cwd=root, timeout=600)
    assert r.returncode == 0, r.stderr[-3000:]
    return collections.Counter(json.loads(r.stdout.strip().splitlines()[-1]))


@pytest.mark.parametrize("path", ["tensorcore", "generic"])
def test_launch_list(path):
    res = {which: _kernels(path, which) for which in ("ex", "state", "empty")}
    # the same kernels, the scan's instance with the state in two pointers in place of the stateless one
    assert any("head_sequence_kernel<false>" in k for k in res["ex"]), res
    assert any("head_sequence_kernel<true>" in k for k in res["state"]), res
    assert collections.Counter({k.replace("head_sequence_kernel<true>", "head_sequence_kernel<false>"): n
                                for k, n in res["state"].items()}) == res["ex"], res
    assert not any("b2cnn::" in k for k in res["empty"]), res          # n_w = 0: no kernel of the library


# ------------------------------------------------------------------ 6. warm-started admission
def _pushes(sc, x, S, age):
    return [sc.push(x[:, :, i:i + S], age=age) for i in range(0, x.shape[2] - S + 1, S)]


def _warm_case(m, path, dtype, T, S, J=6, P=3, p=1, seed=0):
    """Scorers `sc` and `twin` of P patients; after n_pre pushes, patient p is admitted in both from a stay of T samples
    (history = its last W samples; `sc` with the backtest's state, `twin` without), then J pushes.  Returns the stay with
    the pushes appended, the offset o = (T - W) % S, p's scores after each of the J pushes in `sc`, the two scorers'
    outputs and the state given."""
    W, C = m.arch.window, m.arch.in_channels
    stay = _records(1, C, T + J * S, dtype, seed=seed).to(DEV)
    n_pre = max(1, -(-W // S)) + 1
    others = _records(P, C, (n_pre + J) * S, dtype, seed=seed + 1).to(DEV)
    age = tskd_b200.synth.make_ages(P, seed=seed).to(DEV)
    o = (T - W) % S
    _, lstm = m.predict_record(stay[:, :, o:T], S, age[p:p + 1], path=path, mode="sequence", return_state=True)
    sc = tskd_b200.SlidingScorer(m, P, S, dtype=dtype, path=path, mode="sequence")
    twin = tskd_b200.SlidingScorer(m, P, S, dtype=dtype, path=path, mode="sequence")
    _pushes(sc, others[:, :, :n_pre * S], S, age)
    _pushes(twin, others[:, :, :n_pre * S], S, age)
    sc.admit([p], stay[:, :, T - W:T], lstm=lstm)
    twin.admit([p], stay[:, :, T - W:T])
    assert torch.equal(sc.export([p])["lstm"], lstm)                  # the given rows, as written
    assert torch.equal(twin.export([p])["lstm"], torch.zeros_like(lstm))
    live = others[:, :, n_pre * S:].clone()
    live[p] = stay[0, :, T:]
    outs, touts = _pushes(sc, live, S, age), _pushes(twin, live, S, age)
    got = torch.stack([out[p] for out in outs])
    return stay, o, age, got, outs, touts, lstm


@pytest.mark.parametrize("T", ["W", "W+7S+4", "10W"])
@pytest.mark.parametrize("dtype", [F32, BF], ids=["f32", "bf16"])
def test_warm_start_recipe_generic(T, dtype):
    _, m = _golden(5)
    W, S, p = 120, 12, 1
    T = {"W": W, "W+7S+4": W + 7 * S + 4, "10W": 10 * W}[T]
    stay, o, age, got, outs, touts, _ = _warm_case(m, "generic", dtype, T, S, seed=T)
    full = m.predict_record(stay[:, :, o:], S, age[p:p + 1], path="generic", mode="sequence")[0]
    first = (T - W - o) // S + 1                                        # the column of the window after the first push
    assert _same(got, full[first:first + got.shape[0]]), T
    for out, tout in zip(outs, touts):                                  # the other patients: the twin's scores
        assert _same(out[[0, 2]], tout[[0, 2]])


@pytest.mark.parametrize("T", ["W", "W+7S+4", "10W"])
def test_warm_start_recipe_tensorcore(T):
    W, S, p = 7504, 752, 1
    ref, m = _tc_pair("mycnn5", 3, W, 81)
    T = {"W": W, "W+7S+4": W + 7 * S + 4, "10W": 10 * W}[T]
    stay, o, age, got, outs, touts, _ = _warm_case(m, "tensorcore", BF, T, S, seed=T)
    first = (T - W - o) // S + 1
    (t, _), (t32, _) = _truth(ref, stay[:, :, o:], S, age[p:p + 1])
    J = got.shape[0]
    _check([("warm", got, t[0, first:first + J], t32[0, first:first + J], BETA_TC_SEQ)])
    for out, tout in zip(outs, touts):
        assert torch.equal(out[[0, 2]], tout[[0, 2]])


@pytest.mark.parametrize("path", ["generic", "tensorcore"])
def test_short_history_arbitrary_state(path):
    """H < W and a random lstm: the first live step starts from it (float64), and on the generic path the scores are
    predict_record's from that state over the stream since admission"""
    if path == "generic":
        ref, m = _golden(5)
        W, S, dtype, beta = 120, 12, F32, BETA
    else:
        ref, m = _tc_pair("mycnn5", 3, 7504, 83)
        W, S, dtype, beta = 7504, 752, BF, BETA_TC_SEQ
    C, P, p, J = m.arch.in_channels, 4, 2, 5
    H = W - 2 * S - 4
    s0 = H + -(-(W - H) // S) * S                                       # samples_seen at the first scored push
    n = (s0 - H) // S + J - 1                                           # pushes after admission
    hist = _records(1, C, H, dtype, seed=83).to(DEV)
    xs = _records(P, C, (n + 1) * S, dtype, seed=84).to(DEV)
    age = tskd_b200.synth.make_ages(P, seed=83).to(DEV)
    lstm = _state(1, seed=83)
    sc = tskd_b200.SlidingScorer(m, P, S, dtype=dtype, path=path, mode="sequence")
    twin = tskd_b200.SlidingScorer(m, P, S, dtype=dtype, path=path, mode="sequence")
    for s in (sc, twin):
        s.push(xs[:, :, :S], age=age)
        s.admit([p], hist, lstm=lstm if s is sc else None)
    outs = _pushes(sc, xs[:, :, S:], S, age)
    touts = _pushes(twin, xs[:, :, S:], S, age)
    got = torch.stack([o[p] for o in outs if o is not None and not torch.isnan(o[p])])
    assert got.shape == (J,)
    stream = torch.cat([hist, xs[p:p + 1, :, S:]], dim=2)
    (t, ts), (t32, _) = _truth(ref, stream[:, :, s0 - W:], S, age[p:p + 1], lstm.cpu())
    _check([("short-history", got, t[0], t32[0], beta)])
    if path == "generic":
        want = m.predict_record(stream[:, :, s0 - W:], S, age[p:p + 1], path="generic", mode="sequence", state=lstm)[0]
        assert _same(got, want)
    for o, to in zip(outs, touts):
        if o is not None:
            keep = [q for q in range(P) if q != p]
            assert _same(o[keep], to[keep])


def test_admit_refusals():
    _, m = _golden(5)
    S, P = 12, 3
    x = _records(P, 10, 12 * S, F32, seed=9).to(DEV)
    age = torch.tensor([60.0], device=DEV)
    ind = tskd_b200.SlidingScorer(m, P, S, dtype=F32, path="generic", mode="independent")
    seq = tskd_b200.SlidingScorer(m, P, S, dtype=F32, path="generic", mode="sequence")
    ind_twin = tskd_b200.SlidingScorer(m, P, S, dtype=F32, path="generic", mode="independent")
    for s in (ind, seq, ind_twin):
        _pushes(s, x[:, :, :11 * S], S, age)
    before, seq_before = ind.export([0, 1, 2]), seq.export([0, 1, 2])
    with pytest.raises(ValueError, match="sequence-mode"):
        ind.admit([1], x[1:2, :, :120], lstm=torch.zeros(1, 2, 2, 16, device=DEV))
    for bad in (torch.zeros(2, 2, 2, 16), torch.zeros(1, 64), torch.zeros(1, 2, 2, 16, dtype=torch.int64), "zeros"):
        with pytest.raises(ValueError, match="lstm"):
            seq.admit([1], x[1:2, :, :120], lstm=bad)
    after, seq_after = ind.export([0, 1, 2]), seq.export([0, 1, 2])
    for k in before:
        assert (torch.equal(before[k], after[k]) if torch.is_tensor(before[k]) else before[k] == after[k]), k
    for k in seq_before:
        assert (torch.equal(seq_before[k], seq_after[k]) if torch.is_tensor(seq_before[k]) else seq_before[k] == seq_after[k]), k
    # the C ABI refuses an lstm on an independent scorer before any launch
    arr = (ctypes.c_int32 * 1)(1)
    lstm = torch.zeros(1, 2, 2, 16, device=DEV)
    nbytes = int(ind._lib.b2cnn_slide_admit_workspace_bytes(ind._s, 1, 0))
    ws = torch.empty(max(nbytes, 1), dtype=torch.uint8, device=DEV)
    rc = ind._lib.b2cnn_slide_admit_ex(ind._s, arr, 1, None, 0, 0, capi.DTYPE_F32, lstm.data_ptr(), ws.data_ptr(), nbytes,
                                       torch.cuda.current_stream().cuda_stream)
    assert rc == capi.EINVAL and "independent" in capi.last_error()
    assert torch.equal(ind.samples_seen, ind_twin.samples_seen)
    assert _same(ind.push(x[:, :, 11 * S:], age=age), ind_twin.push(x[:, :, 11 * S:], age=age))


# ------------------------------------------------------------------ 7. training on chunks of a recording
from dataclasses import replace                                            # noqa: E402

from oracle import mycnn_torch as O                                        # noqa: E402
from oracle.record_state_ref import train_record_state_reference           # noqa: E402
from oracle.train_ref import MaskDropout                                   # noqa: E402
from tskd_b200.arch import BLOB_KEYS                                       # noqa: E402
from tskd_b200.trainer import B200Trainer                                  # noqa: E402

CONV = ("conv1.weight", "conv1.bias", "conv2.weight", "conv2.bias")
HEAD = [k for k in BLOB_KEYS if k not in CONV]
# (kind, C, W, S, n_w, counts or None) -- counts None: every window of the 3 recordings
TRAIN_CASES = {"m5-s72": ("mycnn5", 10, 120, 72, 8, None), "m5-w7504": ("mycnn5", 3, 7504, 3752, 6, None)}


def _train_pair(kind, C, W, seed=0, trainable=True):
    oarch = O.stretched(O.ARCHS[kind], C, W)
    ref = O.make_ref(oarch, seed=seed)
    ref.dropout = MaskDropout()
    ref.train()
    arch = replace(tskd_b200.ARCH_PRESETS[kind].with_shape(C, W), age_coef=oarch.age_coef)
    cls = tskd_b200.B200TrainableMyCNN if trainable else tskd_b200.B200MyCNN
    m = cls(arch, has_out12=oarch.has_out12).to(DEV)
    m.load_state_dict({k: v for k, v in ref.state_dict().items() if not k.startswith("dropout")})
    return ref, m


def _train_data(arch, B, N, M, seed, p=0.1):
    g = torch.Generator().manual_seed(seed)
    rec = torch.randn(B, arch.in_channels, N, generator=g)
    age = torch.rand(B, generator=g) * 60 + 20
    y = (torch.rand(M, generator=g) > 0.5).float()
    ra = arch.with_shape(arch.in_channels, N)
    m1 = torch.bernoulli(torch.full((B, 4, ra.p1), 1 - p), generator=g) / (1 - p)
    m2 = torch.bernoulli(torch.full((B, ra.l_out), 1 - p), generator=g) / (1 - p)
    s0 = 0.5 * torch.randn(B, 2, 2, 16, generator=g)
    return rec, age, y, m1, m2, s0


def _chunk_masks(arch, m1, m2, s0, n):
    """the recording's masks for the chunk of n samples starting at sample s0"""
    ra = arch.with_shape(arch.in_channels, n)
    a, b = s0 // arch.pool_s, s0 // arch.pool_s ** 2
    return m1[:, :, a:a + ra.p1].contiguous(), m2[:, b:b + ra.l_out].contiguous()


def _params(m):
    named = dict(m.named_parameters())
    return [named[k] for k in BLOB_KEYS]


def _grads(m):
    named = dict(m.named_parameters())
    out = {k: named[k].grad.clone() for k in BLOB_KEYS}
    for q in m.parameters():
        q.grad = None
    return out


def _chunked_forward(m, rec, S, age, k, m1, m2, state, counts):
    """mycnn_train_record_forward over rec cut at window k, chained through the state: (z recording-major, state_out)"""
    arch = m.arch
    W, N = arch.window, rec.shape[2]
    nA = (k - 1) * S + W
    a1, a2 = _chunk_masks(arch, m1, m2, 0, nA)
    b1, b2 = _chunk_masks(arch, m1, m2, k * S, N - k * S)
    ca = [min(c, k) for c in counts]
    cb = [max(c - k, 0) for c in counts]
    za, sa = tskd_b200.mycnn_train_record_forward(rec[:, :, :nA], S, age, _params(m), arch, "sequence", a1, a2, ca, state=state,
                                                  return_state=True)
    zb, sb = tskd_b200.mycnn_train_record_forward(rec[:, :, k * S:], S, age, _params(m), arch, "sequence", b1, b2, cb, state=sa,
                                                  return_state=True)
    # each recording's windows from chunk A, then from chunk B
    parts, oa, ob = [], 0, 0
    for x, y in zip(ca, cb):
        parts += [za[oa:oa + x], zb[ob:ob + y]]
        oa, ob = oa + x, ob + y
    return torch.cat(parts), sb


# The existing training grants: tests/test_gpu_train_record.py's LONG_SUM_BETA for a long window's conv weight gradients
# and d records, and tests/test_gpu_train_long.py's one allowance, a conv layer's bias gradient judged together with its
# weight gradient as one tensor (a bias gradient is one long, sometimes cancelling, sum of the terms its weights' sums hold)
LONG_SUM_BETA = {k: 4e-6 for k in ("conv1.weight+bias", "conv2.weight+bias", "drecords")}


def _grad_pairs(g, drec, truth, ref32, W):
    """check_elems pairs of every parameter gradient and d records against the float64 truth, with ref32 the float32
    reference module's, at the grants above"""
    beta = LONG_SUM_BETA if W > 1000 else {}
    cat = (lambda d, n: torch.cat([d[n + ".weight"].reshape(-1).double().cpu(), d[n + ".bias"].reshape(-1).double().cpu()]))
    pairs = [(k, g[k], truth["grads"][k], ref32["grads"][k], BETA) for k in HEAD]
    pairs += [(n + ".weight+bias", cat(g, n), cat(truth["grads"], n), cat(ref32["grads"], n), beta.get(n + ".weight+bias", BETA))
              for n in ("conv1", "conv2")]
    pairs.append(("drecords", drec, truth["drecords"], ref32["drecords"], beta.get("drecords", BETA)))
    return pairs


@pytest.mark.parametrize("name", sorted(TRAIN_CASES))
def test_chained_forward_record_against_float64(name):
    """two chunks chained through a differentiable state, one backward: every gradient against one float64 pass over the
    whole recordings; the logits and the final state are the unsplit call's bits"""
    kind, C, W, S, n_w, _ = TRAIN_CASES[name]
    ref, m = _train_pair(kind, C, W)
    B, N = 3, W + (n_w - 1) * S + 17
    M = B * n_w
    rec, age, _, m1, m2, s0 = _train_data(m.arch, B, N, M, seed=11)
    r = torch.randn(M, generator=torch.Generator().manual_seed(12))
    ds = torch.randn(B, 2, 2, 16, generator=torch.Generator().manual_seed(13))
    truth = train_record_state_reference(ref, rec, S, age, [n_w] * B, s0, m1, m2, dz=r, dstate=ds)
    ref32 = train_record_state_reference(ref, rec, S, age, [n_w] * B, s0, m1, m2, dz=r, dstate=ds, dtype=torch.float32)
    d1, d2 = m1.to(DEV), m2.to(DEV)

    def run(chained, k=0):
        x = rec.to(DEV).requires_grad_()
        a = age.to(DEV).requires_grad_()
        s = s0.to(DEV).requires_grad_()
        if chained:
            z, so = _chunked_forward(m, x, S, a, k, d1, d2, s, [n_w] * B)
        else:
            z, so = tskd_b200.mycnn_train_record_forward(x, S, a, _params(m), m.arch, "sequence", d1, d2, state=s, return_state=True)
        ((z * r.to(DEV)).sum() + (so * ds.to(DEV)).sum()).backward()
        return z.detach(), so.detach(), _grads(m), x.grad, a.grad, s.grad

    one = run(False)
    for k in (1, n_w // 2, n_w - 1):
        z, so, g, drec, dage, dstate = run(True, k)
        assert torch.equal(z, one[0]) and torch.equal(so, one[1]), k
        _check(_grad_pairs(g, drec, truth, ref32, W) + [("dage", dage, truth["dage"], ref32["dage"], BETA),
                                                         ("dstate", dstate, truth["dstate"], ref32["dstate"], BETA)])
    _check([("z", one[0], truth["z"], ref32["z"], BETA), ("state", one[1], truth["state"], ref32["state"], BETA)])


def test_loss_on_the_final_state_alone():
    ref, m = _train_pair("mycnn5", 10, 120)
    S, n_w, B = 72, 6, 3
    N = 120 + (n_w - 1) * S
    rec, age, _, m1, m2, s0 = _train_data(m.arch, B, N, B * n_w, seed=21)
    ds = torch.randn(B, 2, 2, 16, generator=torch.Generator().manual_seed(22))
    truth = train_record_state_reference(ref, rec, S, age, [n_w] * B, s0, m1, m2, dstate=ds)
    ref32 = train_record_state_reference(ref, rec, S, age, [n_w] * B, s0, m1, m2, dstate=ds, dtype=torch.float32)
    x, a, s = rec.to(DEV).requires_grad_(), age.to(DEV).requires_grad_(), s0.to(DEV).requires_grad_()
    _, so = _chunked_forward(m, x, S, a, 3, m1.to(DEV), m2.to(DEV), s, [n_w] * B)
    (so * ds.to(DEV)).sum().backward()
    g = _grads(m)
    pairs = [(k, g[k], truth["grads"][k], ref32["grads"][k], BETA) for k in BLOB_KEYS]
    pairs += [("drecords", x.grad, truth["drecords"], ref32["drecords"], BETA), ("dage", a.grad, truth["dage"], ref32["dage"], BETA),
              ("dstate", s.grad, truth["dstate"], ref32["dstate"], BETA)]
    _check(pairs)
    # eval mode: predict_record's state, which counts every window
    m.eval()
    with torch.no_grad():
        got = m.forward_record(x, S, a, state=s, return_state=True)
        want = m.predict_record(x, S, a, mode="sequence", state=s, return_state=True)
    assert torch.equal(got[0], want[0]) and torch.equal(got[1], want[1])
    with pytest.raises(ValueError, match="every window"):
        m.forward_record(x, S, a, window_counts=[n_w - 1] * B, state=s)


def test_zero_counts_pass_the_state_and_its_gradient():
    ref, m = _train_pair("mycnn5", 10, 120)
    S, n_w = 72, 8
    counts = [8, 0, 3, 0, 5]
    B, N = len(counts), 120 + (n_w - 1) * S + 30
    rec, age, y, m1, m2, s0 = _train_data(m.arch, B, N, sum(counts), seed=31)
    r = torch.randn(sum(counts), generator=torch.Generator().manual_seed(32))
    ds = torch.randn(B, 2, 2, 16, generator=torch.Generator().manual_seed(33))
    x, a, s = rec.to(DEV).requires_grad_(), age.to(DEV).requires_grad_(), s0.to(DEV).requires_grad_()
    z, so = tskd_b200.mycnn_train_record_forward(x, S, a, _params(m), m.arch, "sequence", m1.to(DEV), m2.to(DEV), counts, state=s,
                                                 return_state=True)
    ((z * r.to(DEV)).sum() + (so * ds.to(DEV)).sum()).backward()
    g = _grads(m)
    for b in (1, 3):
        assert torch.equal(so[b], s0[b].to(DEV)) and torch.equal(s.grad[b], ds[b].to(DEV)), b
    truth = train_record_state_reference(ref, rec, S, age, counts, s0, m1, m2, dz=r, dstate=ds)
    ref32 = train_record_state_reference(ref, rec, S, age, counts, s0, m1, m2, dz=r, dstate=ds, dtype=torch.float32)
    _check([("z", z.detach(), truth["z"], ref32["z"], BETA), ("state", so.detach(), truth["state"], ref32["state"], BETA),
            ("dstate", s.grad, truth["dstate"], ref32["dstate"], BETA)] +
           [(k, g[k], truth["grads"][k], ref32["grads"][k], BETA) for k in HEAD])
    # chained across a cut that leaves recording 2 (and the empty 1 and 3) no window in the second chunk
    x2, s2 = rec.to(DEV).requires_grad_(), s0.to(DEV).requires_grad_()
    zc, soc = _chunked_forward(m, x2, S, age.to(DEV), 4, m1.to(DEV), m2.to(DEV), s2, counts)
    assert torch.equal(zc.detach(), z.detach()) and torch.equal(soc.detach(), so.detach())
    # the fused step: the same final state, passed through for the zero counts
    _, mf = _train_pair("mycnn5", 10, 120, trainable=False)
    loss, sf = B200Trainer(mf, dropout=0.1).step_record(rec, S, age, y, window_counts=counts, masks=(m1, m2), update=False,
                                                       state=s0, return_state=True)
    assert torch.equal(sf, so.detach()) and not sf.requires_grad


@pytest.mark.parametrize("pos_weight", [None, 13.5], ids=["bce", "bce-pw"])
def test_fused_step_with_state(pos_weight):
    """step_record(state=...): TBPTT.  Its gradients and the autograd pair's (BCEWithLogitsLoss on the logits, the state
    detached) both match the float64 graph with that loss; state=None is today's step_record bit for bit"""
    ref, m = _train_pair("mycnn5", 10, 120)
    S, n_w, B = 72, 7, 3
    N = 120 + (n_w - 1) * S + 5
    M = B * n_w
    rec, age, y, m1, m2, s0 = _train_data(m.arch, B, N, M, seed=41)
    truth = train_record_state_reference(ref, rec, S, age, [n_w] * B, s0, m1, m2, target=y, pos_weight=pos_weight)
    ref32 = train_record_state_reference(ref, rec, S, age, [n_w] * B, s0, m1, m2, target=y, pos_weight=pos_weight, dtype=torch.float32)
    _, mf = _train_pair("mycnn5", 10, 120, trainable=False)
    tr = B200Trainer(mf, dropout=0.1, pos_weight=pos_weight)
    loss, so = tr.step_record(rec, S, age, y, masks=(m1, m2), update=False, state=s0, return_state=True)
    g = tr.grads()
    pairs = [(k, g[k], truth["grads"][k], ref32["grads"][k], BETA) for k in BLOB_KEYS]
    pairs += [("loss", loss.reshape(1), truth["loss"].reshape(1), ref32["loss"].reshape(1), BETA),
              ("state", so, truth["state"], ref32["state"], BETA)]
    _check(pairs)
    # the autograd pair on the same inputs and masks
    z, so2 = tskd_b200.mycnn_train_record_forward(rec.to(DEV), S, age.to(DEV), _params(m), m.arch, "sequence", m1.to(DEV), m2.to(DEV),
                                                  state=s0.to(DEV), return_state=True)
    pw = None if pos_weight is None else torch.tensor(pos_weight, device=DEV)
    torch.nn.functional.binary_cross_entropy_with_logits(z, y.to(DEV), pos_weight=pw).backward()
    ga = _grads(m)
    assert torch.equal(so2.detach(), so)
    _check([(k, ga[k], truth["grads"][k], ref32["grads"][k], BETA) for k in BLOB_KEYS])
    # state=None and return_state=False: today's call
    _, mt = _train_pair("mycnn5", 10, 120, trainable=False)
    today = B200Trainer(mt, dropout=0.1, pos_weight=pos_weight)
    want = today.step_record(rec, S, age, y, masks=(m1, m2), update=False)
    _, mn = _train_pair("mycnn5", 10, 120, trainable=False)
    none = B200Trainer(mn, dropout=0.1, pos_weight=pos_weight)
    got, sn = none.step_record(rec, S, age, y, masks=(m1, m2), update=False, return_state=True)
    assert torch.equal(got, want) and torch.equal(none._grads, today._grads)
    _, mz = _train_pair("mycnn5", 10, 120, trainable=False)
    zero = B200Trainer(mz, dropout=0.1, pos_weight=pos_weight)
    got0 = zero.step_record(rec, S, age, y, masks=(m1, m2), update=False, state=torch.zeros(B, 2, 2, 16))
    assert torch.equal(got0, want) and torch.equal(zero._grads, today._grads)


def test_tbptt_loop_updates_and_refusals():
    """a TBPTT loop over 3 chunks with Adam updates runs and carries the state; refusals before anything runs"""
    _, mf = _train_pair("mycnn5", 10, 120, trainable=False)
    S, B = 72, 2
    rec, age, y, _, _, _ = _train_data(mf.arch, B, 120 + 11 * S, B * 12, seed=51)
    tr = B200Trainer(mf, dropout=0.1)
    state, losses = None, []
    for c in range(3):
        chunk = rec[:, :, c * 4 * S:c * 4 * S + 3 * S + 120]
        loss, state = tr.step_record(chunk, S, age, y[:B * 4], state=state, return_state=True)
        losses.append(float(loss))
    assert tr.steps == 3 and all(v == v for v in losses) and state.shape == (B, 2, 2, 16)
    before = tr._params.clone()
    ind = B200Trainer(mf, dropout=0.1, mode="independent")
    with pytest.raises(ValueError, match="sequence"):
        ind.step_record(rec, S, age, y, state=state)
    with pytest.raises(ValueError, match="state"):
        tr.step_record(rec, S, age, y, state=torch.zeros(3, 2, 2, 16))
    assert torch.equal(tr._params, before) and tr.steps == 3
    _, m = _train_pair("mycnn5", 10, 120)
    with pytest.raises(ValueError, match="sequence"):
        tskd_b200.mycnn_train_record_forward(rec.to(DEV), S, age.to(DEV), _params(m), m.arch, "independent", return_state=True)
    # the C ABI refuses independent mode before any CUDA call
    lib = capi.load_library()
    cfg = capi.make_config(m.arch, 0)
    cts = (ctypes.c_int64 * B)(12, 12)
    head = (ctypes.byref(cfg), None, None, B, rec.shape[2], S, cts, capi.MODE_INDEPENDENT)
    assert lib.b2cnn_train_forward_record_state(*head, *(None,) * 7, 0, None) == capi.EINVAL
    assert "mode" in capi.last_error()
    assert lib.b2cnn_train_backward_record_state(*head, *(None,) * 10, 0, None, 0, None) == capi.EINVAL
    assert "mode" in capi.last_error()
