"""GPU: predict_record(mode="sequence") and b2cnn_score_record_ex -- each recording's windows scored as one LSTM sequence,
the reference's utils.run_model per recording.

- the golden of the unmodified utils.run_model (tests/golden/run_model_record.npz), with create_batch's dropped window;
- generic path: every row bit-identical (NaN for NaN) to predict(windows_b, age_b, mode="sequence") with path="generic"
  and small_kernel=0, across models, strides, batch sizes, window counts and views;
- tensor-core path: every element judged with check_elems against the float64 reference at BETA_TC_SEQ (below),
  including a 24 h recording (1431 windows) whose float64 features are computed once on the recording's lattice;
- NaN and +-inf, causality (prefixes), independence of the other recordings, repeatability, the unchanged independent
  mode, a launch list that does not depend on B, N or S, and errors raised before any launch."""
import collections
import copy
import json
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

import tskd_b200
from conftest import GOLDEN
from oracle.infer_ref import infer_reference
from oracle.train_ref import BETA, check_elems
from test_gpu_record import _check, _records, _tc_pair, _wins
from test_gpu_slide_generic import _golden, _pair as _generic_pair, _same
from tskd_b200 import capi

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
BF, F32 = torch.bfloat16, torch.float32
# Tensor-core sequence logits.  Each window's tensor-core features carry their own error (scored independently, the same
# path passes at BETA in tests/test_gpu_record.py); the scan feeds it into the LSTM state, and later windows of the
# recording inherit it.  Measured worst on one H100 80GB HBM3 (700 W): 1.36e-6 on the 24 h recording (1431 steps) and
# 1.15e-6 for MyCNN3 fp32 at S = 752 over 130 recordings; every other tensor-core case, and every generic-path case,
# within 2^-20.
BETA_TC_SEQ = 2e-6


def _n_w(N, W, S):
    return (N - W) // S + 1 if N >= W else 0


def _age_of(age, b):
    return age.reshape(-1)[0 if age.numel() == 1 else b]


def _truth(ref, x, S, age, prob=False):
    """(float64, float32) references of every recording's windows scanned as one sequence, [B, n_w] each"""
    W = ref.arch.window
    t, t32 = [], []
    for b in range(x.shape[0]):
        win = _wins(x[b:b + 1].cpu(), W, S)
        a = _age_of(age, b).reshape(1).cpu()
        t.append(infer_reference(ref, win, a, "sequence")["z"])
        t32.append(infer_reference(ref, win, a, "sequence", dtype=torch.float32)["z"])
    t, t32 = torch.stack(t), torch.stack(t32)
    return (torch.sigmoid(t), torch.sigmoid(t32)) if prob else (t, t32)


# ------------------------------------------------------------------ 1. the golden of utils.run_model
@pytest.mark.parametrize("tag", ["a", "b", "nan"])
def test_run_model_golden(tag):
    g = np.load(os.path.join(GOLDEN, "run_model_record.npz"))
    ref, m = _golden(5)
    frame = torch.from_numpy(g[f"frame_{tag}"]).T.contiguous()       # [10, N]
    x = torch.stack([frame, frame]).to(DEV)                           # one recording at each golden age
    ages = torch.from_numpy(g["ages"]).float().to(DEV)
    out = m.predict_record(x, 120, ages, mode="sequence", return_prob=True)
    gold = torch.from_numpy(g[f"prob_{tag}"])
    N = frame.shape[1]
    assert out.shape == (2, _n_w(N, 120, 120))
    if (N - 120) % 120 == 0:                                          # create_batch drops the last full window
        assert out.shape[1] == gold.shape[1] + 1
        out = out[:, :-1]
    truth, _ = _truth(ref, x[:, :, :N - (120 if (N - 120) % 120 == 0 else 0)], 120, ages, prob=True)
    _check([(f"run_model-{tag}", out, truth[:, :gold.shape[1]], gold, BETA)])
    if tag == "nan":                                                  # the NaN at row 6000 is in window 50
        assert torch.isfinite(out[:, :50]).all() and torch.isnan(out[:, 50:]).all()


# ------------------------------------------------------------------ 2. generic path, bit for bit
def _generic_same(m, x, S, age, prob=False):
    W = m.arch.window
    out = m.predict_record(x, S, age, return_prob=prob, path="generic", mode="sequence")
    n_w = _n_w(x.shape[2], W, S)
    assert tuple(out.shape) == (x.shape[0], n_w) and m.last_path == "generic"
    for b in range(x.shape[0]):
        want = m.predict(_wins(x[b:b + 1], W, S), _age_of(age, b).reshape(1), mode="sequence", return_prob=prob)
        assert _same(out[b], want), b
    return out


@pytest.mark.parametrize("dtype", [F32, BF], ids=["f32", "bf16"])
@pytest.mark.parametrize("S", [120, 72, 12])
def test_generic_golden_bit_identical(dtype, S):
    ref, m = _golden(5)
    x = _records(3, 10, 120 + 9 * S + 5, dtype, seed=S).to(DEV)
    age = tskd_b200.synth.make_ages(3, seed=S).to(DEV)
    out = _generic_same(m, x, S, age)
    _generic_same(m, x, S, age, prob=True)
    t, t32 = _truth(ref, x, S, age)
    _check([(f"golden-S{S}", out, t, t32, BETA)])


@pytest.mark.parametrize("case", ["c10-relu-affine", "pool44"])
def test_generic_models(case):
    if case == "c10-relu-affine":
        geo, act, aff_seed, S, N = (10, 10, 5, 3, 2, 200), "relu", 7, 24, 200 + 11 * 24 + 3
    else:
        geo, act, aff_seed, S, N = (3, 5, 5, 4, 4, 250), "tanh", None, 32, 250 + 7 * 32 + 9   # W % 16 != 0
    _, m, _ = _generic_pair(geo, act=act, aff_seed=aff_seed, seed=11)
    for dtype in (F32, BF):
        x = _records(4, geo[0], N, dtype, seed=5).to(DEV)
        _generic_same(m, x, S, tskd_b200.synth.make_ages(4, seed=5).to(DEV))
        _generic_same(m, x, S, torch.tensor([70.0], device=DEV))


@pytest.mark.parametrize("B,n_w", [(1, 1), (3, 2), (130, 4), (1, 1101), (3, 1001)])
def test_generic_batch_and_window_counts(B, n_w):
    _, m = _golden(5)
    S = 12
    x = _records(B, 10, 120 + (n_w - 1) * S + 7, F32, seed=B + n_w).to(DEV)
    out = _generic_same(m, x, S, tskd_b200.synth.make_ages(B, seed=B).to(DEV))
    assert out.shape == (B, n_w)


def test_generic_views():
    _, m = _golden(5)
    S = 36
    N = 120 + 6 * S
    base = _records(3, 10, N + 7, F32, seed=9).to(DEV)
    age = tskd_b200.synth.make_ages(3, seed=9).to(DEV)
    contiguous = _generic_same(m, base[:, :, :N].contiguous(), S, age)
    assert _same(_generic_same(m, base[:, :, :N], S, age), contiguous)           # row-padded view
    _generic_same(m, base[:, :, 1:N + 1], S, age)                               # one-sample offset view
    _generic_same(m, base[1:2, :, 3:N + 3], S, age[1:2])


# ------------------------------------------------------------------ 3. tensor-core path against float64
TC_CASES = {
    "m5-bf16-w7504-s752-b3": ("mycnn5", 3, BF, 7504, 752, 3, 7504 + 10 * 752 + 5),
    "m5-bf16-w7504-s752-b1": ("mycnn5", 3, BF, 7504, 752, 1, 7504 + 40 * 752),
    "m5-bf16-w7504-s7504-b130": ("mycnn5", 3, BF, 7504, 7504, 130, 7504 + 4 * 7504),
    "m5-bf16-w7504-s9000-b257": ("mycnn5", 3, BF, 7504, 9000, 257, 7504 + 2 * 9000 + 7),
    "m3-f32-w7502-s7500-b3": ("mycnn3", 1, F32, 7502, 7500, 3, 7502 + 6 * 7500),
    "m3-f32-w7502-s752-b130": ("mycnn3", 1, F32, 7502, 752, 130, 7502 + 8 * 752 + 1),
    "m3-f32-w7502-s9000-b257": ("mycnn3", 1, F32, 7502, 9000, 257, 7502 + 9000 + 3),
    "m3-f32-w7502-s752-b1": ("mycnn3", 1, F32, 7502, 752, 1, 7502 + 30 * 752),
}


@pytest.mark.parametrize("name", sorted(TC_CASES))
def test_tensorcore_against_float64(name):
    kind, C, dtype, W, S, B, N = TC_CASES[name]
    seed = 400 + sorted(TC_CASES).index(name)
    ref, m = _tc_pair(kind, C, W, seed)
    x = _records(B, C, N, dtype, seed=seed).to(DEV)
    age = tskd_b200.synth.make_ages(B, seed=seed).to(DEV)
    out = m.predict_record(x, S, age, path="tensorcore", mode="sequence")
    assert m.last_path == "tensorcore" and tuple(out.shape) == (B, _n_w(N, W, S))
    assert torch.equal(m.predict_record(x, S, age, mode="sequence"), out)      # auto takes the tensor cores here
    t, t32 = _truth(ref, x, S, age)
    _check([(name, out, t, t32, BETA_TC_SEQ)])


@torch.no_grad()
def test_long_recording():
    """one 24 h recording at 125 Hz: 1431 windows, one scan; the float64 features are computed once on the recording's
    lattice and window w is features w S / 4 .. w S / 4 + L - 1 of it"""
    W, S, N = 75000, 7500, 10_800_000
    ref, m = _tc_pair("mycnn5", 3, W, 41)
    x = _records(1, 3, N, BF, seed=41)
    age = torch.tensor([63.0])
    out = m.predict_record(x.to(DEV), S, age.to(DEV), mode="sequence")
    n_w = _n_w(N, W, S)
    assert tuple(out.shape) == (1, n_w) == (1, 1431) and m.last_path == "tensorcore"
    zs = []
    for dtype in (torch.float64, torch.float32):
        r = copy.deepcopy(ref).to(dtype).eval()
        v = r.pool(torch.tanh(r.conv2(r.pool(torch.tanh(r.conv1(x.to(dtype)))))))   # [1, 1, L_N]
        f = v.reshape(-1).unfold(0, r.MAGICNUM, S // 4)                              # [n_w, L]
        assert f.shape[0] == n_w
        h, _ = r.lstm(f)
        zs.append((r.out(h) * torch.relu(age.to(dtype).unsqueeze(1) * r.arch.age_coef + 1)).squeeze(1))
    _check([("24h", out[0], zs[0], zs[1], BETA_TC_SEQ)])


# ------------------------------------------------------------------ 4. NaN and +-inf
def _first_window(pos, W, S):
    """the first window holding sample pos"""
    return max(0, -(-(pos - W + 1) // S))


def test_nan_inf_both_paths():
    W, S = 7504, 752
    N = W + 30 * S
    ref, m = _tc_pair("mycnn5", 3, W, 51)
    clean = _records(6, 3, N, BF, seed=51)
    L_N = (N - 24) // 4 + 1
    nr = (L_N + 4095) // 4096
    fold = 4 * (((L_N + nr - 1) // nr + 7) // 8 * 8)                   # first sample of the second folded row
    assert nr >= 2
    x = clean.clone()
    nan_at = {0: 0, 2: fold - 2, 3: N - 5}                             # the first sample, a fold boundary, the last R samples
    x[0, 0, 0] = float("nan")
    x[1, 1, N // 2] = float("inf")                                      # mid-recording
    x[1, 2, fold + 3] = -float("inf")                                   # in the halo both folded rows read
    x[2, 0, fold - 2] = float("nan")
    x[3, 1, N - 5] = float("nan")
    age = tskd_b200.synth.make_ages(6, seed=51).to(DEV)
    t, t32 = _truth(ref, x, S, age)
    for path in ("tensorcore", "generic"):
        out = m.predict_record(x.to(DEV), S, age, path=path, mode="sequence")
        base = m.predict_record(clean.to(DEV), S, age, path=path, mode="sequence")
        assert m.last_path == path
        for b, pos in nan_at.items():
            w0 = _first_window(pos, W, S)
            assert torch.isfinite(out[b, :w0]).all() and torch.isnan(out[b, w0:]).all(), (path, b, w0)
            if path == "generic":                                       # the features before the NaN are the same
                assert torch.equal(out[b, :w0], base[b, :w0]), (path, b)
        assert torch.isfinite(out[1]).all() == torch.isfinite(t[1]).all()
        assert torch.equal(out[4:], base[4:]), path                    # the clean recordings are untouched
        _check([(f"nan-inf-{path}", out, t, t32, BETA_TC_SEQ if path == "tensorcore" else BETA)])


# ------------------------------------------------------------------ 5. causality and independence
def test_causal_and_independent():
    W, S = 7504, 1876
    ref, m = _tc_pair("mycnn5", 3, W, 61)
    N = W + 9 * S + 2
    x = _records(257, 3, N, BF, seed=61).to(DEV)
    age = tskd_b200.synth.make_ages(257, seed=61).to(DEV)
    for path in ("tensorcore", "generic"):
        full = m.predict_record(x, S, age, path=path, mode="sequence")
        alone = m.predict_record(x[5:6], S, age[5:6], path=path, mode="sequence")
        assert torch.equal(full[5:6], alone), path
        assert torch.equal(m.predict_record(x[:130], S, age[:130], path=path, mode="sequence"), full[:130]), path
        for k in (1, 2, 7):
            cut = m.predict_record(x[5:6, :, :W + (k - 1) * S], S, age[5:6], path=path, mode="sequence")
            assert cut.shape == (1, k) and torch.equal(cut, full[5:6, :k]), (path, k)
        assert torch.equal(m.predict_record(x, S, age, path=path, mode="sequence"), full), path


# ------------------------------------------------------------------ 6. independent mode unchanged; the launch list
# torch.profiler runs in a process of its own, as in tests/test_gpu_record.py
_LAUNCH_LIST = r"""
import collections, json, sys
import torch
import tskd_b200
from oracle import mycnn_torch as O
from tskd_b200 import capi
from torch.profiler import ProfilerActivity, profile

def kernels(fn):
    # a session of a process that has run others may miss its first kernel: a torch kernel goes first, and only the
    # library's kernels and memsets are counted
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        torch.ones(1, device=dev).add_(1)
        torch.cuda.synchronize()
        fn()
        torch.cuda.synchronize()
    return collections.Counter(e.name for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA
                               and ("b2cnn::" in e.name or e.name.startswith("Memset")))

path, W = sys.argv[1], 7504
P = {"tensorcore": capi.PATH_TENSORCORE, "generic": capi.PATH_GENERIC}[path]
dev = torch.device("cuda", 0)
ref = O.make_ref(O.stretched(O.ARCH_MYCNN5, 3, W), seed=91)
m = tskd_b200.B200MyCNN(tskd_b200.ARCH_PRESETS["mycnn5"].with_shape(3, W), has_out12=ref.arch.has_out12).to(dev)
m.load_state_dict(ref.state_dict())
lib, h = m._ensure_handle()
st = torch.cuda.current_stream().cuda_stream
age = torch.tensor([60.0], device=dev)
kernels(lambda: torch.ones(1, device=dev).add_(1))                  # profiler warm-up

def call(x, S, mode, ex):
    B, N = x.shape[0], x.shape[2]
    n = lib.b2cnn_record_workspace_bytes_ex(h, B, N, N, S, capi.DTYPE_BF16, P, mode)
    ws = torch.empty(n, dtype=torch.uint8, device=dev)
    out = torch.empty(B, (N - W) // S + 1, device=dev)
    if ex:
        rc = lib.b2cnn_score_record_ex(h, x.data_ptr(), capi.DTYPE_BF16, B, N, N, S, P, mode, age.data_ptr(), 1, 0, out.data_ptr(),
                                       ws.data_ptr(), n, st)
    else:
        rc = lib.b2cnn_score_record(h, x.data_ptr(), capi.DTYPE_BF16, B, N, N, S, P, age.data_ptr(), 1, 0, out.data_ptr(), ws.data_ptr(),
                                    n, st)
    assert rc == 0, capi.last_error()
    return out

res = {"seq": [], "indep": []}
for B, n_w, S in ((1, 10, 4), (257, 10, 4), (1, 1000, 4), (3, 5, 7504)):
    x = tskd_b200.synth.make_windows(B, 3, W + (n_w - 1) * S, "normal", seed=91, dtype=torch.bfloat16).to(dev)
    for mode in (capi.MODE_SEQUENCE, capi.MODE_INDEPENDENT):
        call(x, S, mode, True)                                        # warm-up: attributes, lazy module loads
    res["seq"].append(kernels(lambda: call(x, S, capi.MODE_SEQUENCE, True)))
    old, new = call(x, S, capi.MODE_INDEPENDENT, False), call(x, S, capi.MODE_INDEPENDENT, True)
    assert torch.equal(old, new)
    res["indep"].append([kernels(lambda: call(x, S, capi.MODE_INDEPENDENT, False)),
                         kernels(lambda: call(x, S, capi.MODE_INDEPENDENT, True))])
print(json.dumps(res))
"""


@pytest.mark.parametrize("path", ["tensorcore", "generic"])
def test_launch_lists(path):
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    env = dict(os.environ, PYTHONPATH=os.pathsep.join([root] + [p for p in [os.environ.get("PYTHONPATH")] if p]))
    cmd = [sys.executable] + (["-s"] if sys.flags.no_user_site else []) + ["-c", _LAUNCH_LIST, path]
    r = subprocess.run(cmd, capture_output=True, text=True, env=env, cwd=root, timeout=600)
    assert r.returncode == 0, r.stderr[-3000:]
    res = json.loads(r.stdout.strip().splitlines()[-1])
    seq = [collections.Counter(d) for d in res["seq"]]
    assert all(s == seq[0] for s in seq), seq                           # whatever B, N and S
    assert any("head_sequence_kernel" in k for k in seq[0]), seq[0]
    for old, new in res["indep"]:
        assert collections.Counter(old) == collections.Counter(new), (old, new)
        assert not any("head_sequence_kernel" in k for k in new), new


# ------------------------------------------------------------------ 7. errors before any launch
def test_errors_leave_the_model_usable():
    W, S = 7504, 752
    _, m = _tc_pair("mycnn5", 3, W, 95)
    x = _records(2, 3, W + 2 * S, BF, seed=95).to(DEV)
    age = tskd_b200.synth.make_ages(2, seed=95).to(DEV)
    good = m.predict_record(x, S, age, mode="sequence")
    for bad in ("seq", None, 1):
        with pytest.raises(ValueError, match="mode"):
            m.predict_record(x, S, age, mode=bad)
    lib, h = m._ensure_handle()
    N = x.shape[2]
    st = torch.cuda.current_stream().cuda_stream
    indep = int(lib.b2cnn_record_workspace_bytes(h, 2, N, N, S, capi.DTYPE_BF16, capi.PATH_TENSORCORE))
    seq = int(lib.b2cnn_record_workspace_bytes_ex(h, 2, N, N, S, capi.DTYPE_BF16, capi.PATH_TENSORCORE, capi.MODE_SEQUENCE))
    assert indep == int(lib.b2cnn_record_workspace_bytes_ex(h, 2, N, N, S, capi.DTYPE_BF16, capi.PATH_TENSORCORE, capi.MODE_INDEPENDENT))
    assert seq > indep > 0
    for bad in (2, -1):
        assert lib.b2cnn_record_workspace_bytes_ex(h, 2, N, N, S, capi.DTYPE_BF16, capi.PATH_TENSORCORE, bad) == -1
    ws = torch.empty(seq, dtype=torch.uint8, device=DEV)
    out = torch.full((2, 3), 7.0, device=DEV)

    def call(mode, n):
        return lib.b2cnn_score_record_ex(h, x.data_ptr(), capi.DTYPE_BF16, 2, N, N, S, capi.PATH_TENSORCORE, mode, age.data_ptr(), 2, 0,
                                         out.data_ptr(), ws.data_ptr(), n, st)
    for bad in (2, -1, 99):
        assert call(bad, seq) == capi.EINVAL
        assert "mode" in capi.last_error()
    assert call(capi.MODE_SEQUENCE, indep) == capi.ESTATE               # sized with the independent query
    torch.cuda.synchronize()
    assert (out == 7.0).all()                                           # nothing ran
    assert call(capi.MODE_SEQUENCE, seq) == 0
    torch.cuda.synchronize()
    assert torch.equal(out, good)
    assert torch.equal(m.predict_record(x, S, age, mode="sequence"), good)
    assert m.predict_record(x[:, :, :W - 1], S, age, mode="sequence").shape == (2, 0)
