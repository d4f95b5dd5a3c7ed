"""GPU: every sliding window of whole recordings in one call (B200MyCNN.predict_record, b2cnn_score_record).

- generic path: every element bit-identical (NaN for NaN) to predict(window, path="generic", small_kernel=0) on the
  materialised windows x.unfold(2, W, S): the MyCNN5 golden at W = 120, a C = 10 relu model with a negative-scale
  affine, pool (4, 4) with W % 16 != 0, S > W, (N - W) % S zero and not, contiguous, row-padded and offset views;
- tensor-core path: every element judged with check_elems against the float64 reference of its window at the
  scorer's grant BETA, in both geometries and dtypes, at strides 4, 8, 752, 7500 and > W and B = 1, 3, 130, 257;
- a 24 h recording at 125 Hz (10.8 M samples, W = 75000, S = 7500): 64 random windows, the first and the last;
- NaN and +-inf at the first sample, mid-recording, at a fold boundary and in the last R samples, and a NaN-padded
  tail, on both paths;
- independence of the batch, repeatability, agreement with a SlidingScorer fed the same samples, a launch list that
  does not depend on B or N, and errors raised before any launch."""
import collections
import json
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

import tskd_b200
from oracle import mycnn_torch as O
from oracle.infer_ref import infer_reference
from oracle.train_ref import BETA, check_elems
from test_gpu_infer_elem import _model
from test_gpu_slide_generic import _golden, _pair as _generic_pair, _same
from tskd_b200 import capi

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
BF, F32 = torch.bfloat16, torch.float32


def _check(pairs):
    check_elems(pairs, os.environ.get("PYTEST_CURRENT_TEST", "").split(" ")[0])


def _wins(x, W, S):
    """[B n_w, C, W]: the windows of every recording, recording-major"""
    B, C = x.shape[0], x.shape[1]
    u = x.unfold(2, W, S)                                          # [B, C, n_w, W]
    return u.permute(0, 2, 1, 3).reshape(B * u.shape[2], C, W).contiguous()


def _records(B, C, N, dtype, seed):
    return tskd_b200.synth.make_windows(B, C, N, "normal", seed=seed, dtype=dtype)


def _tc_pair(kind, C, W, seed):
    ref = O.make_ref(O.stretched(O.ARCHS[kind], C, W), seed=seed)
    return ref, _model(ref)


def _judge(tag, out, ref, x, S, age, idx=None):
    """(name, got, truth, ref32, beta) of out [B, n_w] against the float64 reference of the windows (rows idx of the
    flattened [B n_w] windows only, when given)"""
    W = ref.arch.window
    B, n_w = out.shape
    ages = age.reshape(-1).expand(B).repeat_interleave(n_w) if age.numel() == 1 else age.repeat_interleave(n_w)
    got = out.reshape(-1).cpu()
    if idx is None:
        win = _wins(x.cpu(), W, S)
    else:
        idx = torch.as_tensor(idx)
        win = torch.stack([x[i // n_w, :, (i % n_w) * S:(i % n_w) * S + W].cpu() for i in idx.tolist()])
        got, ages = got[idx], ages[idx]
    t, t32 = infer_reference(ref, win, ages), infer_reference(ref, win, ages, dtype=torch.float32)
    return [(f"z[{tag}]", got, t["z"], t32["z"], BETA)]


# ------------------------------------------------------------------ 1. generic path, bit for bit
def _generic_same(m, x, S, age, prob=False):
    W = m.arch.window
    out = m.predict_record(x, S, age, return_prob=prob, path="generic")
    n_w = (x.shape[2] - W) // S + 1 if x.shape[2] >= W else 0
    assert tuple(out.shape) == (x.shape[0], n_w)
    assert m.last_path == "generic"
    ages = age.reshape(-1).expand(x.shape[0]).repeat_interleave(n_w) if age.numel() == 1 else age.repeat_interleave(n_w)
    want = m.predict(_wins(x, W, S), ages.to(DEV), return_prob=prob).reshape(x.shape[0], n_w)
    assert _same(out, want)
    return out


@pytest.mark.parametrize("dtype", [F32, BF], ids=["f32", "bf16"])
@pytest.mark.parametrize("S", [72, 12])
def test_generic_golden_bit_identical(dtype, S):
    ref, m = _golden(5)
    C, W = ref.arch.in_channels, ref.arch.window
    x = _records(3, C, W + 9 * S + 5, dtype, seed=S).to(DEV)
    age = tskd_b200.synth.make_ages(3, seed=S).to(DEV)
    out = _generic_same(m, x, S, age)
    _generic_same(m, x, S, age, prob=True)
    _check(_judge(f"golden-S{S}", out, ref, x, S, age))


@pytest.mark.parametrize("case", ["c10-relu-affine", "pool44", "s-gt-w-exact", "s-gt-w-rest"])
def test_generic_models_and_strides(case):
    if case == "c10-relu-affine":
        geo, act, aff_seed, S, N = (10, 10, 5, 3, 2, 200), "relu", 7, 24, 200 + 11 * 24 + 3
    elif case == "pool44":
        geo, act, aff_seed, S, N = (3, 5, 5, 4, 4, 250), "tanh", None, 32, 250 + 7 * 32 + 9
    elif case == "s-gt-w-exact":
        geo, act, aff_seed, S, N = (3, 10, 5, 3, 2, 200), "tanh", None, 260, 200 + 4 * 260
    else:
        geo, act, aff_seed, S, N = (3, 10, 5, 3, 2, 200), "tanh", None, 260, 200 + 4 * 260 + 100
    ref, m, _ = _generic_pair(geo, act=act, aff_seed=aff_seed, seed=11)
    C = geo[0]
    for dtype in (F32, BF):
        x = _records(4, C, N, dtype, seed=5).to(DEV)
        age = tskd_b200.synth.make_ages(4, seed=5).to(DEV)
        _generic_same(m, x, S, age)
        _generic_same(m, x, S, torch.tensor([70.0], device=DEV))


def test_generic_views():
    ref, m = _golden(5)
    C, W, S = ref.arch.in_channels, ref.arch.window, 36
    N = W + 6 * S
    base = _records(3, C, N + 7, F32, seed=9).to(DEV)
    age = tskd_b200.synth.make_ages(3, seed=9).to(DEV)
    contiguous = _generic_same(m, base[:, :, :N].contiguous(), S, age)
    assert _same(_generic_same(m, base[:, :, :N], S, age), contiguous)           # row-padded view
    _generic_same(m, base[:, :, 1:N + 1], S, age)                               # one-sample offset view
    _generic_same(m, base[1:2, :, 3:N + 3], S, age[1:2])


# ------------------------------------------------------------------ 2. tensor-core path against float64
TC_CASES = {
    "m5-bf16-w7504-s752-b3": ("mycnn5", 3, BF, 7504, 752, 3, 7504 + 10 * 752 + 5),
    "m5-bf16-w7500-s4-b1": ("mycnn5", 3, BF, 7500, 4, 1, 7500 + 40),
    "m5-bf16-w7500-s8-b3": ("mycnn5", 3, BF, 7500, 8, 3, 7500 + 80 + 3),
    "m5-f32-w7500-s7500-b3": ("mycnn5", 3, F32, 7500, 7500, 3, 7500 + 3 * 7500),
    "m3-f32-w7502-s7500-b3": ("mycnn3", 1, F32, 7502, 7500, 3, 3 * 7500 + 7502),
    "m3-f32-w7502-s9000-b130": ("mycnn3", 1, F32, 7502, 9000, 130, 7502 + 9000 + 100),
    "m3-bf16-w7502-s8-b3": ("mycnn3", 1, BF, 7502, 8, 3, 7502 + 8 * 8 + 1),
    "m5-bf16-w7504-s7500-b257": ("mycnn5", 3, BF, 7504, 7500, 257, 7504 + 7500),
}


@pytest.mark.parametrize("name", sorted(TC_CASES))
def test_tensorcore_against_float64(name):
    kind, C, dtype, W, S, B, N = TC_CASES[name]
    seed = 300 + sorted(TC_CASES).index(name)
    ref, m = _tc_pair(kind, C, W, seed)
    x = _records(B, C, N, dtype, seed=seed).to(DEV)
    age = tskd_b200.synth.make_ages(B, seed=seed).to(DEV)
    out = m.predict_record(x, S, age, path="tensorcore")
    assert m.last_path == "tensorcore"
    assert tuple(out.shape) == (B, (N - W) // S + 1)
    auto = m.predict_record(x, S, age)                             # auto takes the tensor cores for these models
    assert torch.equal(auto, out)
    _check(_judge(name, out, ref, x, S, age))


# ------------------------------------------------------------------ 3. one 24 h recording
def test_long_recording():
    W, S, N = 75000, 7500, 10_800_000
    ref, m = _tc_pair("mycnn5", 3, W, 41)
    x = _records(1, 3, N, BF, seed=41).to(DEV)
    age = torch.tensor([63.0], device=DEV)
    out = m.predict_record(x, S, age)
    n_w = (N - W) // S + 1
    assert tuple(out.shape) == (1, n_w) and m.last_path == "tensorcore"
    g = torch.Generator().manual_seed(41)
    idx = sorted(set([0, n_w - 1] + torch.randint(1, n_w - 1, (64,), generator=g).tolist()))
    _check(_judge("24h", out, ref, x, S, age, idx))


# ------------------------------------------------------------------ 4. NaN and +-inf
def test_nan_inf_both_paths():
    W, S = 7504, 752
    N = W + 30 * 752
    ref, m = _tc_pair("mycnn5", 3, W, 51)
    x = _records(3, 3, N, BF, seed=51)
    L_N = (N - 24) // 4 + 1
    nr = (L_N + 4095) // 4096
    K = ((L_N + nr - 1) // nr + 7) // 8 * 8
    fold = 4 * K                                                   # first sample of the second folded row
    assert nr >= 2
    x[0, 0, 0] = float("nan")                                       # the first sample
    x[0, 1, N // 2] = float("inf")                                  # mid-recording
    x[0, 2, fold + 3] = -float("inf")                               # in the halo both rows read
    x[2, 0, fold - 2] = float("nan")                                # at the fold boundary
    x[2, 1, N - 5] = float("nan")                                   # in the last R samples
    true_len = N - 3000
    x[1, :, true_len:] = float("nan")                               # a NaN-padded tail
    xd = x.to(DEV)
    age = tskd_b200.synth.make_ages(3, seed=51).to(DEV)
    n_full = (true_len - W) // S + 1
    for path in ("tensorcore", "generic"):
        out = m.predict_record(xd, S, age, path=path)
        assert m.last_path == path
        assert torch.isfinite(out[1, :n_full]).all() and torch.isnan(out[1, n_full:]).all(), path
        assert torch.isnan(out[0, 0]) and torch.isnan(out[2, -1])
        _check(_judge(f"nan-inf-{path}", out, ref, xd, S, age))


# ------------------------------------------------------------------ 5. independence and repeatability
def test_independent_of_the_batch():
    W, S = 7504, 1876
    ref, m = _tc_pair("mycnn5", 3, W, 61)
    x = _records(258, 3, W + 3 * S + 2, BF, seed=61).to(DEV)
    age = tskd_b200.synth.make_ages(258, seed=61).to(DEV)
    for path in ("tensorcore", "generic"):
        alone = m.predict_record(x[5:6], S, age[5:6], path=path)
        for n in (131, 258):
            batch = m.predict_record(x[:n], S, age[:n], path=path)
            assert torch.equal(batch[5:6], alone), (path, n)
        again = m.predict_record(x, S, age, path=path)
        assert torch.equal(again, m.predict_record(x, S, age, path=path)), path


# ------------------------------------------------------------------ 6. agreement with a SlidingScorer
def test_agrees_with_the_scorer_tensorcore():
    W, S, B = 7500, 1500, 3
    ref, m = _tc_pair("mycnn5", 3, W, 71)
    N = W + 5 * S
    x = _records(B, 3, N, BF, seed=71).to(DEV)
    age = tskd_b200.synth.make_ages(B, seed=71).to(DEV)
    out = m.predict_record(x, S, age, path="tensorcore")
    sc = tskd_b200.SlidingScorer(m, B, S, BF, path="tensorcore")
    pushed = []
    for n in range(1, N // S + 1):
        got = sc.push(x[:, :, (n - 1) * S:n * S], age)
        if n * S >= W:
            assert sc.window_index == n - W // S
            pushed.append(got.clone())
    sc.close()
    pushed = torch.stack(pushed, 1)
    assert pushed.shape == out.shape
    _check(_judge("record", out, ref, x, S, age) + _judge("scorer", pushed, ref, x, S, age))


def test_agrees_with_the_scorer_generic():
    ref, m = _golden(5)
    C, W, S, B = ref.arch.in_channels, ref.arch.window, 24, 4
    N = W + 8 * S
    x = _records(B, C, N, F32, seed=81).to(DEV)
    age = tskd_b200.synth.make_ages(B, seed=81).to(DEV)
    out = m.predict_record(x, S, age, path="generic")
    sc = tskd_b200.SlidingScorer(m, B, S, F32, path="generic")
    for n in range(1, N // S + 1):
        got = sc.push(x[:, :, (n - 1) * S:n * S], age)
        if n * S >= W:
            assert _same(got, out[:, n - W // S]), n
    sc.close()


# ------------------------------------------------------------------ 7. the launch list
# torch.profiler runs in a process of its own: a profiler session changes what later sessions of the same process record
# (the first one may miss its first kernel), and other test files compare kernel lists in the pytest process.
_LAUNCH_LIST = r"""
import collections, json, sys
import torch
import tskd_b200
from oracle import mycnn_torch as O
from torch.profiler import ProfilerActivity, profile

def kernels(fn):
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    return collections.Counter(e.name for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA)

path, W, S = sys.argv[1], 7504, 4
dev = torch.device("cuda", 0)
ref = O.make_ref(O.stretched(O.ARCH_MYCNN5, 3, W), seed=91)
m = tskd_b200.B200MyCNN(tskd_b200.ARCH_PRESETS["mycnn5"].with_shape(3, W), has_out12=ref.arch.has_out12).to(dev)
m.load_state_dict(ref.state_dict())
age = torch.tensor([60.0], device=dev)
kernels(lambda: torch.ones(1, device=dev).add_(1))                  # profiler warm-up
lists = []
for B, n_w in ((1, 10), (257, 10), (1, 1000)):
    x = tskd_b200.synth.make_windows(B, 3, W + (n_w - 1) * S, "normal", seed=91, dtype=torch.bfloat16).to(dev)
    m.predict_record(x, S, age, path=path)                          # warm-up: attributes, lazy module loads
    assert m.last_path == path
    lists.append(kernels(lambda: m.predict_record(x, S, age, path=path)))
print(json.dumps(lists))
"""


@pytest.mark.parametrize("path", ["tensorcore", "generic"])
def test_launch_list_does_not_depend_on_the_input(path):
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    env = dict(os.environ, PYTHONPATH=os.pathsep.join([root] + [p for p in [os.environ.get("PYTHONPATH")] if p]))
    cmd = [sys.executable] + (["-s"] if sys.flags.no_user_site else []) + ["-c", _LAUNCH_LIST, path]
    r = subprocess.run(cmd, capture_output=True, text=True, env=env, cwd=root, timeout=600)
    assert r.returncode == 0, r.stderr[-3000:]
    lists = [collections.Counter(d) for d in json.loads(r.stdout.strip().splitlines()[-1])]
    assert sum(lists[0].values()) >= 5, lists
    assert lists[0] == lists[1] == lists[2], lists


# ------------------------------------------------------------------ 8. errors before any launch
def test_errors_leave_the_model_usable():
    W, S = 7504, 752
    ref, m = _tc_pair("mycnn5", 3, W, 95)
    x = _records(2, 3, W + 2 * S, BF, seed=95).to(DEV)
    age = tskd_b200.synth.make_ages(2, seed=95).to(DEV)
    good = m.predict_record(x, S, age)
    with pytest.raises(ValueError):
        m.predict_record(x[0], S, age)                              # rank
    with pytest.raises(ValueError):
        m.predict_record(x[:, :2], S, age)                          # channels
    with pytest.raises(ValueError):
        m.predict_record(x.half(), S, age)                          # dtype
    for bad in (0, -4, 6):
        with pytest.raises(ValueError):
            m.predict_record(x, bad, age)
    with pytest.raises(ValueError):
        m.predict_record(x, S, torch.ones(3, device=DEV))
    _, g, _ = _generic_pair((10, 10, 5, 3, 2, 200), seed=3, path="auto")
    xg = _records(2, 10, 400, F32, seed=3).to(DEV)
    with pytest.raises(RuntimeError, match="tensor-core path covers"):
        g.predict_record(xg, 8, path="tensorcore")
    assert g.predict_record(xg, 8).shape == (2, 26)
    # the C ABI: a workspace one byte short, and none
    lib, h = m._ensure_handle()
    need = int(lib.b2cnn_record_workspace_bytes(h, 2, x.shape[2], x.shape[2], S, capi.DTYPE_BF16, capi.PATH_AUTO))
    assert need > 0
    ws = torch.empty(need, dtype=torch.uint8, device=DEV)
    out = torch.full((2, 3), 7.0, device=DEV)
    st = torch.cuda.current_stream().cuda_stream
    for ptr, n in ((ws.data_ptr(), need - 1), (None, 0)):
        rc = lib.b2cnn_score_record(h, x.data_ptr(), capi.DTYPE_BF16, 2, x.shape[2], x.shape[2], S, capi.PATH_AUTO, age.data_ptr(), 2,
                                    0, out.data_ptr(), ptr, n, st)
        assert rc == capi.ESTATE
    rc = lib.b2cnn_score_record(h, x.data_ptr(), capi.DTYPE_BF16, 2, x.shape[2], x.shape[2], 6, capi.PATH_AUTO, age.data_ptr(), 2, 0,
                                out.data_ptr(), ws.data_ptr(), need, st)
    assert rc == capi.EINVAL
    torch.cuda.synchronize()
    assert (out == 7.0).all()                                       # nothing ran
    assert torch.equal(m.predict_record(x, S, age), good)
    assert m.predict_record(x[:, :, :W - 1], S, age).shape == (2, 0)
