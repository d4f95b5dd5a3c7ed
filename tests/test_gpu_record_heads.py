"""GPU: candidate heads over whole recordings (B200MyCNN.predict_record(heads=[...]), b2cnn_score_record_heads,
csrc/b2cnn_record.cu).

The criterion is bit identity.  M0 and heads M1..MK share M0's conv weights; their LSTM, Linear and age_coef are seeded
per head (as tests/test_gpu_slide_heads.py builds them).  Row 0 of M0.predict_record(..., heads=[M1..MK]) must be
torch.equal to M0.predict_record(...) and row i to Mi.predict_record(...) with the same arguments, NaN for NaN, on
records holding NaN and +-inf:
- tensor cores: MyCNN5 geometry (C = 3 bf16, W = 7504, S = 752) and MyCNN3 geometry (C = 1 fp32, W = 7502), K in {1, 2,
  3, 8}, B in {1, 3, 130}, both modes; one 24 h recording with K = 3;
- generic path: the MyCNN5.pth golden at W = 120, S = 12 (fp32 and bf16) and a relu, negative-scale-affine C = 10 model;
- sequence mode with a random start state per row, and chained chunk calls equal to one call;
- the model's own handle as a head, a head trained with conv1 / conv2 frozen, float64 judgement per path at the existing
  grants, the launch list, and every refusal of the C ABI before any launch."""
import collections
import ctypes
import gc
import json
import os
import subprocess
import sys
from dataclasses import replace

import pytest
import torch

import tskd_b200
from oracle import mycnn_torch as O
from oracle.train_ref import check_elems
from test_gpu_record import _judge, _records
from test_gpu_slide_generic import _same
from test_gpu_slide_heads import _gen_family, _head_sd, _like
from tskd_b200 import capi

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
BF, F32 = torch.bfloat16, torch.float32
TC_GEOS = {"mycnn5": (3, BF, 7504, 752), "mycnn3": (1, F32, 7502, 752)}


def _n_w(N, W, S):
    return (N - W) // S + 1 if N >= W else 0


def _poison(x, W, S):
    """NaN and +-inf samples: in the first window, mid-recording, in the last window"""
    B, C, N = x.shape
    x[0, 0, 3] = float("nan")
    x[B - 1, C - 1, N // 2] = float("inf")
    x[B // 2, 0, N - 7] = -float("inf")
    return x


_FAMILIES = {}


@pytest.fixture(autouse=True, scope="module")
def _release_families():
    """the module's models (handles, device weights) and the allocator's blocks go when the module ends: the files
    after this one see the process as they would without it"""
    yield
    _FAMILIES.clear()
    gc.collect()
    torch.cuda.synchronize()
    torch.cuda.empty_cache()


def _tc_family(kind):
    """(ref, M0, 8 heads) of a tensor-core geometry: M0's conv weights, seeded LSTM / Linear, age_coef per head; built
    once per module"""
    if kind not in _FAMILIES:
        _FAMILIES[kind] = _build_tc_family(kind)
    return _FAMILIES[kind]


def _build_tc_family(kind):
    C, _, W, _ = TC_GEOS[kind]
    ref = O.make_ref(O.stretched(O.ARCHS[kind], C, W), seed=7)
    arch = replace(tskd_b200.ARCH_PRESETS[kind].with_shape(C, W), age_coef=ref.arch.age_coef)
    m0 = tskd_b200.B200MyCNN(arch, has_out12=ref.arch.has_out12).to(DEV)
    sd = dict(ref.state_dict())
    m0.load_state_dict(sd)
    return ref, m0, sd, tuple(_like(m0, _head_sd(sd, 70 + i), 1e-3 * (i + 1), False) for i in range(8))


def _rows_equal(out, models, x, S, age, **kw):
    """every row of a heads call torch.equal (NaN for NaN) to its model's own call"""
    assert out.shape[0] == len(models)
    for i, m in enumerate(models):
        assert _same(out[i], m.predict_record(x, S, age, **kw)), i


# ------------------------------------------------------------------ 1. tensor cores, bit for bit
@pytest.mark.parametrize("mode", ["independent", "sequence"])
@pytest.mark.parametrize("B", [1, 3, 130])
@pytest.mark.parametrize("K", [1, 2, 3, 8])
@pytest.mark.parametrize("kind", ["mycnn5", "mycnn3"])
def test_tc_rows(kind, K, B, mode):
    _, m0, _, heads = _tc_family(kind)
    C, dtype, W, S = TC_GEOS[kind]
    x = _poison(_records(B, C, W + 9 * S + 5, dtype, seed=K * 100 + B).to(DEV), W, S)
    age = tskd_b200.synth.make_ages(B, seed=K + B).to(DEV)
    hs = list(heads[:K])
    out = m0.predict_record(x, S, age, path="tensorcore", mode=mode, heads=hs)
    assert tuple(out.shape) == (1 + K, B, _n_w(x.shape[2], W, S)) and m0.last_path == "tensorcore"
    assert torch.isnan(out).any()
    _rows_equal(out, [m0] + hs, x, S, age, path="tensorcore", mode=mode)


def test_tc_prob_and_auto():
    """return_prob and path "auto" (the tensor cores for these models) row for row"""
    _, m0, _, heads = _tc_family("mycnn5")
    C, dtype, W, S = TC_GEOS["mycnn5"]
    x = _records(3, C, W + 4 * S, dtype, seed=5).to(DEV)
    age = torch.tensor([70.0], device=DEV)
    out = m0.predict_record(x, S, age, return_prob=True, heads=list(heads[:3]))
    _rows_equal(out, [m0] + list(heads[:3]), x, S, age, return_prob=True)


def test_empty_heads_is_plain_call():
    _, m0, _, _ = _tc_family("mycnn5")
    C, dtype, W, S = TC_GEOS["mycnn5"]
    x = _records(2, C, W + 3 * S, dtype, seed=6).to(DEV)
    want = m0.predict_record(x, S, 65.0)
    for h in (None, []):
        got = m0.predict_record(x, S, 65.0, heads=h)
        assert got.shape == want.shape and torch.equal(got, want)


def test_long_recording():
    """one 24 h recording at 125 Hz, W = 75000, S = 7500, K = 3 on the tensor cores"""
    W, S, N = 75000, 7500, 10_800_000
    ref = O.make_ref(O.stretched(O.ARCH_MYCNN5, 3, W), seed=41)
    arch = replace(tskd_b200.ARCH_PRESETS["mycnn5"].with_shape(3, W), age_coef=ref.arch.age_coef)
    m0 = tskd_b200.B200MyCNN(arch, has_out12=ref.arch.has_out12).to(DEV)
    sd = dict(ref.state_dict())
    m0.load_state_dict(sd)
    hs = [_like(m0, _head_sd(sd, 410 + i), 1e-3 * (i + 1), False) for i in range(3)]
    x = _records(1, 3, N, BF, seed=41).to(DEV)
    age = torch.tensor([63.0], device=DEV)
    for mode in ("independent", "sequence"):
        out = m0.predict_record(x, S, age, mode=mode, heads=hs)
        assert tuple(out.shape) == (4, 1, _n_w(N, W, S)) and m0.last_path == "tensorcore"
        _rows_equal(out, [m0] + hs, x, S, age, mode=mode)


# ------------------------------------------------------------------ 2. generic path, bit for bit
@pytest.mark.parametrize("mode", ["independent", "sequence"])
@pytest.mark.parametrize("dtype", [F32, BF], ids=["f32", "bf16"])
def test_generic_golden(dtype, mode):
    m0, _, heads = _gen_family(None, 3, seed=3)
    S, B = 12, 3
    x = _poison(_records(B, 10, 120 + 20 * S + 5, dtype, seed=8).to(DEV), 120, S)
    age = tskd_b200.synth.make_ages(B, seed=8).to(DEV)
    out = m0.predict_record(x, S, age, path="generic", mode=mode, heads=heads)
    assert tuple(out.shape) == (4, B, 21) and m0.last_path == "generic"
    _rows_equal(out, [m0] + heads, x, S, age, path="generic", mode=mode)


@pytest.mark.parametrize("mode", ["independent", "sequence"])
def test_generic_relu_affine(mode):
    m0, _, heads = _gen_family((10, 5, 3, 2, 2, 200), 2, seed=9, act="relu", aff_seed=9)
    assert m0.arch.affine
    S, B = 8, 130
    x = _poison(_records(B, 10, 200 + 6 * S + 3, F32, seed=9).to(DEV), 200, S)
    age = tskd_b200.synth.make_ages(B, seed=9).to(DEV)
    out = m0.predict_record(x, S, age, path="generic", mode=mode, heads=heads)
    _rows_equal(out, [m0] + heads, x, S, age, path="generic", mode=mode)


# ------------------------------------------------------------------ 3. sequence mode with state, chained chunks
def _state(rows, B, seed):
    g = torch.Generator().manual_seed(seed)
    return (0.5 * torch.randn(rows, B, 2, 2, 16, generator=g)).to(DEV)


@pytest.mark.parametrize("path", ["tensorcore", "generic"])
def test_state_rows_and_chunks(path):
    if path == "tensorcore":
        _, m0, _, heads = _tc_family("mycnn5")
        C, dtype, W, S = TC_GEOS["mycnn5"]
        hs = list(heads[:3])
    else:
        m0, _, hs = _gen_family(None, 3, seed=4)
        C, dtype, W, S = 10, F32, 120, 12
    B, n_w = 3, 10
    x = _records(B, C, W + (n_w - 1) * S + 3, dtype, seed=12).to(DEV)
    if path == "generic":
        # the tensor-core front end re-computes a folded row that holds NaN / inf exactly, and a chunk folds its rows
        # elsewhere: chunked calls there are bit-identical on finite records (test_tc_rows covers NaN per row)
        x = _poison(x, W, S)
    age = tskd_b200.synth.make_ages(B, seed=12).to(DEV)
    st = _state(4, B, 12)
    out, so = m0.predict_record(x, S, age, path=path, mode="sequence", state=st, return_state=True, heads=hs)
    assert tuple(so.shape) == (4, B, 2, 2, 16)
    for i, m in enumerate([m0] + hs):
        o, s = m.predict_record(x, S, age, path=path, mode="sequence", state=st[i], return_state=True)
        assert _same(out[i], o) and _same(so[i], s), i
    for k in (1, n_w // 2, n_w - 1):
        a, sa = m0.predict_record(x[:, :, :(k - 1) * S + W], S, age, path=path, mode="sequence", state=st, return_state=True,
                                  heads=hs)
        b, sb = m0.predict_record(x[:, :, k * S:], S, age, path=path, mode="sequence", state=sa, return_state=True, heads=hs)
        assert _same(torch.cat([a, b], dim=2), out) and _same(sb, so), k
    # no window: every row's state passes through
    e, se = m0.predict_record(x[:, :, :W - 4], S, age, path=path, mode="sequence", state=st, return_state=True, heads=hs)
    assert tuple(e.shape) == (4, B, 0) and torch.equal(se, st)
    e, se = m0.predict_record(x[:, :, :W - 4], S, age, path=path, mode="sequence", return_state=True, heads=hs)
    assert not se.any()


# ------------------------------------------------------------------ 4. own handle, a trained candidate
def test_own_handle_as_head():
    _, m0, _, _ = _tc_family("mycnn3")
    C, dtype, W, S = TC_GEOS["mycnn3"]
    x = _records(3, C, W + 5 * S, dtype, seed=13).to(DEV)
    for mode in ("independent", "sequence"):
        out = m0.predict_record(x, S, 60.0, mode=mode, heads=[m0])
        assert _same(out[1], out[0])


def test_trained_candidate():
    """a B200TrainableMyCNN fine-tuned with conv1 / conv2 frozen keeps the front end: a valid head"""
    m0, sd, _ = _gen_family(None, 0, seed=5)
    cand = tskd_b200.B200TrainableMyCNN(m0.arch, path="generic").to(DEV)
    cand.load_state_dict(sd)
    cand.conv1.requires_grad_(False)
    cand.conv2.requires_grad_(False)
    opt = torch.optim.Adam([p for p in cand.parameters() if p.requires_grad], lr=1e-2)
    xw = tskd_b200.synth.make_windows(16, 10, 120, "normal", seed=5).to(DEV)
    y = (torch.arange(16, device=DEV) % 2).float()
    cand.train()
    for _ in range(3):
        opt.zero_grad()
        torch.nn.functional.binary_cross_entropy_with_logits(cand(xw, torch.full((16,), 60.0, device=DEV)), y).backward()
        opt.step()
    cand.eval()
    cand.set_option("small_kernel", 0)
    x = _records(2, 10, 120 + 9 * 12, F32, seed=5).to(DEV)
    for mode in ("independent", "sequence"):
        out = m0.predict_record(x, 12, 60.0, path="generic", mode=mode, heads=[cand])
        _rows_equal(out, [m0, cand], x, 12, 60.0, path="generic", mode=mode)
        assert not torch.equal(out[1], out[0])


# ------------------------------------------------------------------ 5. float64, one case per path
def _head_ref(ref, sd, m):
    r = O.RefMyCNN(replace(ref.arch, age_coef=m.arch.age_coef))
    r.load_state_dict({k: v for k, v in sd.items()})
    return r.eval()


def test_float64_tensorcore():
    ref, m0, sd, heads = _tc_family("mycnn5")
    C, dtype, W, S = TC_GEOS["mycnn5"]
    x = _records(3, C, W + 6 * S, dtype, seed=14).to(DEV)
    age = tskd_b200.synth.make_ages(3, seed=14).to(DEV)
    out = m0.predict_record(x, S, age, path="tensorcore", heads=list(heads[:2]))
    pairs = _judge("row0", out[0], ref, x, S, age)
    for i, m in enumerate(heads[:2]):
        pairs += _judge(f"row{i + 1}", out[i + 1], _head_ref(ref, _head_sd(sd, 70 + i), m), x, S, age)
    check_elems(pairs, "test_float64_tensorcore")


def test_float64_generic():
    m0, sd, heads = _gen_family((10, 5, 3, 2, 2, 200), 2, seed=15)
    ref = O.make_ref(O.RefArch(in_channels=10, k1=5, k2=3, pool_k=2, pool_s=2, window=200, age_coef=1e-4, has_out12=False), seed=15)
    x = _records(2, 10, 200 + 8 * 8, F32, seed=15).to(DEV)
    age = tskd_b200.synth.make_ages(2, seed=15).to(DEV)
    out = m0.predict_record(x, 8, age, path="generic", heads=heads)
    pairs = _judge("row0", out[0], ref, x, 8, age)
    for i, m in enumerate(heads):
        pairs += _judge(f"row{i + 1}", out[i + 1], _head_ref(ref, _head_sd(sd, 150 + i), m), x, 8, age)
    check_elems(pairs, "test_float64_generic")


# ------------------------------------------------------------------ 6. launch list
# torch.profiler runs in a process of its own, as in tests/test_gpu_record_state.py, and the reported session brackets
# the call with torch kernels and counts only when all four were recorded
_LAUNCH_LIST = r"""
import collections, json, sys
from dataclasses import replace
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

path, mode, W, S = sys.argv[1], sys.argv[2], 7504, 752
dev = torch.device("cuda", 0)
ref = O.make_ref(O.stretched(O.ARCH_MYCNN5, 3, W), seed=91)
arch = tskd_b200.ARCH_PRESETS["mycnn5"].with_shape(3, W)
models = []
for i in range(4):
    m = tskd_b200.B200MyCNN(replace(arch, age_coef=1e-3 * (i + 1)), has_out12=ref.arch.has_out12).to(dev)
    m.load_state_dict(ref.state_dict())
    models.append(m)
x = tskd_b200.synth.make_windows(3, 3, W + 9 * S, "normal", seed=91, dtype=torch.bfloat16).to(dev)
age = torch.tensor([60.0], device=dev)
res = {}
for K in (None, 0, 1, 2, 3):
    call = (lambda: models[0].predict_record(x, S, age, path=path, mode=mode)) if K is None else \
           (lambda K=K: models[0].predict_record(x, S, age, path=path, mode=mode, heads=models[1:1 + K]))
    call()                                                                 # warm-up: attributes, lazy module loads
    session(lambda: None)                                                 # profiler warm-up, torch kernels only
    res[str(K)] = kernels(call)
print(json.dumps(res))
"""


def _launches(path, mode):
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    env = dict(os.environ, PYTHONPATH=os.pathsep.join([root] + [p for p in [os.environ.get("PYTHONPATH")] if p]))
    cmd = [sys.executable] + (["-s"] if sys.flags.no_user_site else []) + ["-c", _LAUNCH_LIST, path, mode]
    r = subprocess.run(cmd, capture_output=True, text=True, env=env, cwd=root, timeout=900)
    assert r.returncode == 0, r.stderr[-3000:]
    return {k: collections.Counter(v) for k, v in json.loads(r.stdout.strip().splitlines()[-1]).items()}


def _split(c):
    """(projection HP = 1, projection HP = 2, the per-row head kernels, the rest) of a launch Counter"""
    proj1 = sum(n for k, n in c.items() if "slide_record_proj_kernel<1>" in k)
    proj2 = sum(n for k, n in c.items() if "slide_record_proj_kernel<2>" in k)
    per_row = ("::proj_kernel", "::record_proj_kernel", "reduce_gates_kernel", "head_")
    head = collections.Counter({k: n for k, n in c.items() if "slide_record_proj_kernel" not in k and any(t in k for t in per_row)})
    rest = collections.Counter({k: n for k, n in c.items() if "slide_record_proj_kernel" not in k and k not in head})
    return proj1, proj2, head, rest


@pytest.mark.parametrize("mode", ["independent", "sequence"])
@pytest.mark.parametrize("path", ["tensorcore", "generic"])
def test_launch_list(path, mode):
    res = _launches(path, mode)
    assert res["0"] == res["None"], res                                  # K = 0: exactly predict_record's kernels
    p1, p2, head0, rest0 = _split(res["0"])
    for K in (1, 2, 3):
        q1, q2, head, rest = _split(res[str(K)])
        assert rest == rest0, (K, res)                                   # stage, front end, flags, age: once
        assert head == collections.Counter({k: n * (1 + K) for k, n in head0.items()}), (K, res)   # one head per row
        if path == "tensorcore":
            assert (p1, p2) == (1, 0)
            assert q2 == (1 + K) // 2 and q1 == (1 + K) % 2, (K, res)   # pairs, HP = 1 for an odd last row only
        else:
            assert q1 == q2 == 0


# ------------------------------------------------------------------ 7. refusals of the C ABI, before any launch
def test_refusals():
    _, m0, sd, heads = _tc_family("mycnn5")
    C, dtype, W, S = TC_GEOS["mycnn5"]
    lib, h = m0._ensure_handle()
    hs = [m._ensure_handle()[1].value for m in heads[:2]]
    B, N = 2, W + 3 * S
    n_w = _n_w(N, W, S)
    x = _records(B, C, N, dtype, seed=16).to(DEV)
    age = torch.tensor([60.0], device=DEV)
    seq, ind = capi.MODE_SEQUENCE, capi.MODE_INDEPENDENT
    need = int(lib.b2cnn_record_workspace_bytes_heads(h, 2, B, N, N, S, capi.DTYPE_BF16, capi.PATH_TENSORCORE, seq))
    base = int(lib.b2cnn_record_workspace_bytes_ex(h, B, N, N, S, capi.DTYPE_BF16, capi.PATH_TENSORCORE, seq))
    assert int(lib.b2cnn_record_workspace_bytes_heads(h, 0, B, N, N, S, capi.DTYPE_BF16, capi.PATH_TENSORCORE, seq)) == base
    n_ranges = (need - base) // (4 * B * n_w * 64)
    assert need - base == (4 * n_ranges * B * n_w * 64 + 255) // 256 * 256 and n_ranges >= 1   # one partial buffer
    gen = int(lib.b2cnn_record_workspace_bytes_ex(h, B, N, N, S, capi.DTYPE_BF16, capi.PATH_GENERIC, seq))
    assert int(lib.b2cnn_record_workspace_bytes_heads(h, 3, B, N, N, S, capi.DTYPE_BF16, capi.PATH_GENERIC, seq)) == gen
    for n in (-1, 9):
        assert lib.b2cnn_record_workspace_bytes_heads(h, n, B, N, N, S, capi.DTYPE_BF16, capi.PATH_TENSORCORE, seq) == -1
    ws = torch.empty(need, dtype=torch.uint8, device=DEV)
    out = torch.full((3, B, n_w), 7.0, device=DEV)
    sin, sout = _state(3, B, 16), torch.full((3, B, 64), 7.0, device=DEV)
    sin_keep = sin.clone()
    arr = lambda v: (ctypes.c_void_p * max(len(v), 1))(*v)
    st = torch.cuda.current_stream().cuda_stream

    def call(handle=h, heads_=hs, n=2, mode=seq, s_in=sin.data_ptr(), s_out=sout.data_ptr(), stride=S, wsb=need, path=capi.PATH_TENSORCORE):
        return lib.b2cnn_score_record_heads(handle, arr(heads_) if heads_ is not None else None, n, x.data_ptr(), capi.DTYPE_BF16, B, N,
                                            N, stride, path, mode, age.data_ptr(), 1, 0, out.data_ptr(), s_in, s_out, ws.data_ptr(),
                                            wsb, st)

    other_arch = tskd_b200.B200MyCNN(tskd_b200.ARCH_PRESETS["mycnn5"].with_shape(3, 7512)).to(DEV)
    other_conv = dict(sd)
    other_conv["conv1.weight"] = sd["conv1.weight"] + 1e-3
    stale = _like(m0, other_conv, 1e-3, False)
    cfg = capi.make_config(m0.arch, 0)
    bare = ctypes.c_void_p()
    capi.check(lib.b2cnn_create(ctypes.byref(cfg), ctypes.byref(bare)), "b2cnn_create")     # no weights set
    try:
        cases = [
            (capi.EINVAL, dict(handle=None), ""),
            (capi.EINVAL, dict(n=-1), "n_heads"),
            (capi.EINVAL, dict(n=9, heads_=hs * 5), "n_heads"),
            (capi.EINVAL, dict(heads_=None), "null"),
            (capi.EINVAL, dict(heads_=[hs[0], None]), "head 1: null handle"),
            (capi.EINVAL, dict(heads_=[hs[0], bare.value]), "head 1: weights not set"),
            (capi.EINVAL, dict(mode=ind), "sequence mode"),
            (capi.EINVAL, dict(s_out=sin.data_ptr() + 4 * 64), "overlap"),
            (capi.EINVAL, dict(stride=S + 2), "stride"),
            (capi.EARCH, dict(heads_=[hs[0], other_arch._ensure_handle()[1].value]), "head 1: another architecture"),
            (capi.ESTATE, dict(heads_=[hs[0], stale._ensure_handle()[1].value]), "head 1: other front-end"),
            (capi.ESTATE, dict(wsb=need - 256), "workspace"),
        ]
        torch.cuda.synchronize()
        for code, kw, msg in cases:
            assert call(**kw) == code, kw
            assert msg in capi.last_error(), (kw, capi.last_error())
        torch.cuda.synchronize()
        assert (out == 7.0).all() and (sout == 7.0).all() and torch.equal(sin, sin_keep)      # nothing ran
    finally:
        lib.b2cnn_destroy(bare)
    # the model still scores, row for row
    assert call() == 0
    torch.cuda.synchronize()
    want, wso = m0.predict_record(x, S, age, mode="sequence", state=sin_keep.reshape(3, B, 2, 2, 16), return_state=True,
                                  heads=list(heads[:2]))
    assert _same(out, want) and torch.equal(sout.reshape(3, B, 2, 2, 16), wso)


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs a second GPU")
def test_other_device_refused():
    _, m0, sd, _ = _tc_family("mycnn5")
    other = _like(m0, sd, 1e-3, False).to("cuda:1")
    C, dtype, W, S = TC_GEOS["mycnn5"]
    x = _records(1, C, W + S, dtype, seed=17).to(DEV)
    with pytest.raises(ValueError, match="heads\\[0\\] is on cuda:1"):
        m0.predict_record(x, S, 60.0, heads=[other])
    lib, h = m0._ensure_handle()
    arr = (ctypes.c_void_p * 1)(other._ensure_handle()[1].value)
    ws = torch.empty(1 << 24, dtype=torch.uint8, device=DEV)
    out = torch.empty(2, 1, 2, device=DEV)
    rc = lib.b2cnn_score_record_heads(h, arr, 1, x.data_ptr(), capi.DTYPE_BF16, 1, x.shape[2], x.shape[2], S, capi.PATH_AUTO,
                                      capi.MODE_INDEPENDENT, torch.tensor([60.0], device=DEV).data_ptr(), 1, 0, out.data_ptr(), None,
                                      None, ws.data_ptr(), ws.numel(), None)
    assert rc == capi.EINVAL and "another device" in capi.last_error()
