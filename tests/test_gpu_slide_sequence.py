"""GPU: SlidingScorer(mode="sequence") -- each patient scored as utils.run_model scores a recording, live: its LSTM state
carried from one scored window to the next.

The identity checked throughout: for a patient whose stream is s (history first), s0 its samples_seen at the first push
with samples_seen >= W and o = s0 - W, the push at samples_seen == s0 + j S returns
predict_record(s[:, :, o : s0 + j S], S, age, mode="sequence")[:, j] -- bit for bit (NaN for NaN) on the generic
path, and on the tensor-core path within BETA_TC_SEQ of the float64 sequence truth.  predict_record is causal bit for
bit (tests/test_gpu_record_sequence.py), so column j of one call over the whole stream stands for every prefix.

Also: the front end is untouched (features() equal to an independent scorer's), a patient's result does not depend on
P or on the run, the lifecycle (admit with any history, discharge, re-admit), NaN and +-inf, ages, export / restore
with the LSTM state, return_prob, reset, heads refused, the launch list of a push and errors raised before any launch."""
import collections
import ctypes
import json
import os
import subprocess
import sys

import pytest
import torch

import tskd_b200
from test_gpu_record import _records, _tc_pair
from test_gpu_record_sequence import BETA_TC_SEQ, _check, _truth
from test_gpu_slide_generic import _golden, _pair as _generic_pair, _same
from oracle.train_ref import BETA
from tskd_b200 import capi

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
BF, F32 = torch.bfloat16, torch.float32


def _pushes(sc, x, S, age, prob=False, start=0):
    """push x [P, C, N] S samples at a time from sample `start`; the outputs (None or [P]) of every push"""
    return [sc.push(x[:, :, i:i + S], age=age, return_prob=prob) for i in range(start, x.shape[2] - S + 1, S)]


def _s0(W, S, H=0):
    """samples_seen at the first push with samples_seen >= W, for a stream admitted with H history samples"""
    return H + max(1, -(-(W - H) // S)) * S


def _stack(outs):
    return torch.stack([o for o in outs if o is not None], dim=1)           # [P, scored pushes]


def _expect(m, s, S, age, path, H=0, prob=False):
    """[P, J]: the identity's right-hand side for streams s [P, C, H + pushes] admitted with H history samples (0: from
    reset), J the scored pushes"""
    W = m.arch.window
    o = _s0(W, S, H) - W
    return m.predict_record(s[:, :, o:], S, age, path=path, mode="sequence", return_prob=prob)


def _scorer(m, P, S, dtype, path, mode="sequence"):
    return tskd_b200.SlidingScorer(m, P, S, dtype=dtype, path=path, mode=mode)


# ------------------------------------------------------------------ 1. generic path, bit for bit
@pytest.mark.parametrize("dtype", [F32, BF], ids=["f32", "bf16"])
@pytest.mark.parametrize("S", [4, 12, 120])
@pytest.mark.parametrize("P", [1, 3, 130])
def test_generic_golden_bit_identical(dtype, S, P):
    _, m = _golden(5)
    W = 120
    n = _s0(W, S) // S + 8
    x = _records(P, 10, n * S, dtype, seed=S + P).to(DEV)
    age = tskd_b200.synth.make_ages(P, seed=S).to(DEV)
    sc = _scorer(m, P, S, dtype, "generic")
    assert sc.mode == "sequence" and sc.path == "generic"
    outs = _pushes(sc, x, S, age)
    assert all(o is None for o in outs[:_s0(W, S) // S - 1])
    got = _stack(outs)
    want = _expect(m, x, S, age, "generic")
    assert got.shape == want.shape == (P, 9) and _same(got, want)
    # one prefix call per push, as the identity states it
    o = _s0(W, S) - W
    for j in (0, 4):
        assert _same(got[:, j], m.predict_record(x[:, :, o:_s0(W, S) + j * S], S, age, path="generic", mode="sequence")[:, j])


@pytest.mark.parametrize("case", ["c10-relu-affine", "pool44"])
def test_generic_models(case):
    if case == "c10-relu-affine":
        geo, act, aff_seed, S = (10, 10, 5, 3, 2, 200), "relu", 7, 24
    else:
        geo, act, aff_seed, S = (3, 5, 5, 4, 4, 250), "tanh", None, 32                     # W % 16 != 0
    _, m, _ = _generic_pair(geo, act=act, aff_seed=aff_seed, seed=11)
    W = geo[5]
    for dtype in (F32, BF):
        x = _records(3, geo[0], _s0(W, S) + 7 * S, dtype, seed=5).to(DEV)
        age = tskd_b200.synth.make_ages(3, seed=5).to(DEV)
        got = _stack(_pushes(_scorer(m, 3, S, dtype, "generic"), x, S, age))
        assert _same(got, _expect(m, x, S, age, "generic")), (case, dtype)


# ------------------------------------------------------------------ 2. tensor cores against float64
TC_CASES = {
    "m5-bf16-w7504-s752-p3": ("mycnn5", 3, BF, 7504, 752, 3, 8),
    "m5-bf16-w7504-s752-p1": ("mycnn5", 3, BF, 7504, 752, 1, 12),
    "m5-bf16-w7504-s7504-p130": ("mycnn5", 3, BF, 7504, 7504, 130, 4),
    "m3-f32-w7502-s752-p130": ("mycnn3", 1, F32, 7502, 752, 130, 5),
    "m3-f32-w7502-s752-p3": ("mycnn3", 1, F32, 7502, 752, 3, 10),
}


@pytest.mark.parametrize("name", sorted(TC_CASES))
def test_tensorcore_against_float64(name):
    kind, C, dtype, W, S, P, J = TC_CASES[name]
    seed = 700 + sorted(TC_CASES).index(name)
    ref, m = _tc_pair(kind, C, W, seed)
    x = _records(P, C, _s0(W, S) + (J - 1) * S, dtype, seed=seed).to(DEV)
    age = tskd_b200.synth.make_ages(P, seed=seed).to(DEV)
    sc = _scorer(m, P, S, dtype, "tensorcore")
    got = _stack(_pushes(sc, x, S, age))
    assert got.shape == (P, J)
    o = _s0(W, S) - W
    t, t32 = _truth(ref, x[:, :, o:], S, age)
    _check([(name, got, t, t32, BETA_TC_SEQ)])


def test_tensorcore_long_window():
    """MyCNN5 at W = 75000, S = 7500 (600 s every 60 s at 125 Hz): 31 scored pushes"""
    W, S, P, J = 75000, 7500, 2, 31
    ref, m = _tc_pair("mycnn5", 3, W, 741)
    x = _records(P, 3, W + (J - 1) * S, BF, seed=741).to(DEV)
    age = torch.tensor([55.0, 81.0], device=DEV)
    got = _stack(_pushes(_scorer(m, P, S, BF, "tensorcore"), x, S, age))
    assert got.shape == (P, J)
    t, t32 = _truth(ref, x, S, age)
    _check([("long", got, t, t32, BETA_TC_SEQ)])


# ------------------------------------------------------------------ 3. the front end is untouched; 4. independence
@pytest.mark.parametrize("path", ["tensorcore", "generic"])
def test_features_and_independence(path):
    W, S = 7504, 1876
    _, m = _tc_pair("mycnn5", 3, W, 61)
    x = _records(130, 3, W + 5 * S, BF, seed=61).to(DEV)
    age = tskd_b200.synth.make_ages(130, seed=61).to(DEV)
    seq, ind = _scorer(m, 130, S, BF, path), _scorer(m, 130, S, BF, path, mode="independent")
    outs = []
    for i in range(0, x.shape[2], S):
        outs.append(seq.push(x[:, :, i:i + S], age=age))
        ind.push(x[:, :, i:i + S], age=age)
        if outs[-1] is not None:
            assert torch.equal(seq.features(), ind.features()), (path, i)
    full = _stack(outs)
    alone = _stack(_pushes(_scorer(m, 1, S, BF, path), x[7:8], S, age[7:8]))
    assert torch.equal(full[7:8], alone), path
    assert torch.equal(_stack(_pushes(_scorer(m, 130, S, BF, path), x, S, age)), full), path        # a second run
    if path == "generic":
        assert _same(full, _expect(m, x, S, age, "generic"))


# ------------------------------------------------------------------ 5. lifecycle
def _admit_case(path, m, S, dtype):
    """Twin scorers of P = 6; `sc` admits patients 1 (no history, before the first window), 2 (H = W - S, at push 1),
    3 (H = W, unaligned view, at the first window), 4 (H = S + R, later) and discharges then re-admits patient 5.  Returns the
    pieces each patient's identity needs."""
    W, P = m.arch.window, 6
    R = 24 if path == "tensorcore" else m.arch.pool_s * (m.arch.pool_k + m.arch.k2 - 2) + m.arch.pool_k + m.arch.k1 - 1
    n0 = _s0(W, S) // S
    n_push = 2 * n0 + 5
    x = _records(P, m.arch.in_channels, n_push * S, dtype, seed=S).to(DEV)
    hist_base = _records(P, m.arch.in_channels, W + 1, dtype, seed=S + 1).to(DEV)
    age = tskd_b200.synth.make_ages(P, seed=S).to(DEV)
    plan = {1: (0, 0), 2: (1, W - S), 3: (n0 - 1, W), 4: (n0 + 2, S + R)}          # patient: (pushes before, H)
    sc, twin = _scorer(m, P, S, dtype, path), _scorer(m, P, S, dtype, path)
    outs, touts = [], []
    dis_at, re_at = 2, n0 + 1
    for n in range(n_push):
        for p, (at, H) in plan.items():
            if n == at:
                sc.admit([p], hist_base[p:p + 1, :, 1:H + 1] if H else None)            # offset 1: an unaligned view
        if n == dis_at:
            sc.discharge([5])
        if n == re_at:
            sc.admit([5])
        outs.append(sc.push(x[:, :, n * S:(n + 1) * S], age=age))
        touts.append(twin.push(x[:, :, n * S:(n + 1) * S], age=age))
    return W, x, hist_base, age, plan, (dis_at, re_at), outs, touts


@pytest.mark.parametrize("path", ["generic", "tensorcore"])
def test_lifecycle(path):
    if path == "generic":
        ref, m = _golden(5)
        S, dtype = 12, F32
    else:
        ref, m = _tc_pair("mycnn5", 3, 7504, 81)
        S, dtype = 1876, BF
    W, x, hist, age, plan, (dis_at, re_at), outs, touts = _admit_case(path, m, S, dtype)
    for p, (at, H) in list(plan.items()) + [(5, (re_at, 0))]:
        s = torch.cat([hist[p:p + 1, :, 1:H + 1], x[p:p + 1, :, at * S:]], dim=2)
        first = at + (_s0(W, S, H) - H) // S - 1                                         # the push index of s0
        got = torch.stack([outs[n][p] for n in range(first, len(outs))]).reshape(1, -1)
        for n in range(at, first):
            assert outs[n] is None or torch.isnan(outs[n][p]), (p, n)
        want = _expect(m, s, S, age[p:p + 1], path, H=H)
        assert got.shape == want.shape, (p, got.shape, want.shape)
        if path == "generic":
            assert _same(got, want), p
        else:
            o = _s0(W, S, H) - W
            t, t32 = _truth(ref, s[:, :, o:], S, age[p:p + 1])
            _check([(f"admit-{p}", got, t, t32, BETA_TC_SEQ)])
    for n in range(dis_at, re_at + _s0(W, S) // S - 1):
        assert outs[n] is None or torch.isnan(outs[n][5]), n                          # discharged, then filling again
    for n, (o, t) in enumerate(zip(outs, touts)):                                     # patient 0 is never touched
        if t is not None:
            assert o is not None and _same(o[0], t[0]), n


# ------------------------------------------------------------------ 6. NaN and +-inf
def test_nan_poisons_until_admit():
    _, m = _golden(5)
    W, S, P = 120, 12, 4
    n_push = _s0(W, S) // S + 10
    x = _records(P, 10, n_push * S, F32, seed=3).to(DEV)
    pos = _s0(W, S) + 3 * S + 5                                                        # inside the 4th scored push
    bad = x.clone()
    bad[1, 4, pos] = float("nan")
    age = tskd_b200.synth.make_ages(P, seed=3).to(DEV)
    sc, clean = _scorer(m, P, S, F32, "generic"), _scorer(m, P, S, F32, "generic")
    readmit = n_push - 3
    outs, couts = [], []
    for n in range(n_push):
        if n == readmit:
            sc.admit([1], x[1:2, :, n * S - W:n * S])
        outs.append(sc.push(bad[:, :, n * S:(n + 1) * S], age=age))
        couts.append(clean.push(x[:, :, n * S:(n + 1) * S], age=age))
    got = _stack(outs[:readmit])
    want = _expect(m, bad[:, :, :readmit * S], S, age, "generic")
    assert _same(got, want)
    j_nan = (pos + 1 - _s0(W, S) + S - 1) // S                                        # the first window holding pos
    assert torch.isfinite(got[1, :j_nan]).all() and torch.isnan(got[1, j_nan:]).all()
    for n in range(n_push):
        if outs[n] is not None:
            keep = [0, 2, 3]
            assert torch.equal(outs[n][keep], couts[n][keep]), n
    # admit clears the state: patient 1 from its readmission is a fresh stream with a full-window history
    s = x[1:2, :, readmit * S - W:]
    after = torch.stack([outs[n][1] for n in range(readmit, n_push)]).reshape(1, -1)
    assert torch.isfinite(after).all()
    assert _same(after, _expect(m, s, S, age[1:2], "generic", H=W))


def test_inf_follows_the_truth():
    W, S, P = 7504, 1876, 3
    ref, m = _tc_pair("mycnn5", 3, W, 91)
    x = _records(P, 3, W + 6 * S, BF, seed=91)
    x[0, 1, W + 2 * S + 17] = float("inf")
    x[2, 0, 100] = -float("inf")
    age = tskd_b200.synth.make_ages(P, seed=91).to(DEV)
    x = x.to(DEV)
    t, t32 = _truth(ref, x, S, age)
    for path in ("tensorcore", "generic"):
        got = _stack(_pushes(_scorer(m, P, S, BF, path), x, S, age))
        _check([(f"inf-{path}", got, t, t32, BETA_TC_SEQ if path == "tensorcore" else BETA)])
        if path == "generic":
            assert _same(got, _expect(m, x, S, age, "generic"))


# ------------------------------------------------------------------ 7. ages
@pytest.mark.parametrize("path", ["generic", "tensorcore"])
def test_age_scales_the_output_only(path):
    W, S, P = 7504, 1876, 3
    _, m = _tc_pair("mycnn5", 3, W, 95)
    x = _records(P, 3, W + 6 * S, BF, seed=95).to(DEV)
    a1, a2 = torch.tensor([30.0, 50.0, 70.0], device=DEV), torch.tensor([90.0, 20.0, 40.0], device=DEV)
    k = _s0(W, S) // S + 2
    s1, s2 = _scorer(m, P, S, BF, path), _scorer(m, P, S, BF, path)
    for n in range(x.shape[2] // S):
        seg = x[:, :, n * S:(n + 1) * S]
        o1, o2 = s1.push(seg, age=a1 if n < k else 61.0), s2.push(seg, age=a2 if n < k else 61.0)
        if n >= k:
            assert torch.equal(o1, o2), (path, n)
        elif o1 is not None:
            assert not torch.equal(o1, o2)


# ------------------------------------------------------------------ 8. export and restore
@pytest.mark.parametrize("path", ["generic", "tensorcore"])
def test_export_restore_continues(path):
    W, S = 7504, 1876
    _, m = _tc_pair("mycnn5", 3, W, 97)
    PA, PB = 5, 7
    n_a = _s0(W, S) // S + 3
    x = _records(PA, 3, (n_a + 5) * S, BF, seed=97).to(DEV)
    y = _records(PB, 3, 9 * S, BF, seed=98).to(DEV)
    age = tskd_b200.synth.make_ages(PA, seed=97).to(DEV)
    A, B = _scorer(m, PA, S, BF, path), _scorer(m, PB, S, BF, path)
    _pushes(A, x[:, :, :n_a * S], S, age)
    _pushes(B, y, S, 50.0)                                                            # another push count
    A.discharge([3])
    move, slots = [0, 2, 3], [6, 1, 4]
    state = A.export(move)
    assert state["lstm"].shape == (3, 2, 2, 16) and state["lstm"].dtype == F32 and state["lstm"].device == torch.device(DEV)
    assert torch.count_nonzero(state["lstm"][0]) > 0 and torch.count_nonzero(state["lstm"][2]) == 0
    B.restore(slots, state)
    ageB = torch.full((PB,), 45.0, device=DEV)
    ageB[slots] = age[move]
    for n in range(n_a, n_a + 5):
        oa = A.push(x[:, :, n * S:(n + 1) * S], age=age)
        segB = _records(PB, 3, S, BF, seed=200 + n).to(DEV)
        segB[slots] = x[move, :, n * S:(n + 1) * S]
        ob = B.push(segB, age=ageB)
        assert _same(ob[slots], oa[move]), (path, n)
        assert torch.isnan(ob[4]).all()
    ind = _scorer(m, PB, S, BF, path, mode="independent")
    with pytest.raises(ValueError, match="another mode"):
        ind.restore(slots, state)
    plain = ind.export([0])
    with pytest.raises(ValueError, match="another mode"):
        B.restore([0], plain)


def test_import_without_state_zeroes_the_rows():
    """b2cnn_slide_import (no LSTM array) into a sequence scorer: the patients' LSTM starts from zero, as restoring the
    same state with lstm = 0 does"""
    W, S, P = 7504, 1876, 3
    _, m = _tc_pair("mycnn5", 3, W, 99)
    x = _records(P, 3, W + 6 * S, BF, seed=99).to(DEV)
    A = _scorer(m, P, S, BF, "tensorcore")
    n_a = _s0(W, S) // S + 2
    _pushes(A, x[:, :, :n_a * S], S, 60.0)
    state = A.export(range(P))
    zero = dict(state, lstm=torch.zeros_like(state["lstm"]))
    B, Z = _scorer(m, P, S, BF, "tensorcore"), _scorer(m, P, S, BF, "tensorcore")
    _pushes(B, x[:, :, :n_a * S], S, 60.0)                                             # a non-zero state to overwrite
    Z.restore(range(P), zero)
    lib, hdr = B._lib, capi.SlideStateHeader(**{n: int(state[n]) for n in B.STATE_HEADER})
    arr = (ctypes.c_int32 * P)(*range(P))
    ws = torch.empty(int(lib.b2cnn_slide_state_workspace_bytes(B._s, P)), dtype=torch.uint8, device=DEV)
    st = torch.cuda.current_stream().cuda_stream
    assert lib.b2cnn_slide_import(B._s, arr, P, ctypes.byref(hdr), state["features"].data_ptr(), state["tail"].data_ptr(),
                                  state["seen"].data_ptr(), ws.data_ptr(), ws.numel(), st) == 0, capi.last_error()
    assert torch.equal(B.export(range(P))["lstm"], zero["lstm"])
    for n in range(n_a, n_a + 3):
        seg = x[:, :, n * S:(n + 1) * S]
        assert torch.equal(B.push(seg, age=60.0), Z.push(seg, age=60.0)), n


# ------------------------------------------------------------------ 9. probabilities, reset and heads
def test_prob_reset_and_heads():
    ref, m = _golden(5)
    W, S, P = 120, 12, 3
    x = _records(P, 10, W + 8 * S, F32, seed=13).to(DEV)
    age = tskd_b200.synth.make_ages(P, seed=13).to(DEV)
    sc = _scorer(m, P, S, F32, "generic")
    prob = _stack(_pushes(sc, x, S, age, prob=True))
    assert _same(prob, _expect(m, x, S, age, "generic", prob=True))
    t, t32 = _truth(ref, x, S, age, prob=True)
    _check([("prob", prob, t, t32, BETA)])
    sc.reset()                                                                        # every state back to zero
    assert torch.count_nonzero(sc.export(range(P))["lstm"]) == 0
    assert _same(_stack(_pushes(sc, x, S, age, prob=True)), prob)
    with pytest.raises(ValueError, match="heads"):
        sc.set_heads([m])
    lib = sc._lib
    h = m._ensure_handle()[1]
    arr = (ctypes.c_void_p * 1)(h.value)
    assert lib.b2cnn_slide_set_heads(sc._s, arr, 1, None) == capi.EINVAL
    assert lib.b2cnn_slide_set_heads_ex(sc._s, arr, 1, 0, None) == capi.EINVAL
    assert lib.b2cnn_slide_n_heads(sc._s) == 0
    sc.set_heads([])
    sc.reset()
    outs = [sc.push(x[:, :, i:i + S], age=age, heads=True) for i in range(0, x.shape[2], S)]
    got = torch.cat([o for o in outs if o is not None], dim=0).T                       # [1, P] per push
    assert _same(got, _expect(m, x, S, age, "generic"))


# ------------------------------------------------------------------ 10. the launch list of a push
_LAUNCH_LIST = r"""
import collections, json, sys
import torch
import tskd_b200
from oracle import mycnn_torch as O
from torch.profiler import ProfilerActivity, profile

def kernels(fn):
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        torch.ones(1, device=dev).add_(1)
        torch.cuda.synchronize()
        fn()
        torch.cuda.synchronize()
    return collections.Counter(e.name for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA
                               and ("b2cnn::" in e.name or e.name.startswith("Memset")))

path, W, S = sys.argv[1], 7504, 1876
dev = torch.device("cuda", 0)
ref = O.make_ref(O.stretched(O.ARCH_MYCNN5, 3, W), seed=91)
m = tskd_b200.B200MyCNN(tskd_b200.ARCH_PRESETS["mycnn5"].with_shape(3, W), has_out12=ref.arch.has_out12).to(dev)
m.load_state_dict(ref.state_dict())
kernels(lambda: torch.ones(1, device=dev).add_(1))                  # profiler warm-up
first = -(-W // S)
res = []
for P, n in ((1, first), (257, first), (257, 40)):
    x = tskd_b200.synth.make_windows(P, 3, S, "normal", seed=P, dtype=torch.bfloat16).to(dev)
    row = {}
    for mode in ("sequence", "independent"):
        sc = tskd_b200.SlidingScorer(m, P, S, path=path, mode=mode)
        for _ in range(n - 1):
            sc.push(x, age=60.0)
        row[mode] = kernels(lambda: sc.push(x, age=60.0))
    res.append(row)
print(json.dumps(res))
"""


@pytest.mark.parametrize("path", ["tensorcore", "generic"])
def test_launch_list(path):
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    env = dict(os.environ, PYTHONPATH=os.pathsep.join([root] + [p for p in [os.environ.get("PYTHONPATH")] if p]))
    cmd = [sys.executable] + (["-s"] if sys.flags.no_user_site else []) + ["-c", _LAUNCH_LIST, path]
    r = subprocess.run(cmd, capture_output=True, text=True, env=env, cwd=root, timeout=600)
    assert r.returncode == 0, r.stderr[-3000:]
    res = json.loads(r.stdout.strip().splitlines()[-1])
    heads = ("head_reduce_independent_kernel",) if path == "tensorcore" else ("reduce_gates_kernel", "head_independent_kernel")
    # whatever P and n; on the generic path the front end's launches follow the ring's wrap, in both modes alike
    seq = [collections.Counter({k: v for k, v in row["sequence"].items() if path == "tensorcore" or "frontend" not in k}) for row in res]
    assert all(s == seq[0] for s in seq), seq
    for row in res:
        ind, sq = collections.Counter(row["independent"]), collections.Counter(row["sequence"])
        step = [k for k in sq if "slide_seq_step_kernel" in k]
        assert len(step) == 1 and sq[step[0]] == 1, sq
        hk = [k for k in ind if any(h in k for h in heads)]
        assert len(hk) == len(heads) and all(ind[k] == 1 for k in hk), ind
        assert ind - collections.Counter(hk) == sq - collections.Counter(step), (ind, sq)


# ------------------------------------------------------------------ 11. errors before any launch
def test_errors_leave_the_scorer_usable():
    _, m = _golden(5)
    W, S, P = 120, 12, 3
    x = _records(P, 10, W + 4 * S, F32, seed=17).to(DEV)
    for bad in ("seq", None, 1, "Sequence"):
        with pytest.raises(ValueError, match="mode"):
            tskd_b200.SlidingScorer(m, P, S, dtype=F32, path="generic", mode=bad)
    lib, h = m._ensure_handle()
    s = ctypes.c_void_p()
    for bad in (2, -1):
        assert lib.b2cnn_slide_create_ex(h, P, S, capi.DTYPE_F32, capi.PATH_GENERIC, bad, ctypes.byref(s)) == capi.EINVAL
        assert "mode" in capi.last_error() and not s.value
    assert lib.b2cnn_slide_mode(None) == -1
    seq, ind = _scorer(m, P, S, F32, "generic"), _scorer(m, P, S, F32, "generic", mode="independent")
    assert lib.b2cnn_slide_mode(seq._s) == capi.MODE_SEQUENCE and lib.b2cnn_slide_mode(ind._s) == capi.MODE_INDEPENDENT
    _pushes(seq, x[:, :, :W], S, 60.0)
    _pushes(ind, x[:, :, :W], S, 60.0)
    ref_seq = _scorer(m, P, S, F32, "generic")
    _pushes(ref_seq, x[:, :, :W], S, 60.0)
    # a non-null lstm array for an independent scorer, on export and import
    k = 2
    arr = (ctypes.c_int32 * k)(0, 1)
    state = ind.export([0, 1])
    feats, tail, seen = state["features"], state["tail"], state["seen"]
    lstm = torch.full((k, 2, 2, 16), 7.0, device=DEV)
    hdr = capi.SlideStateHeader()
    ws = torch.empty(256, dtype=torch.uint8, device=DEV)
    st = torch.cuda.current_stream().cuda_stream
    f2 = torch.full_like(feats, 3.0)
    assert lib.b2cnn_slide_export_ex(ind._s, arr, k, f2.data_ptr(), tail.data_ptr(), seen.data_ptr(), lstm.data_ptr(), ctypes.byref(hdr),
                                     ws.data_ptr(), 256, st) == capi.EINVAL
    hdr = capi.SlideStateHeader(**{n: int(state[n]) for n in ind.STATE_HEADER})
    assert lib.b2cnn_slide_import_ex(ind._s, arr, k, ctypes.byref(hdr), feats.data_ptr(), tail.data_ptr(), seen.data_ptr(),
                                     lstm.data_ptr(), ws.data_ptr(), 256, st) == capi.EINVAL
    torch.cuda.synchronize()
    assert (f2 == 3.0).all() and (lstm == 7.0).all()                                 # nothing written
    # wrongly shaped or typed "lstm"
    good = seq.export([0, 1])
    for bad in (good["lstm"][:1], good["lstm"].reshape(2, 4, 16), good["lstm"].double(), good["lstm"].tolist()):
        with pytest.raises(ValueError):
            seq.restore([0, 1], dict(good, lstm=bad))
    for n in range(W // S, W // S + 4):                                              # both still as before
        seg = x[:, :, n * S:(n + 1) * S]
        assert _same(seq.push(seg, age=60.0), ref_seq.push(seg, age=60.0)), n
        assert ind.push(seg, age=60.0) is not None
