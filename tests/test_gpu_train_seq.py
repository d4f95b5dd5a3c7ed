"""GPU: many patients' window sequences in one call (seq_lengths).  The batch is N consecutive sequences, each scanned
by the LSTM from the zero state; the truth is one call of the reference module per sequence, concatenated
(oracle/train_seq_ref.py), compared element by element in float64 with the float32 graph as the yardstick
(oracle/train_ref.py: assert_close_elem) at the grants of test_gpu_train_edges.py.  Then the identities ([B] is
today's sequence mode, [1] * B independent mode), the absence of leakage between sequences, determinism, Adam, the frozen
front end, the launch list, the inference path and the refusals."""
import collections
import ctypes
import json
import os
import subprocess
import sys
from dataclasses import replace

import numpy as np
import pytest
import torch
from torch import nn

import tskd_b200
from tskd_b200 import capi
from tskd_b200.arch import BLOB_KEYS
from tskd_b200.trainer import B200Trainer
from oracle import mycnn_torch as O
from oracle.train_ref import BETA, MaskDropout, assert_close_elem, check_elems, train_reference
from oracle.train_seq_ref import train_reference_seq

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
POS_WEIGHT = 13.5
# the grants of tests/test_gpu_train_edges.py: the LSTM's recurrent sums (LSTM_BETA) and, from B = 257 on, the conv
# gradients' long cancelling sums (BIG_B_BETA); every other element at BETA
LSTM_BETA = {k: 4e-6 for k in BLOB_KEYS if k.startswith("lstm.")}
BIG_B_BETA = {k: 4e-6 for k in ("conv1.weight", "conv1.bias", "conv2.weight", "conv2.bias")}
# and, for waveform windows, tests/test_gpu_train_long.py's LONG_SUM_BETA (the conv backward's long sums over a window)
LONG_SUM_BETA = {k: 4e-6 for k in ("conv1.weight", "conv2.weight", "dx")}


def _pair(kind, C, W, seed=0, trainable=False):
    oarch = O.stretched(O.ARCHS[kind], C, W)
    ref = O.make_ref(oarch, seed=seed)
    ref.dropout = MaskDropout()
    ref.train()
    arch = replace(tskd_b200.ARCH_PRESETS[kind].with_shape(C, W), age_coef=oarch.age_coef)
    cls = tskd_b200.B200TrainableMyCNN if trainable else tskd_b200.B200MyCNN
    m = cls(arch, has_out12=oarch.has_out12).to(DEV)
    m.load_state_dict({k: v for k, v in ref.state_dict().items() if not k.startswith("dropout")})
    if trainable:
        m.dropout.p = oarch.dropout
    return oarch, ref, m


def _batch(oarch, B, seed, p):
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(B, oarch.in_channels, oarch.window, generator=g)
    age = torch.rand(B, generator=g) * 60 + 20
    y = (torch.rand(B, generator=g) > 0.5).float()
    if p > 0:
        m1 = torch.bernoulli(torch.full((B, 4, oarch.p1), 1 - p), generator=g) / (1 - p)
        m2 = torch.bernoulli(torch.full((B, oarch.l_out), 1 - p), generator=g) / (1 - p)
    else:
        m1 = m2 = None
    return x, age, y, m1, m2


def _lengths(n, lo, hi, seed):
    return torch.randint(lo, hi + 1, (n,), generator=torch.Generator().manual_seed(seed)).tolist()


def _dev(t):
    return None if t is None else t.to(DEV)


def _params(m):
    named = dict(m.named_parameters())
    return [named[k] for k in BLOB_KEYS]


def _check(label, got, truth, ref32, B, W=120):
    beta = {**LSTM_BETA, **(BIG_B_BETA if B >= 257 else {}), **(LONG_SUM_BETA if W > 1000 else {})}
    pairs = [(k, got[k], truth["grads"][k], ref32["grads"][k], beta.get(k, BETA)) for k in BLOB_KEYS]
    for k in ("loss", "dx", "dage"):
        if k in got:
            t, r = truth[k].reshape(-1), ref32[k].reshape(-1)
            pairs.append((k, got[k].reshape(-1), t, r, beta.get(k, BETA)))
    check_elems(pairs, label)


# (kind, C, W, lengths, dropout): mixed lengths at the training shape; the older revision; a waveform window of several
# conv tiles; and N = 300 > 256 sequences, where a scan CTA takes two consecutive sequences
CASES = [
    ("mycnn5", 10, 120, [1, 7, 32, 3, 1, 20], 0.1),
    ("mycnn5", 10, 120, [1, 7, 32, 3, 1, 20], 0.0),
    ("mycnn2", 7, 120, [5, 1, 10, 2], 0.5),
    ("mycnn5", 3, 7504, [2, 1, 3], 0.1),
    ("mycnn5", 10, 120, _lengths(300, 1, 3, 7), 0.0),
]
IDS = ["mycnn5-mixed-p0.1", "mycnn5-mixed-p0", "mycnn2-c7", "mycnn5-w7504", "mycnn5-n300-grouped"]


# ------------------------------------------------------------------ 1. against float64, element by element
@pytest.mark.parametrize("kind,C,W,lens,p", CASES, ids=IDS)
@pytest.mark.parametrize("pos_weight", [None, POS_WEIGHT])
def test_fused_step_matches_float64(kind, C, W, lens, p, pos_weight):
    oarch, ref, m = _pair(kind, C, W)
    B = sum(lens)
    x, age, y, m1, m2 = _batch(oarch, B, seed=5, p=p)
    tr = B200Trainer(m, dropout=p, pos_weight=pos_weight)
    loss = tr.step(x, age, y, masks=(m1, m2), update=False, seq_lengths=lens)
    head = "bce" if pos_weight is None else "bce_pw"
    truth = train_reference_seq(ref, x, age, lens, m1, m2, target=y, pos_weight=pos_weight)[head]
    ref32 = train_reference_seq(ref, x, age, lens, m1, m2, target=y, pos_weight=pos_weight, dtype=torch.float32)[head]
    _check(f"fused {kind} {C}x{W} N={len(lens)} {head}", {**tr.grads(), "loss": loss.cpu()}, truth, ref32, B, W)


@pytest.mark.parametrize("kind,C,W,lens,p", CASES, ids=IDS)
def test_autograd_matches_float64(kind, C, W, lens, p):
    oarch, ref, m = _pair(kind, C, W, trainable=True)
    B = sum(lens)
    x, age, _, m1, m2 = _batch(oarch, B, seed=6, p=p)
    r = torch.randn(B, generator=torch.Generator().manual_seed(9))
    xd, ad = x.to(DEV).requires_grad_(), age.to(DEV).requires_grad_()
    z = tskd_b200.mycnn_train_forward(xd, ad, _params(m), m.arch, "sequence", _dev(m1), _dev(m2), seq_lengths=lens)
    (z * r.to(DEV)).sum().backward()
    full = train_reference_seq(ref, x, age, lens, m1, m2, dz=r)
    full32 = train_reference_seq(ref, x, age, lens, m1, m2, dz=r, dtype=torch.float32)
    assert_close_elem("z", z, full["z"], full32["z"])
    named = dict(m.named_parameters())
    _check(f"autograd {kind} {C}x{W} N={len(lens)}", {**{k: named[k].grad for k in BLOB_KEYS}, "dx": xd.grad, "dage": ad.grad},
           full["dz"], full32["dz"], B, W)


# ------------------------------------------------------------------ 2. identities
@pytest.mark.parametrize("pos_weight", [None, POS_WEIGHT])
def test_one_sequence_is_todays_sequence_mode_bit_for_bit(pos_weight):
    oarch, _, m = _pair("mycnn5", 10, 120)
    _, _, m_b = _pair("mycnn5", 10, 120)
    B = 48
    tr_a = B200Trainer(m, lr=1e-3, dropout=0.1, pos_weight=pos_weight)
    tr_b = B200Trainer(m_b, lr=1e-3, dropout=0.1, pos_weight=pos_weight)
    for step in range(2):
        x, age, y, m1, m2 = _batch(oarch, B, seed=30 + step, p=0.1)
        la = tr_a.step(x, age, y, masks=(m1, m2))
        lb = tr_b.step(x, age, y, masks=(m1, m2), seq_lengths=[B])
        assert torch.equal(la, lb)
        assert torch.equal(tr_a._grads, tr_b._grads)
        assert torch.equal(tr_a._params, tr_b._params) and torch.equal(tr_a._m, tr_b._m) and torch.equal(tr_a._v, tr_b._v)


def test_one_sequence_through_autograd_bit_for_bit():
    oarch, _, m = _pair("mycnn5", 3, 1528, trainable=True)
    x, age, _, m1, m2 = _batch(oarch, 12, seed=8, p=0.1)
    r = torch.randn(12, generator=torch.Generator().manual_seed(2)).to(DEV)
    outs = []
    for lens in (None, [12], torch.tensor([12])):
        for p in m.parameters():
            p.grad = None
        xd, ad = x.to(DEV).requires_grad_(), age.to(DEV).requires_grad_()
        z = tskd_b200.mycnn_train_forward(xd, ad, _params(m), m.arch, "sequence", _dev(m1), _dev(m2), seq_lengths=lens)
        (z * r).sum().backward()
        outs.append([z.detach(), xd.grad, ad.grad] + [dict(m.named_parameters())[k].grad.clone() for k in BLOB_KEYS])
    for other in outs[1:]:
        assert all(torch.equal(a, b) for a, b in zip(outs[0], other))


def test_all_ones_is_independent_mode():
    oarch, ref, m = _pair("mycnn5", 10, 120, trainable=True)
    B = 40
    x, age, _, m1, m2 = _batch(oarch, B, seed=12, p=0.1)
    r = torch.randn(B, generator=torch.Generator().manual_seed(3))
    xd, ad = x.to(DEV).requires_grad_(), age.to(DEV).requires_grad_()
    z = tskd_b200.mycnn_train_forward(xd, ad, _params(m), m.arch, "sequence", _dev(m1), _dev(m2), seq_lengths=[1] * B)
    zi = tskd_b200.mycnn_train_forward(x.to(DEV), age.to(DEV), _params(m), m.arch, "independent", _dev(m1), _dev(m2))
    assert torch.equal(z.detach(), zi.detach())
    (z * r.to(DEV)).sum().backward()
    truth = train_reference(ref, x, age, "independent", m1, m2, dz=r)["dz"]
    ref32 = train_reference(ref, x, age, "independent", m1, m2, dz=r, dtype=torch.float32)["dz"]
    named = dict(m.named_parameters())
    _check("ones", {**{k: named[k].grad for k in BLOB_KEYS}, "dx": xd.grad, "dage": ad.grad}, truth, ref32, B)


# ------------------------------------------------------------------ 3. no leakage between sequences
def _autograd_run(m, x, age, lens, m1, m2, r):
    for p in m.parameters():
        p.grad = None
    xd, ad = x.to(DEV).requires_grad_(), age.to(DEV).requires_grad_()
    z = tskd_b200.mycnn_train_forward(xd, ad, _params(m), m.arch, "sequence", _dev(m1), _dev(m2), seq_lengths=lens)
    (z * r.to(DEV)).sum().backward()
    return z.detach(), xd.grad, ad.grad


def test_permuting_the_sequences_permutes_every_per_window_result():
    oarch, ref, m = _pair("mycnn5", 10, 120, trainable=True)
    lens = [4, 1, 9, 2, 6]
    B = sum(lens)
    x, age, _, m1, m2 = _batch(oarch, B, seed=14, p=0.1)
    r = torch.randn(B, generator=torch.Generator().manual_seed(4))
    starts = np.cumsum([0] + lens[:-1])
    order = [3, 0, 4, 2, 1]
    idx = torch.cat([torch.arange(starts[s], starts[s] + lens[s]) for s in order])
    z, dx, dage = _autograd_run(m, x, age, lens, m1, m2, r)
    zp, dxp, dagep = _autograd_run(m, x[idx], age[idx], [lens[s] for s in order], m1[idx], m2[idx], r[idx])
    assert torch.equal(zp, z[idx.to(DEV)]) and torch.equal(dxp, dx[idx.to(DEV)]) and torch.equal(dagep, dage[idx.to(DEV)])
    # the parameter gradients are the same sums in another sequence order: within the grants of the float64 truth
    named = dict(m.named_parameters())
    truth = train_reference_seq(ref, x[idx], age[idx], [lens[s] for s in order], m1[idx], m2[idx], dz=r[idx])["dz"]
    ref32 = train_reference_seq(ref, x[idx], age[idx], [lens[s] for s in order], m1[idx], m2[idx], dz=r[idx], dtype=torch.float32)["dz"]
    _check("permuted", {k: named[k].grad for k in BLOB_KEYS}, truth, ref32, B)


# (lengths, the poisoned sequence, the window in it): one sequence per scan CTA, and N = 300 with two per CTA, where the
# poisoned sequence 150 shares its CTA with sequence 151
@pytest.mark.parametrize("lens,seq,win", [([5, 8, 3, 6], 1, 3), ([2] * 300, 150, 0)], ids=["n4", "n300-grouped"])
def test_a_nan_stays_inside_its_sequence(lens, seq, win):
    oarch, _, m = _pair("mycnn5", 10, 120)
    B = sum(lens)
    x, age, y, _, _ = _batch(oarch, B, seed=15, p=0.0)
    clean = tskd_b200.mycnn_train_forward(x.to(DEV), age.to(DEV), _params(m), m.arch, "sequence", seq_lengths=lens)
    o = sum(lens[:seq])
    xb = x.clone()
    xb[o + win, 2, 40] = float("nan")
    bad = tskd_b200.mycnn_train_forward(xb.to(DEV), age.to(DEV), _params(m), m.arch, "sequence", seq_lengths=lens)
    nan = torch.isnan(bad).cpu()
    want = torch.zeros(B, dtype=torch.bool)
    want[o + win:o + lens[seq]] = True
    assert torch.equal(nan, want), nan
    keep = ~want.to(DEV)
    assert torch.equal(bad[keep], clean[keep])
    # the same through the inference path
    pc = m.predict(x.to(DEV), age.to(DEV), mode="sequence", seq_lengths=lens)
    pb = m.predict(xb.to(DEV), age.to(DEV), mode="sequence", seq_lengths=lens)
    assert torch.equal(torch.isnan(pb).cpu(), want) and torch.equal(pb[keep], pc[keep])


# ------------------------------------------------------------------ 4. determinism, Adam, frozen conv
@pytest.mark.parametrize("n", [64, 512])
def test_two_runs_give_the_same_bits(n):
    oarch, _, m = _pair("mycnn5", 10, 120)
    B = 2048
    x, age, y, m1, m2 = _batch(oarch, B, seed=16, p=0.1)
    lens = [B // n] * n
    runs = []
    for _ in range(2):
        tr = B200Trainer(m, dropout=0.1)
        loss = tr.step(x, age, y, masks=(m1, m2), update=False, seq_lengths=lens)
        runs.append((loss.clone(), tr._grads.clone()))
    assert torch.equal(runs[0][0], runs[1][0]) and torch.equal(runs[0][1], runs[1][1])


def test_three_adam_steps_follow_torch_optim():
    oarch, ref, m = _pair("mycnn5", 10, 120)
    tr = B200Trainer(m, lr=1e-3, dropout=0.1)
    opt = torch.optim.Adam(ref.parameters(), lr=1e-3)
    for step in range(3):
        lens = _lengths(5, 1, 9, 40 + step)
        B = sum(lens)
        x, age, y, m1, m2 = _batch(oarch, B, seed=100 + step, p=0.1)
        loss = tr.step(x, age, y, masks=(m1, m2), seq_lengths=lens)
        opt.zero_grad()
        zs, o = [], 0
        for n in lens:
            ref.dropout.set(m1[o:o + n], m2[o:o + n])
            zs.append(ref(x[o:o + n], age[o:o + n]).reshape(-1))
            o += n
        want = nn.BCEWithLogitsLoss()(torch.cat(zs), y)
        want.backward()
        opt.step()
        assert abs(float(loss) - float(want)) <= 2e-5 * max(1.0, abs(float(want))), (step, float(loss), float(want))
    sd, named = m.state_dict(), dict(ref.named_parameters())
    for k in BLOB_KEYS:
        a, b = sd[k].cpu().numpy().ravel(), named[k].detach().numpy().ravel()
        g = np.abs(named[k].grad.numpy().ravel())
        sel = g > 1e-4 * g.max()
        assert np.abs(a[sel] - b[sel]).max() <= 2e-5, (k, np.abs(a[sel] - b[sel]).max())
        assert np.abs(a - b).max() <= 6.1e-3


def test_frozen_conv_gives_the_same_head_gradients_and_skips_the_conv_backward():
    from torch.profiler import ProfilerActivity, profile
    oarch, _, m = _pair("mycnn5", 10, 120, trainable=True)
    lens = [3, 9, 1, 11]
    x, age, _, m1, m2 = _batch(oarch, sum(lens), seed=17, p=0.1)
    r = torch.randn(sum(lens), generator=torch.Generator().manual_seed(5)).to(DEV)

    def grads():
        for p in m.parameters():
            p.grad = None
        z = tskd_b200.mycnn_train_forward(x.to(DEV), age.to(DEV), _params(m), m.arch, "sequence", _dev(m1), _dev(m2), seq_lengths=lens)
        (z * r).sum().backward()
        return {k: v.grad for k, v in m.named_parameters() if v.grad is not None}

    full = grads()
    m.conv1.requires_grad_(False)
    m.conv2.requires_grad_(False)
    grads()
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        frozen = grads()
        torch.cuda.synchronize()
    names = {e.name for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA}
    assert not any("train_conv_bwd" in n or "train_conv_grad_reduce" in n or "train_dfeat" in n for n in names), names
    assert any("train_head_reduce" in n for n in names), names
    assert set(frozen) == {k for k in full if not k.startswith("conv")}
    for k, v in frozen.items():
        assert torch.equal(v, full[k]), k


# ------------------------------------------------------------------ 5. the launch list does not depend on N
_LAUNCH_LIST = r"""
import collections, json
import torch
import tskd_b200
from torch.profiler import ProfilerActivity, profile
from tskd_b200.trainer import B200Trainer

dev = torch.device("cuda", 0)
def kernels(fn):
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        torch.ones(1, device=dev).add_(1)
        torch.cuda.synchronize()
        fn()
        torch.cuda.synchronize()
    return collections.Counter(e.name for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA
                               and ("b2cnn::" in e.name or e.name.startswith("Memset")))
m = tskd_b200.B200MyCNN(tskd_b200.ARCH_PRESETS["mycnn5"]).to(dev)
tr = B200Trainer(m, dropout=0.0)
g = torch.Generator().manual_seed(0)
B = 1200
x, age, y = torch.randn(B, 10, 120, generator=g).to(dev), torch.full((B,), 60.0, device=dev), torch.zeros(B, device=dev)
kernels(lambda: torch.ones(1, device=dev).add_(1))
res = {"train": [], "predict": []}
for lens in ([600, 600], [1] * B, [B - 63] + [1] * 63, [3] * 400, [7, 1193]):
    tr.step(x, age, y, update=False, seq_lengths=lens)
    res["train"].append(kernels(lambda: tr.step(x, age, y, update=True, seq_lengths=lens)))
    m.predict(x, age, mode="sequence", seq_lengths=lens)
    res["predict"].append(kernels(lambda: m.predict(x, age, mode="sequence", seq_lengths=lens)))
print(json.dumps(res))
"""


def test_launch_list_does_not_depend_on_the_lengths():
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    env = dict(os.environ, PYTHONPATH=os.pathsep.join([root] + [p for p in [os.environ.get("PYTHONPATH")] if p]))
    cmd = [sys.executable] + (["-s"] if sys.flags.no_user_site else []) + ["-c", _LAUNCH_LIST]
    r = subprocess.run(cmd, capture_output=True, text=True, env=env, cwd=root, timeout=600)
    assert r.returncode == 0, r.stderr[-3000:]
    res = json.loads(r.stdout.strip().splitlines()[-1])
    for key in ("train", "predict"):
        lists = [collections.Counter(d) for d in res[key]]
        assert all(c == lists[0] for c in lists), (key, lists)
    assert any("train_head_reduce" in k for k in res["train"][0]), res["train"][0]
    assert any("head_sequence_kernel" in k for k in res["predict"][0]), res["predict"][0]


# ------------------------------------------------------------------ 6. inference
def _per_sequence(m, x, age, lens, **kw):
    outs, o = [], 0
    for n in lens:
        outs.append(m.predict(x[o:o + n], age[o:o + n], mode="sequence", **kw))
        o += n
    return torch.cat(outs)


@pytest.mark.parametrize("path,C,W,dtype", [
    ("generic", 10, 120, torch.float32),
    ("stream", 3, 7504, torch.float32),          # fp32 windows through the streaming kernel
    ("tensorcore", 3, 7504, torch.bfloat16),
    ("generic", 3, 7504, torch.bfloat16),
])
def test_predict_equals_a_per_sequence_loop(path, C, W, dtype):
    oarch, _, m = _pair("mycnn5", C, W)
    m.set_path("generic" if path == "generic" else "auto")
    m.set_option("small_kernel", 0)
    lens = [1, 7, 12, 3, 1, 6]
    B = sum(lens)
    x = tskd_b200.synth.make_windows(B, C, W, "normal", seed=18, dtype=dtype).to(DEV)
    age = tskd_b200.synth.make_ages(B, seed=18).to(DEV)
    got = m.predict(x, age, mode="sequence", seq_lengths=lens)
    assert m.last_path == path
    want = _per_sequence(m, x, age, lens)
    assert torch.equal(got, want), (got - want).abs().max()
    assert torch.equal(m.predict(x, age, mode="sequence", seq_lengths=lens, return_prob=True),
                       _per_sequence(m, x, age, lens, return_prob=True))
    assert torch.equal(m(x, age, seq_lengths=lens), got)
    assert torch.equal(m.predict(x, age[:1], mode="sequence", seq_lengths=lens), _per_sequence(m, x, age[:1].expand(B), lens))


def test_windows_cut_from_recordings_equal_predict_record():
    oarch, _, m = _pair("mycnn5", 3, 1528)
    S, n_w, R = 200, 9, 4
    N = 1528 + (n_w - 1) * S
    rec = tskd_b200.synth.make_windows(R, 3, N, "normal", seed=19, dtype=torch.float32).to(DEV)
    age = tskd_b200.synth.make_ages(R, seed=19).to(DEV)
    want = m.predict_record(rec, S, age, path="generic", mode="sequence")
    m.set_path("generic")
    windows = rec.unfold(2, 1528, S).permute(0, 2, 1, 3).reshape(R * n_w, 3, 1528).contiguous()
    got = m.predict(windows, age.repeat_interleave(n_w), mode="sequence", seq_lengths=[n_w] * R)
    assert torch.equal(got.reshape(R, n_w), want)


def test_trainable_eval_with_lengths_equals_predict():
    oarch, _, m = _pair("mycnn5", 10, 120, trainable=True)
    lens = [4, 1, 10]
    x, age, _, _, _ = _batch(oarch, sum(lens), seed=20, p=0.0)
    m.eval()
    assert torch.equal(m(x.to(DEV), age.to(DEV), seq_lengths=lens), m.predict(x.to(DEV), age.to(DEV), mode="sequence", seq_lengths=lens))


# ------------------------------------------------------------------ 7. errors and workspace
def test_bad_lengths_fail_before_any_launch_and_leave_everything_usable():
    oarch, _, m = _pair("mycnn5", 10, 120, trainable=True)
    x, age, y, _, _ = _batch(oarch, 8, seed=21, p=0.0)
    x, age, y = x.to(DEV), age.to(DEV), y.to(DEV)
    plain = tskd_b200.B200MyCNN(m.arch).to(DEV)
    plain.load_state_dict(m.state_dict())
    tr = B200Trainer(plain, dropout=0.0)
    good_p = plain.predict(x, age, mode="sequence", seq_lengths=[3, 5])
    good_l = tr.step(x, age, y, update=False, seq_lengths=[3, 5])
    m.train()
    for bad in ([3, 4], [8, 0], [9, -1], [4.0, 4], [], torch.tensor([4.0, 4.0])):
        with pytest.raises(ValueError):
            plain.predict(x, age, mode="sequence", seq_lengths=bad)
        with pytest.raises(ValueError):
            tr.step(x, age, y, seq_lengths=bad)
        with pytest.raises(ValueError):
            m(x, age, seq_lengths=bad)
    with pytest.raises(ValueError):
        B200Trainer(plain, mode="independent").step(x, age, y, seq_lengths=[8])
    with pytest.raises(ValueError):
        plain(x, age.reshape(1, 8), seq_lengths=[8])            # run_model's (1, n) age is not combined with seq_lengths
    assert tr.steps == 0
    assert torch.equal(plain.predict(x, age, mode="sequence", seq_lengths=[3, 5]), good_p)
    assert torch.equal(tr.step(x, age, y, update=False, seq_lengths=[3, 5]), good_l)


def test_c_abi_null_lengths_short_workspace_and_guard_region():
    oarch, _, m = _pair("mycnn5", 10, 120)
    lib, h = m._ensure_handle()
    B = 24
    x, age, _, _, _ = _batch(oarch, B, seed=22, p=0.0)
    x, age = x.to(DEV), age.to(DEV)
    lens = (ctypes.c_int64 * 3)(10, 4, 10)
    st = torch.cuda.current_stream().cuda_stream
    need = int(lib.b2cnn_workspace_bytes_seq(h, B, lens, 3))
    assert need > int(lib.b2cnn_workspace_bytes(h, B, capi.MODE_SEQUENCE))
    out = torch.full((B,), 7.0, device=DEV)
    guard = 4096
    ws = torch.full((need + guard,), 0xA5, dtype=torch.uint8, device=DEV)
    args = lambda L, n, nbytes: (h, x.data_ptr(), capi.DTYPE_F32, B, 120, age.data_ptr(), B, L, n, 0, out.data_ptr(), ws.data_ptr(), nbytes, st)
    assert lib.b2cnn_forward_seq(*args(None, 3, need)) == capi.EINVAL
    assert lib.b2cnn_forward_seq(*args(lens, 0, need)) == capi.EINVAL
    assert lib.b2cnn_forward_seq(*args((ctypes.c_int64 * 3)(10, 4, 9), 3, need)) == capi.EINVAL
    assert lib.b2cnn_forward_seq(*args(lens, 3, int(lib.b2cnn_workspace_bytes(h, B, capi.MODE_SEQUENCE)))) == capi.ESTATE
    torch.cuda.synchronize()
    assert torch.equal(out, torch.full((B,), 7.0, device=DEV))            # nothing ran
    assert lib.b2cnn_forward_seq(*args(lens, 3, need)) == capi.OK, capi.last_error()
    torch.cuda.synchronize()
    assert bool((ws[need:] == 0xA5).all())
    assert torch.equal(out, m.predict(x, age, mode="sequence", seq_lengths=[10, 4, 10]))
    # training: NULL lengths, a workspace of the plain query, and the guard region past the _seq query
    cfg = capi.make_config(m.arch, 0)
    params = m.packed_weights().to(DEV)
    z = torch.full((B,), 7.0, device=DEV)
    tneed = int(lib.b2cnn_train_workspace_bytes_seq(ctypes.byref(cfg), B, lens, 3))
    tws = torch.full((tneed + guard,), 0xA5, dtype=torch.uint8, device=DEV)
    targs = lambda L, n, nbytes: (ctypes.byref(cfg), params.data_ptr(), x.data_ptr(), B, age.data_ptr(), L, n, None, None, z.data_ptr(),
                                  tws.data_ptr(), nbytes, st)
    assert lib.b2cnn_train_forward_seq(*targs(None, 3, tneed)) == capi.EINVAL
    assert lib.b2cnn_train_forward_seq(*targs(lens, 3, int(lib.b2cnn_train_workspace_bytes(ctypes.byref(cfg), B)))) == capi.ESTATE
    torch.cuda.synchronize()
    assert torch.equal(z, torch.full((B,), 7.0, device=DEV))
    assert lib.b2cnn_train_forward_seq(*targs(lens, 3, tneed)) == capi.OK, capi.last_error()
    dz, grads = torch.ones(B, device=DEV), torch.empty_like(params)
    assert lib.b2cnn_train_backward_seq(ctypes.byref(cfg), params.data_ptr(), x.data_ptr(), B, age.data_ptr(), lens, 3, None, None,
                                        dz.data_ptr(), grads.data_ptr(), None, None, 0, tws.data_ptr(), tneed, st) == capi.OK
    torch.cuda.synchronize()
    assert bool((tws[tneed:] == 0xA5).all())
