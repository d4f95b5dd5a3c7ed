"""GPU: training on whole recordings.  step_record / mycnn_train_record_forward over every counted window of [B, C, N]
recordings against the same step on the windows cut out as copies (tskd_b200.autograd.cut_record_windows): the logits,
the loss, every LSTM and Linear gradient (W_ih_l0 included), the per-window d age and those parameters after Adam are
the same bits; the conv gradients and d records, whose sums over windows are ordered differently, are judged element
by element against the float64 oracle (oracle/train_record_ref.py) at the grants of test_gpu_train_seq.py.  Then the
samples no counted window reads (NaN / inf change nothing), determinism, Adam, the frozen front end, the launch list,
the workspace and eval mode."""
import collections
import ctypes
import json
import os
import subprocess
import sys
from dataclasses import replace

import pytest
import torch

import tskd_b200
from tskd_b200 import capi
from tskd_b200.arch import BLOB_KEYS
from tskd_b200.autograd import _Call, _TrainForward, cut_record_windows
from tskd_b200.trainer import B200Trainer
from oracle import mycnn_torch as O
from oracle.train_ref import BETA, MaskDropout, check_elems
from oracle.train_record_ref import train_reference_record

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
POS_WEIGHT = 13.5
CONV = ("conv1.weight", "conv1.bias", "conv2.weight", "conv2.bias")
HEAD = [k for k in BLOB_KEYS if k not in CONV]
# the grants of tests/test_gpu_train_seq.py
BIG_B_BETA = {k: 4e-6 for k in CONV}
LONG_SUM_BETA = {k: 4e-6 for k in ("conv1.weight", "conv2.weight", "drecords")}


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


def _records(arch, B, N, S, counts, seed, p):
    """recordings, ages per recording, targets per window and the recording's masks (None for p = 0)"""
    g = torch.Generator().manual_seed(seed)
    rec = torch.randn(B, arch.in_channels, N, generator=g)
    age = torch.rand(B, generator=g) * 60 + 20
    y = (torch.rand(sum(counts), generator=g) > 0.5).float()
    if p > 0:
        ra = arch.with_shape(arch.in_channels, N)
        m1 = torch.bernoulli(torch.full((B, 4, ra.p1), 1 - p), generator=g) / (1 - p)
        m2 = torch.bernoulli(torch.full((B, ra.l_out), 1 - p), generator=g) / (1 - p)
    else:
        m1 = m2 = None
    return rec, age, y, m1, m2


def _dev(t):
    return None if t is None else t.to(DEV)


def _params(m):
    named = dict(m.named_parameters())
    return [named[k] for k in BLOB_KEYS]


def _cut(arch, rec, S, counts, age, m1, m2):
    x, c1, c2 = cut_record_windows(rec, arch.window, S, counts, arch.pool_s, m1, m2)
    return x, age.repeat_interleave(torch.tensor(counts)), c1, c2


def _lens(counts, mode):
    return [c for c in counts if c > 0] if mode == "sequence" else None


def _beta(W, M):
    return {**(BIG_B_BETA if M >= 257 else {}), **(LONG_SUM_BETA if W > 1000 else {})}


def _yardstick(truth, ref32, cut):
    """per element, whichever float32 computation of the same gradient lands farther from the truth: the reference module
    in float32, or the shipped kernels on the cut windows.  A conv bias gradient is one long cancelling sum (a few 1e-5
    left of terms a thousand times larger), where torch's float32 reduction can land within 1e-12 of the truth; the
    record path sums the same terms in another order, and is held to what the cut path itself achieves there."""
    return torch.where((cut.double().cpu() - truth).abs() > (ref32.double() - truth).abs(), cut.double().cpu(), ref32.double())


# (kind, C, W, N, S, counts): create_batch's 40 % overlap, abutting windows, gaps (S > W) and a stride of one feature;
# the older revision; a waveform window of many conv tiles on recordings of many tiles; ragged counts with 0 and n_w - 1
CASES = [
    ("mycnn5", 10, 120, 120 + 72 * 6 + 40, 72, [7, 7, 7]),
    ("mycnn5", 10, 120, 120 * 5, 120, [5, 5]),
    ("mycnn5", 10, 120, 120 + 200 * 4 + 50, 200, [5, 5, 5]),
    ("mycnn5", 10, 120, 120 + 4 * 30, 4, [31, 31]),
    ("mycnn2", 7, 120, 120 + 72 * 5, 72, [6, 6, 6]),
    ("mycnn5", 3, 7504, 7504 + 3752 * 3 + 100, 3752, [4, 4]),
    ("mycnn5", 10, 120, 120 + 72 * 8 + 30, 72, [9, 0, 3, 8, 1, 0, 9]),
]
IDS = ["m5-s72", "m5-s120", "m5-s200-gaps", "m5-s4", "m2-c7-s72", "m5-w7504", "m5-ragged"]


def _fused_pair(case, mode, p, pos_weight, seed):
    kind, C, W, N, S, counts = case
    oarch, ref, m = _pair(kind, C, W)
    _, _, mc = _pair(kind, C, W)
    rec, age, y, m1, m2 = _records(m.arch, len(counts), N, S, counts, seed, p)
    tr = B200Trainer(m, lr=1e-3, dropout=p, pos_weight=pos_weight, mode=mode)
    tc = B200Trainer(mc, lr=1e-3, dropout=p, pos_weight=pos_weight, mode=mode)
    return oarch, ref, m, rec, age, y, m1, m2, tr, tc


# ------------------------------------------------------------------ 1. the identity and the float64 truth
@pytest.mark.parametrize("case", CASES, ids=IDS)
@pytest.mark.parametrize("mode", ["sequence", "independent"])
@pytest.mark.parametrize("p,pos_weight", [(0.1, None), (0.0, POS_WEIGHT)], ids=["p0.1", "p0-pw"])
def test_fused_step_equals_the_cut_windows(case, mode, p, pos_weight):
    kind, C, W, N, S, counts = case
    oarch, ref, m, rec, age, y, m1, m2, tr, tc = _fused_pair(case, mode, p, pos_weight, seed=5)
    x, age_w, c1, c2 = _cut(m.arch, rec, S, counts, age, m1, m2)
    loss = tr.step_record(rec, S, age, y, window_counts=counts, masks=(m1, m2))
    want = tc.step(x, age_w, y, masks=(c1, c2), seq_lengths=_lens(counts, mode))
    assert torch.equal(loss, want)
    g, gc = tr.grads(), tc.grads()
    for k in HEAD:
        assert torch.equal(g[k], gc[k]), k
    got_p, want_p = tr._views(tr._params), tc._views(tc._params)
    for k in HEAD:
        assert torch.equal(got_p[k], want_p[k]), k
    head = "bce" if pos_weight is None else "bce_pw"
    truth = train_reference_record(ref, rec, S, age, counts, mode, m1, m2, target=y, pos_weight=pos_weight)[head]
    ref32 = train_reference_record(ref, rec, S, age, counts, mode, m1, m2, target=y, pos_weight=pos_weight, dtype=torch.float32)[head]
    beta = _beta(W, sum(counts))
    check_elems([(k, g[k], truth["grads"][k], _yardstick(truth["grads"][k], ref32["grads"][k], gc[k]), beta.get(k, BETA)) for k in CONV],
                f"fused {kind} {N}/{S} {mode}")


def _record_autograd(m, rec, S, age_w, counts, mode, m1, m2, r):
    """z, the parameter gradients, d records and the per-window d age through the autograd Function of the _record calls"""
    for q in m.parameters():
        q.grad = None
    B, N = rec.shape[0], rec.shape[2]
    cts = (ctypes.c_int64 * B)(*counts)
    call = _Call(m.arch, torch.device(DEV), tskd_b200.autograd._MODES[mode], _dev(m1), _dev(m2), rec=(N, S, cts, sum(counts)))
    rd, ad = rec.to(DEV).requires_grad_(), age_w.to(DEV).requires_grad_()
    z = _TrainForward.apply(call, rd, ad, *_params(m))
    (z * r.to(DEV)).sum().backward()
    named = dict(m.named_parameters())
    return z.detach(), {k: named[k].grad.clone() for k in BLOB_KEYS}, rd.grad, ad.grad


def _cut_autograd(m, x, age_w, counts, mode, c1, c2, r):
    for q in m.parameters():
        q.grad = None
    xd, ad = x.to(DEV).requires_grad_(), age_w.to(DEV).requires_grad_()
    z = tskd_b200.mycnn_train_forward(xd, ad, _params(m), m.arch, mode, _dev(c1), _dev(c2), seq_lengths=_lens(counts, mode))
    (z * r.to(DEV)).sum().backward()
    named = dict(m.named_parameters())
    return z.detach(), {k: named[k].grad.clone() for k in BLOB_KEYS}, xd.grad, ad.grad


@pytest.mark.parametrize("case", CASES, ids=IDS)
@pytest.mark.parametrize("mode", ["sequence", "independent"])
@pytest.mark.parametrize("p", [0.1, 0.0])
def test_autograd_equals_the_cut_windows(case, mode, p):
    kind, C, W, N, S, counts = case
    oarch, ref, m = _pair(kind, C, W, trainable=True)
    rec, age, _, m1, m2 = _records(m.arch, len(counts), N, S, counts, seed=6, p=p)
    x, age_w, c1, c2 = _cut(m.arch, rec, S, counts, age, m1, m2)
    r = torch.randn(sum(counts), generator=torch.Generator().manual_seed(9))
    z, g, drec, dage = _record_autograd(m, rec, S, age_w, counts, mode, m1, m2, r)
    zc, gc, _, dagec = _cut_autograd(m, x, age_w, counts, mode, c1, c2, r)
    assert torch.equal(z, zc) and torch.equal(dage, dagec)
    for k in HEAD:
        assert torch.equal(g[k], gc[k]), k
    full = train_reference_record(ref, rec, S, age, counts, mode, m1, m2, dz=r)["dz"]
    full32 = train_reference_record(ref, rec, S, age, counts, mode, m1, m2, dz=r, dtype=torch.float32)["dz"]
    beta = _beta(W, sum(counts))
    pairs = [(k, g[k], full["grads"][k], _yardstick(full["grads"][k], full32["grads"][k], gc[k]), beta.get(k, BETA)) for k in CONV]
    pairs.append(("drecords", drec, full["drecords"], full32["drecords"], beta.get("drecords", BETA)))
    check_elems(pairs, f"autograd {kind} {N}/{S} {mode}")
    # the public function: the same logits, and d age per recording summed over its windows
    for q in m.parameters():
        q.grad = None
    ar = age.to(DEV).requires_grad_()
    zf = tskd_b200.mycnn_train_record_forward(rec.to(DEV), S, ar, _params(m), m.arch, mode, _dev(m1), _dev(m2), counts)
    assert torch.equal(zf.detach(), z)
    (zf * r.to(DEV)).sum().backward()
    check_elems([("dage_rec", ar.grad, full["dage_rec"], full32["dage_rec"], BETA)], "age per recording")


# ------------------------------------------------------------------ 2. samples no counted window reads
def _poison(rec, W, S, counts, value):
    """rec with `value` at every sample no counted window reads, and the mask of those samples"""
    B, C, N = rec.shape
    read = torch.zeros(B, N, dtype=torch.bool)
    for b, n in enumerate(counts):
        for w in range(n):
            read[b, w * S:w * S + W] = True
    out = rec.clone()
    out[(~read)[:, None, :].expand(B, C, N)] = value
    return out, ~read


@pytest.mark.parametrize("case", [CASES[2], CASES[5], CASES[6]], ids=["gaps", "w7504", "ragged"])
@pytest.mark.parametrize("mode", ["sequence", "independent"])
def test_unread_samples_change_nothing(case, mode):
    kind, C, W, N, S, counts = case
    _, _, m = _pair(kind, C, W, trainable=True)
    rec, age, y, m1, m2 = _records(m.arch, len(counts), N, S, counts, seed=7, p=0.1)
    age_w = age.repeat_interleave(torch.tensor(counts))
    r = torch.randn(sum(counts), generator=torch.Generator().manual_seed(3))
    zero, unread = _poison(rec, W, S, counts, 0.0)
    assert bool(unread.any())
    base = _record_autograd(m, zero, S, age_w, counts, mode, m1, m2, r)
    losses = []
    for value in (float("nan"), float("inf"), float("-inf")):
        bad, _ = _poison(rec, W, S, counts, value)
        z, g, drec, dage = _record_autograd(m, bad, S, age_w, counts, mode, m1, m2, r)
        assert torch.equal(z, base[0]) and torch.equal(dage, base[3])
        for k in BLOB_KEYS:
            assert torch.equal(g[k], base[1][k]), (value, k)
        assert torch.equal(drec, base[2]), value
        assert float(drec.permute(0, 2, 1)[unread.to(DEV)].abs().max()) == 0.0
        _, _, mf = _pair(kind, C, W)
        tr = B200Trainer(mf, dropout=0.1, mode=mode)
        losses.append((tr.step_record(bad, S, age, y, window_counts=counts, masks=(m1, m2), update=False), tr._grads.clone()))
    _, _, mf = _pair(kind, C, W)
    tr = B200Trainer(mf, dropout=0.1, mode=mode)
    want = tr.step_record(zero, S, age, y, window_counts=counts, masks=(m1, m2), update=False)
    for loss, grads in losses:
        assert torch.equal(loss, want) and torch.equal(grads, tr._grads)


def test_nan_inside_a_window_gives_the_cut_logits_and_loss():
    kind, C, W, N, S, counts = CASES[0]
    _, _, m = _pair(kind, C, W)
    rec, age, y, m1, m2 = _records(m.arch, len(counts), N, S, counts, seed=8, p=0.1)
    rec[1, 3, 2 * S + 50] = float("nan")                    # windows 1 and 2 of recording 1 read it
    x, age_w, c1, c2 = _cut(m.arch, rec, S, counts, age, m1, m2)
    z = tskd_b200.mycnn_train_record_forward(rec.to(DEV), S, age.to(DEV), _params(m), m.arch, "sequence", _dev(m1), _dev(m2), counts)
    zc = tskd_b200.mycnn_train_forward(x.to(DEV), age_w.to(DEV), _params(m), m.arch, "sequence", _dev(c1), _dev(c2), seq_lengths=counts)
    nan = torch.isnan(z)
    assert bool(nan.any()) and torch.equal(nan, torch.isnan(zc)) and torch.equal(z[~nan], zc[~nan])
    _, _, mc = _pair(kind, C, W)
    loss = B200Trainer(m, dropout=0.1).step_record(rec, S, age, y, window_counts=counts, masks=(m1, m2), update=False)
    want = B200Trainer(mc, dropout=0.1).step(x, age_w, y, masks=(c1, c2), update=False, seq_lengths=counts)
    assert torch.isnan(loss) and torch.isnan(want)


# ------------------------------------------------------------------ 3. determinism, Adam, frozen conv
def test_two_runs_give_the_same_bits_at_scale():
    _, _, m = _pair("mycnn5", 3, 75000)
    B, N, S = 64, 142500, 7500
    counts = [10] * B
    rec, age, y, m1, m2 = _records(m.arch, B, N, S, counts, seed=16, p=0.1)
    rec, m1, m2 = rec.to(DEV), m1.to(DEV), m2.to(DEV)
    runs = []
    for _ in range(2):
        tr = B200Trainer(m, dropout=0.1)
        loss = tr.step_record(rec, S, age, y, masks=(m1, m2), update=False)
        runs.append((loss.clone(), tr._grads.clone()))
    assert torch.isfinite(runs[0][0]) and torch.equal(runs[0][0], runs[1][0]) and torch.equal(runs[0][1], runs[1][1])


def test_three_adam_steps_follow_the_cut_path():
    kind, C, W, N, S, _ = CASES[6]
    _, ref, m = _pair(kind, C, W)
    _, _, mc = _pair(kind, C, W)
    tr, tc = B200Trainer(m, lr=1e-3, dropout=0.1), B200Trainer(mc, lr=1e-3, dropout=0.1)
    for step, counts in enumerate(([9, 0, 3, 8, 1, 0, 9], [1, 2, 3, 4, 5, 6, 7], [9] * 7)):
        rec, age, y, m1, m2 = _records(m.arch, len(counts), N, S, counts, seed=100 + step, p=0.1)
        x, age_w, c1, c2 = _cut(m.arch, rec, S, counts, age, m1, m2)
        loss = tr.step_record(rec, S, age, y, window_counts=counts, masks=(m1, m2))
        want = tc.step(x, age_w, y, masks=(c1, c2), seq_lengths=_lens(counts, "sequence"))
        assert torch.equal(loss, want) if step == 0 else abs(float(loss) - float(want)) <= 1e-5 * max(1.0, abs(float(want)))
    # the first step is the identity; after it the conv weights differ by the conv gradients' rounding, so the features
    # and with them every later gradient do too: within what Adam makes of that (tests/test_gpu_train_seq.py's bounds)
    got, exp, g = tr._views(tr._params), tc._views(tc._params), tc.grads()
    for k in BLOB_KEYS:
        d = (got[k] - exp[k]).abs()
        sel = g[k].abs() > 1e-4 * g[k].abs().max()
        assert float(d[sel].max()) <= 2e-5 and float(d.max()) <= 6.1e-3, (k, float(d[sel].max()), float(d.max()))
    assert tr.steps == 3


def test_three_adam_steps_on_a_frozen_front_end_are_bit_identical():
    kind, C, W, N, S, _ = CASES[6]
    _, _, m = _pair(kind, C, W, trainable=True)
    _, _, mc = _pair(kind, C, W, trainable=True)
    for mm in (m, mc):
        mm.conv1.requires_grad_(False)
        mm.conv2.requires_grad_(False)
    opt = torch.optim.Adam([q for q in m.parameters() if q.requires_grad], lr=1e-3)
    optc = torch.optim.Adam([q for q in mc.parameters() if q.requires_grad], lr=1e-3)
    for step, counts in enumerate(([9, 0, 3, 8, 1, 0, 9], [1, 2, 3, 4, 5, 6, 7], [9] * 7)):
        rec, age, y, m1, m2 = _records(m.arch, len(counts), N, S, counts, seed=110 + step, p=0.1)
        x, age_w, c1, c2 = _cut(m.arch, rec, S, counts, age, m1, m2)
        crit = torch.nn.BCEWithLogitsLoss()
        opt.zero_grad()
        z = tskd_b200.mycnn_train_record_forward(rec.to(DEV), S, age.to(DEV), _params(m), m.arch, "sequence", _dev(m1), _dev(m2), counts)
        crit(z, y.to(DEV)).backward()
        opt.step()
        optc.zero_grad()
        zc = tskd_b200.mycnn_train_forward(x.to(DEV), age_w.to(DEV), _params(mc), mc.arch, "sequence", _dev(c1), _dev(c2),
                                           seq_lengths=_lens(counts, "sequence"))
        crit(zc, y.to(DEV)).backward()
        optc.step()
        assert torch.equal(z.detach(), zc.detach())
    for (k, a), (_, b) in zip(m.named_parameters(), mc.named_parameters()):
        assert torch.equal(a, b), k


def _run_script(script):
    """the JSON of a script's last output line, run in a process of its own: a profiler session leaves state behind in
    the process that runs it (CUPTI, kineto), and the tests that run after this file must see the process as it was"""
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    env = dict(os.environ, PYTHONPATH=os.pathsep.join([root] + [p for p in [os.environ.get("PYTHONPATH")] if p]))
    cmd = [sys.executable] + (["-s"] if sys.flags.no_user_site else []) + ["-c", script]
    r = subprocess.run(cmd, capture_output=True, text=True, env=env, cwd=root, timeout=600)
    assert r.returncode == 0, r.stderr[-3000:]
    return json.loads(r.stdout.strip().splitlines()[-1])


_FROZEN_KERNELS = r"""
import json
import torch
import tskd_b200
from torch.profiler import ProfilerActivity, profile

dev = torch.device("cuda", 0)
m = tskd_b200.B200TrainableMyCNN(tskd_b200.ARCH_PRESETS["mycnn5"]).to(dev)
m.conv1.requires_grad_(False)
m.conv2.requires_grad_(False)
g = torch.Generator().manual_seed(0)
rec = torch.randn(3, 10, 592, generator=g).to(dev)
counts = [7, 0, 5]
m1, m2 = m.draw_masks(3, 592)
params = [dict(m.named_parameters())[k] for k in tskd_b200.arch.BLOB_KEYS]

def step():
    z = tskd_b200.mycnn_train_record_forward(rec, 72, 60.0, params, m.arch, "sequence", m1, m2, counts)
    z.sum().backward()

step()
torch.cuda.synchronize()
with profile(activities=[ProfilerActivity.CUDA]) as prof:
    step()
    torch.cuda.synchronize()
print(json.dumps(sorted({e.name for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA})))
"""


def test_frozen_conv_skips_the_conv_backward():
    kind, C, W, N, S, counts = CASES[0]
    _, _, m = _pair(kind, C, W, trainable=True)
    rec, age, _, m1, m2 = _records(m.arch, len(counts), N, S, counts, seed=17, p=0.1)
    r = torch.randn(sum(counts), generator=torch.Generator().manual_seed(5)).to(DEV)

    def grads():
        for q in m.parameters():
            q.grad = None
        z = tskd_b200.mycnn_train_record_forward(rec.to(DEV), S, age.to(DEV), _params(m), m.arch, "sequence", _dev(m1), _dev(m2), counts)
        (z * r).sum().backward()
        return {k: v.grad for k, v in m.named_parameters() if v.grad is not None}

    full = grads()
    m.conv1.requires_grad_(False)
    m.conv2.requires_grad_(False)
    frozen = grads()
    assert set(frozen) == {k for k in full if not k.startswith("conv")}
    for k, v in frozen.items():
        assert torch.equal(v, full[k]), k
    # the kernels of a frozen front end's backward, profiled in a process of its own
    names = _run_script(_FROZEN_KERNELS)
    assert not any(n in k for k in names for n in ("train_conv_bwd", "train_conv_grad_reduce", "train_dfeat")), names
    assert any("train_wih0_grad_record" in k for k in names) and any("train_conv_fwd_record" in k for k in names), names


# ------------------------------------------------------------------ 4. the launch list does not depend on the shape
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
                               and ("b2cnn::" in e.name or e.name.startswith("Memset") or e.name.startswith("Memcpy")))
m = tskd_b200.B200MyCNN(tskd_b200.ARCH_PRESETS["mycnn5"]).to(dev)
tr = B200Trainer(m, dropout=0.1)
g = torch.Generator().manual_seed(0)
kernels(lambda: torch.ones(1, device=dev).add_(1))
res = []
for B, N, S, counts in ((4, 1200, 72, None), (3, 600, 200, [3, 0, 1]), (9, 300, 4, [46] * 9), (2, 5000, 120, [2, 40])):
    rec = torch.randn(B, 10, N, generator=g).to(dev)
    M = sum(counts) if counts else B * ((N - 120) // S + 1)
    y = torch.zeros(M, device=dev)
    tr.step_record(rec, S, 60.0, y, window_counts=counts, update=False)
    res.append(kernels(lambda: tr.step_record(rec, S, 60.0, y, window_counts=counts)))
print(json.dumps(res))
"""


def test_launch_list_does_not_depend_on_the_shape():
    lists = [collections.Counter(d) for d in _run_script(_LAUNCH_LIST)]
    assert all(c == lists[0] for c in lists), lists
    assert any("train_dfeat_fold" in k for k in lists[0]), lists[0]


# ------------------------------------------------------------------ 5. workspace and eval mode
def test_undersized_workspace_and_guard_region():
    kind, C, W, N, S, counts = CASES[6]
    _, _, m = _pair(kind, C, W)
    B, M = len(counts), sum(counts)
    rec, age, _, m1, m2 = _records(m.arch, B, N, S, counts, seed=22, p=0.1)
    rec, m1, m2 = rec.to(DEV), m1.to(DEV), m2.to(DEV)
    age_w = age.repeat_interleave(torch.tensor(counts)).to(DEV)
    lib, cfg = capi.load_library(), capi.make_config(m.arch, 0)
    params = m.packed_weights().to(DEV)
    cts = (ctypes.c_int64 * B)(*counts)
    st = torch.cuda.current_stream().cuda_stream
    need = int(lib.b2cnn_train_workspace_bytes_record(ctypes.byref(cfg), B, N, S, cts, capi.MODE_SEQUENCE))
    guard = 4096
    ws = torch.full((need + guard,), 0xA5, dtype=torch.uint8, device=DEV)
    z = torch.full((M,), 7.0, device=DEV)
    args = lambda nbytes: (ctypes.byref(cfg), params.data_ptr(), rec.data_ptr(), B, N, S, cts, capi.MODE_SEQUENCE, age_w.data_ptr(),
                           m1.data_ptr(), m2.data_ptr(), z.data_ptr(), ws.data_ptr(), nbytes, st)
    assert lib.b2cnn_train_forward_record(*args(need - 4)) == capi.ESTATE
    torch.cuda.synchronize()
    assert torch.equal(z, torch.full((M,), 7.0, device=DEV))             # nothing ran
    assert lib.b2cnn_train_forward_record(*args(need)) == capi.OK, capi.last_error()
    dz, grads, drec, dage = torch.ones(M, device=DEV), torch.empty_like(params), torch.empty_like(rec), torch.empty(M, device=DEV)
    assert lib.b2cnn_train_backward_record(ctypes.byref(cfg), params.data_ptr(), rec.data_ptr(), B, N, S, cts, capi.MODE_SEQUENCE,
                                           age_w.data_ptr(), m1.data_ptr(), m2.data_ptr(), dz.data_ptr(), grads.data_ptr(),
                                           drec.data_ptr(), dage.data_ptr(), 0, ws.data_ptr(), need, st) == capi.OK
    torch.cuda.synchronize()
    assert bool((ws[need:] == 0xA5).all())
    assert bool(torch.isfinite(z).all()) and bool(torch.isfinite(grads).all())


@pytest.mark.parametrize("batch_mode", ["sequence", "independent"])
def test_eval_forward_record_is_predict_record_cut_to_the_counts(batch_mode):
    kind, C, W, N, S, counts = CASES[6]
    _, _, m = _pair(kind, C, W, trainable=True)
    m.batch_mode = batch_mode
    m.eval()
    rec, age, _, _, _ = _records(m.arch, len(counts), N, S, counts, seed=23, p=0.0)
    rec, age = rec.to(DEV), age.to(DEV)
    got = m.forward_record(rec, S, age, window_counts=counts)
    full = m.predict_record(rec, S, age, mode=batch_mode)
    assert torch.equal(got, torch.cat([full[b, :n] for b, n in enumerate(counts)]))
    m.train()
    m.dropout.p = 0.0
    zt = m.forward_record(rec, S, age, window_counts=counts)
    assert zt.shape == got.shape and zt.requires_grad
