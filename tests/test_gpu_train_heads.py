"""GPU: B200HeadTrainer -- K candidate heads trained on one frozen front end in one fused step.

Head i's loss and gradients (every blob entry from lstm.weight_ih_l0 on) must be the bits B200Trainer computes on a copy
of head i with the same masks, in both modes, with seq_lengths, with and without pos_weight and dropout, for K in
{1, 2, 3, 8}, at the training shape and on waveform windows, and for step_record over ragged recordings.  Then: Adam
steps with per-head learning rates equal each head trained alone; a K = 1 trainer follows autograd with frozen convs and
torch.optim.Adam; the front end never changes; trained heads plug into predict_record(heads=) and SlidingScorer.set_heads;
the launch list does not depend on K; the C ABI's refusals leave everything untouched; two runs give the same bits."""
import collections
import copy
import ctypes
import json
import os
import subprocess
import sys

import numpy as np
import pytest
import torch
from torch import nn

import tskd_b200
from tskd_b200 import capi
from tskd_b200.arch import BLOB_KEYS
from tskd_b200.trainer import B200HeadTrainer, B200Trainer

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HEAD_KEYS = BLOB_KEYS[BLOB_KEYS.index("lstm.weight_ih_l0"):]
CONV_KEYS = BLOB_KEYS[:BLOB_KEYS.index("lstm.weight_ih_l0")]


def _golden_model():
    g = np.load(os.path.join(ROOT, "tests", "golden", "mycnn5_xtestinput.npz"))
    sd = {k[3:]: torch.from_numpy(g[k]) for k in g.files if k.startswith("sd.")}
    return tskd_b200.B200MyCNN.from_reference(sd).to(DEV)


def _model(C, W, seed=0):
    if (C, W) == (10, 120):
        return _golden_model()
    torch.manual_seed(seed)
    return tskd_b200.B200MyCNN(tskd_b200.ARCH_PRESETS["mycnn5"].with_shape(C, W)).to(DEV)


def _heads(m, K, seed=1):
    """K candidates on m's front end: m's LSTM / Linear weights, each perturbed differently"""
    g = torch.Generator().manual_seed(seed)
    hs = []
    for i in range(K):
        h = copy.deepcopy(m)
        with torch.no_grad():
            sd = h.state_dict()
            for k in HEAD_KEYS:
                sd[k].add_(0.05 * torch.randn(sd[k].shape, generator=g).to(DEV))
        h.sync_weights()
        hs.append(h)
    return hs


def _batch(arch, B, seed, p):
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(B, arch.in_channels, arch.window, generator=g).to(DEV)
    age = (torch.rand(B, generator=g) * 60 + 20).to(DEV)
    y = (torch.rand(B, generator=g) > 0.7).float().to(DEV)
    if p > 0:
        m1 = (torch.bernoulli(torch.full((B, 4, arch.p1), 1 - p), generator=g) / (1 - p)).to(DEV)
        m2 = (torch.bernoulli(torch.full((B, arch.l_out), 1 - p), generator=g) / (1 - p)).to(DEV)
    else:
        m1 = m2 = None
    return x, age, y, (m1, m2)


def _alone(h, mode, pos_weight, fn):
    """loss and head gradients of B200Trainer on a copy of h"""
    tr = B200Trainer(copy.deepcopy(h), mode=mode, pos_weight=pos_weight)
    loss = fn(tr)
    return loss, {k: tr.grads()[k].clone() for k in HEAD_KEYS}


def _check_rows(losses, grads, heads, mode, pos_weight, fn):
    assert losses.shape == (len(heads),)
    for i, h in enumerate(heads):
        want_loss, want_g = _alone(h, mode, pos_weight, fn)
        assert torch.equal(losses[i], want_loss.reshape(())), (i, float(losses[i]), float(want_loss))
        assert set(grads[i]) == set(HEAD_KEYS)
        for k in HEAD_KEYS:
            assert torch.equal(grads[i][k], want_g[k]), (i, k, (grads[i][k] - want_g[k]).abs().max().item())


# (C, W, B, K, mode, seq_lengths, dropout, pos_weight)
CASES = [
    (10, 120, 1, 1, "sequence", None, 0.1, None),
    (10, 120, 33, 2, "independent", None, 0.0, 13.5),
    (10, 120, 33, 3, "sequence", [5, 1, 20, 7], 0.1, 13.5),
    (10, 120, 257, 8, "sequence", None, 0.1, None),
    (10, 120, 257, 3, "independent", None, 0.1, None),
    (10, 120, 600, 8, "sequence", [2] * 300, 0.0, 13.5),        # 300 sequences: two per scan CTA, the rows reduced
    (3, 7504, 5, 2, "sequence", None, 0.1, None),
    (3, 7504, 7, 3, "sequence", [3, 4], 0.1, 13.5),
    (3, 7504, 6, 8, "independent", None, 0.0, None),
]


@pytest.mark.parametrize("C,W,B,K,mode,lens,p,pw", CASES, ids=[f"c{c[0]}w{c[1]}-b{c[2]}-k{c[3]}-{c[4][:3]}{'-lens' if c[5] else ''}-p{c[6]}{'-pw' if c[7] else ''}"
                                                               for c in CASES])
def test_rows_equal_the_fused_step_on_each_head(C, W, B, K, mode, lens, p, pw):
    m = _model(C, W)
    heads = _heads(m, K)
    x, age, y, masks = _batch(m.arch, B, seed=B + K, p=p)
    tr = B200HeadTrainer(m, heads, mode=mode, pos_weight=pw, dropout=p)
    losses = tr.step(x, age, y, masks=masks, update=False, seq_lengths=lens)
    _check_rows(losses, tr.grads(), heads, mode, pw, lambda t: t.step(x, age, y, masks=masks, update=False, seq_lengths=lens))
    n_conv = sum(m.state_dict()[k].numel() for k in CONV_KEYS)
    assert torch.count_nonzero(tr._grads[:, :n_conv]) == 0    # the conv entries of every head's gradients are zero


def _records(arch, B, n_w, S, seed, nan=True):
    g = torch.Generator().manual_seed(seed)
    N = arch.window + (n_w - 1) * S + 37                   # a tail no window reads
    rec = torch.randn(B, arch.in_channels, N, generator=g)
    return rec, N


@pytest.mark.parametrize("mode", ["sequence", "independent"])
@pytest.mark.parametrize("K", [1, 3, 8])
def test_step_record_rows_equal_the_fused_step_on_each_head(mode, K):
    m = _model(3, 7504)
    heads = _heads(m, K, seed=7)
    S, n_w = 1504, 4
    rec, N = _records(m.arch, 4, n_w, S, seed=K)
    counts = [4, 0, 2, 3]
    # NaN / inf where no counted window reads: the tail, the whole of recording 1, the windows recording 2 does not count
    rec[:, :, -10:] = float("nan")
    rec[1] = float("inf")
    rec[2, :, 2 * S + m.arch.window:] = float("nan")
    rec = rec.to(DEV)
    M = sum(counts)
    g = torch.Generator().manual_seed(3)
    y = (torch.rand(M, generator=g) > 0.5).float().to(DEV)
    ages = torch.tensor([30.0, 40.0, 50.0, 60.0], device=DEV)
    rarch = m.arch.with_shape(3, N)
    m1 = (torch.bernoulli(torch.full((4, 4, rarch.p1), 0.9), generator=g) / 0.9).to(DEV)
    m2 = (torch.bernoulli(torch.full((4, rarch.l_out), 0.9), generator=g) / 0.9).to(DEV)
    for pw in (None, 13.5):
        tr = B200HeadTrainer(m, heads, mode=mode, pos_weight=pw)
        losses = tr.step_record(rec, S, ages, y, window_counts=counts, masks=(m1, m2), update=False)
        assert torch.isfinite(losses).all()
        _check_rows(losses, tr.grads(), heads, mode, pw,
                    lambda t: t.step_record(rec, S, ages, y, window_counts=counts, masks=(m1, m2), update=False))
    with pytest.raises(ValueError, match="state"):
        tr.step_record(rec, S, ages, y, window_counts=counts, return_state=True)


def test_adam_steps_with_per_head_lr_equal_each_head_alone():
    m = _model(10, 120)
    conv_before = {k: v.clone() for k, v in m.state_dict().items() if k in CONV_KEYS}
    heads = _heads(m, 3, seed=11)
    alone = [copy.deepcopy(h) for h in heads]
    lrs = [1e-3, 3e-4, 5e-3]
    tr = B200HeadTrainer(m, heads, lr=lrs, dropout=0.1)
    solo = [B200HeadTrainer(m, [a], lr=lr, dropout=0.1) for a, lr in zip(alone, lrs)]
    for step in range(3):
        x, age, y, masks = _batch(m.arch, 40, seed=50 + step, p=0.1)
        losses = tr.step(x, age, y, masks=masks, seq_lengths=[10, 30])
        for i, s in enumerate(solo):
            li = s.step(x, age, y, masks=masks, seq_lengths=[10, 30])
            assert torch.equal(losses[i:i + 1], li), (step, i)
    assert tr.steps == 3
    for h, a in zip(heads, alone):
        hs, as_ = h.state_dict(), a.state_dict()
        for k in BLOB_KEYS:
            assert torch.equal(hs[k], as_[k]), k
        for k in CONV_KEYS:
            assert torch.equal(hs[k], conv_before[k]), k
    for k in CONV_KEYS:
        assert torch.equal(m.state_dict()[k], conv_before[k]), k
    # the heads differ from where they started and from each other
    assert not torch.equal(heads[0].state_dict()["lstm.weight_hh_l0"], heads[1].state_dict()["lstm.weight_hh_l0"])


def test_one_head_follows_autograd_with_frozen_convs_and_torch_adam():
    """the bounds of test_gpu_train_seq.py's three Adam steps against the reference"""
    m = _model(10, 120)
    head = _heads(m, 1, seed=5)[0]
    ref = tskd_b200.B200TrainableMyCNN(m.arch, has_out12="out1.weight" in head.state_dict()).to(DEV)
    ref.load_state_dict(head.state_dict())
    ref.conv1.requires_grad_(False)
    ref.conv2.requires_grad_(False)
    named = dict(ref.named_parameters())
    params = [named[k] for k in BLOB_KEYS]
    opt = torch.optim.Adam([named[k] for k in HEAD_KEYS], lr=1e-3)
    tr = B200HeadTrainer(m, [head], lr=1e-3, dropout=0.1)
    for step in range(3):
        lens = [4, 9, 1, 6]
        x, age, y, (m1, m2) = _batch(m.arch, sum(lens), seed=80 + step, p=0.1)
        loss = tr.step(x, age, y, masks=(m1, m2), seq_lengths=lens)
        opt.zero_grad()
        z = tskd_b200.mycnn_train_forward(x, age, params, m.arch, "sequence", m1, m2, seq_lengths=lens)
        want = nn.BCEWithLogitsLoss()(z.reshape(-1), y)
        want.backward()
        opt.step()
        assert abs(float(loss[0]) - float(want)) <= 2e-5 * max(1.0, abs(float(want))), (step, float(loss[0]), float(want))
    sd = head.state_dict()
    for k in BLOB_KEYS:
        a, b = sd[k].cpu().numpy().ravel(), named[k].detach().cpu().numpy().ravel()
        if k in CONV_KEYS:
            assert np.array_equal(a, b), k
            continue
        g = np.abs(named[k].grad.cpu().numpy().ravel())
        sel = g > 1e-4 * g.max()
        assert np.abs(a[sel] - b[sel]).max() <= 2e-5, (k, np.abs(a[sel] - b[sel]).max())
        assert np.abs(a - b).max() <= 6.1e-3


def test_trained_heads_plug_into_backtesting_and_the_scorer():
    m = _model(3, 7504)
    heads = _heads(m, 3, seed=13)
    tr = B200HeadTrainer(m, [m] + heads, lr=1e-3)              # the model itself fine-tuned beside three candidates
    for step in range(2):
        x, age, y, _ = _batch(m.arch, 6, seed=90 + step, p=0.0)
        tr.step(x, age, y)
    S = 1504
    rec = torch.randn(2, 3, 7504 + 3 * S, generator=torch.Generator().manual_seed(4)).to(DEV)
    ages = torch.tensor([45.0, 70.0], device=DEV)
    rows = m.predict_record(rec, S, ages, heads=heads)
    assert rows.shape[0] == 1 + len(heads)
    assert torch.equal(rows[0], m.predict_record(rec, S, ages))
    for i, h in enumerate(heads):
        assert torch.equal(rows[1 + i], h.predict_record(rec, S, ages)), i
    scorer = tskd_b200.SlidingScorer(m, 2, S)
    scorer.set_heads(list(heads))


def test_c_abi_refusals_leave_everything_untouched():
    m = _model(10, 120)
    heads = _heads(m, 3, seed=17)
    tr = B200HeadTrainer(m, heads)
    x, age, y, (m1, m2) = _batch(m.arch, 16, seed=19, p=0.1)
    tr.step(x, age, y, masks=(m1, m2))                          # a real Adam state to guard
    lib, K = capi.load_library(), 3
    before = [t.clone() for t in (tr._params, tr._m, tr._v, tr._grads)]
    need = lib.b2cnn_train_heads_workspace_bytes(ctypes.byref(tr._cfg), K, 16, None, 0)
    ws = torch.zeros(need, dtype=torch.uint8, device=DEV)
    loss = torch.full((K,), -7.0, device=DEV)
    p = lambda t: ctypes.c_void_p(t.data_ptr()) if t is not None else None
    arr = lambda ts: (ctypes.c_void_p * len(ts))(*[t.data_ptr() if t is not None else 0 for t in ts])
    rows = lambda t: [t[i] for i in range(K)]
    lr = (ctypes.c_float * K)(1e-3, 1e-3, 1e-3)
    lens = (ctypes.c_int64 * 2)(6, 10)
    base = dict(cfg=ctypes.byref(tr._cfg), front=p(tr._front), n=K, prm=arr(rows(tr._params)), m=arr(rows(tr._m)), v=arr(rows(tr._v)),
                g=arr(rows(tr._grads)), lr=lr, step=2, opt=ctypes.byref(tr._opt), upd=1, x=p(x), B=16, age=p(age), y=p(y), pw=None,
                mode=capi.MODE_SEQUENCE, lens=None, n_seq=0, m1=p(m1), m2=p(m2), loss=p(loss), ws=p(ws), wsb=need, st=None)

    def call(**kw):
        a = {**base, **kw}
        return lib.b2cnn_train_heads_step(*a.values())

    shared = rows(tr._params)
    overlap = rows(tr._grads)
    overlap[2] = tr._params[1][10:]
    cases = {
        "n_heads 0": dict(n=0), "n_heads 9": dict(n=9),
        "null params": dict(prm=None), "null lr": dict(lr=None), "null head blob": dict(prm=arr(rows(tr._params)[:2] + [None])),
        "null adam": dict(m=None), "null frontend": dict(front=None), "null x": dict(x=None), "null loss": dict(loss=None),
        "shared blob": dict(prm=arr([shared[0], shared[1], shared[0]])), "overlapping grads": dict(g=arr(overlap)),
        "bad mode": dict(mode=7), "lengths in independent mode": dict(mode=capi.MODE_INDEPENDENT, lens=lens, n_seq=2),
        "bad lengths": dict(lens=lens, n_seq=1), "step 0": dict(step=0), "pos_weight": dict(pw=ctypes.byref(ctypes.c_float(-1.0))),
        "batch 0": dict(B=0),
    }
    for name, kw in cases.items():
        assert call(**kw) == capi.EINVAL, (name, capi.last_error())
    assert call(wsb=need - 1) == capi.ESTATE, capi.last_error()
    counts = (ctypes.c_int64 * 2)(1, 0)
    rec = torch.zeros(2, 10, 120, device=DEV)
    assert lib.b2cnn_train_heads_step_record(ctypes.byref(tr._cfg), p(tr._front), 9, base["prm"], base["m"], base["v"], base["g"], lr, 2,
                                             ctypes.byref(tr._opt), 1, p(rec), 2, 120, 8, counts, capi.MODE_SEQUENCE, p(age), p(y), None,
                                             None, None, p(loss), p(ws), need, None) == capi.EINVAL
    torch.cuda.synchronize()
    for a, b in zip(before, (tr._params, tr._m, tr._v, tr._grads)):
        assert torch.equal(a, b)
    assert torch.equal(loss, torch.full((K,), -7.0, device=DEV))
    # and the trainer still works
    assert torch.isfinite(tr.step(x, age, y, masks=(m1, m2))).all()


def test_two_runs_give_the_same_bits():
    m = _model(10, 120)
    x, age, y, masks = _batch(m.arch, 300, seed=23, p=0.1)
    runs = []
    for _ in range(2):
        heads = _heads(m, 5, seed=29)
        tr = B200HeadTrainer(m, heads, lr=[1e-3, 2e-3, 3e-3, 4e-3, 5e-3])
        losses = [tr.step(x, age, y, masks=masks, seq_lengths=[100, 200]) for _ in range(2)]
        runs.append((torch.stack(losses), tr._grads.clone(), tr._params.clone()))
    for a, b in zip(*runs):
        assert torch.equal(a, b)


_LAUNCH_LIST = r"""
import collections, copy, json
import torch
import tskd_b200
from torch.profiler import ProfilerActivity, profile

dev = torch.device("cuda", 0)
def kernels(fn):
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        torch.ones(1, device=dev).add_(1)
        torch.cuda.synchronize()
        fn()
        torch.cuda.synchronize()
    # the step's own kernels: after an update each head's sync_weights() also refreshes its inference weights
    return collections.Counter(e.name for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA
                               and "b2cnn::train_" in e.name)
m = tskd_b200.B200MyCNN(tskd_b200.ARCH_PRESETS["mycnn5"]).to(dev)
g = torch.Generator().manual_seed(0)
B = 700
x, age, y = torch.randn(B, 10, 120, generator=g).to(dev), torch.full((B,), 60.0, device=dev), torch.zeros(B, device=dev)
rec = torch.randn(3, 10, 600, generator=g).to(dev)
kernels(lambda: torch.ones(1, device=dev).add_(1))
res = {"step": [], "seq": [], "record": []}
for K in (1, 8):
    tr = tskd_b200.B200HeadTrainer(m, [copy.deepcopy(m) for _ in range(K)], dropout=0.1)
    tr.step(x, age, y)
    res["step"].append(kernels(lambda: tr.step(x, age, y)))
    res["seq"].append(kernels(lambda: tr.step(x, age, y, seq_lengths=[2] * 350)))
    res["record"].append(kernels(lambda: tr.step_record(rec, 8, 50.0, torch.zeros(3 * 61, device=dev))))
print(json.dumps(res))
"""


def test_launch_list_does_not_depend_on_k():
    env = dict(os.environ, PYTHONPATH=os.pathsep.join([ROOT] + [p for p in [os.environ.get("PYTHONPATH")] if p]))
    cmd = [sys.executable] + (["-s"] if sys.flags.no_user_site else []) + ["-c", _LAUNCH_LIST]
    r = subprocess.run(cmd, capture_output=True, text=True, env=env, cwd=ROOT, timeout=600)
    assert r.returncode == 0, r.stderr[-3000:]
    res = json.loads(r.stdout.strip().splitlines()[-1])
    for key, (k1, k8) in res.items():
        assert collections.Counter(k1) == collections.Counter(k8), (key, k1, k8)
        names = list(k1)
        assert sum(v for n, v in k1.items() if "train_conv_fwd" in n) == 1, (key, k1)
        assert not any(s in n for n in names for s in ("train_conv_bwd", "train_conv_grad_reduce", "train_dfeat")), (key, names)
        assert any("train_pre0_partial_heads" in n for n in names) and any("train_wih0_grad_heads" in n for n in names), names
        assert any("train_adam_heads" in n for n in names), names
    assert any("train_head_reduce" in n for n in res["seq"][0]), res["seq"][0]
