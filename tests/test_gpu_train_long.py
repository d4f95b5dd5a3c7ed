"""GPU: the training kernels of csrc/b2cnn_train.cu at long windows (position tiles of 128 final features, the conv
backward recomputed per tile, W_ih_l0 products as GEMMs) element by element against the float64 reference of
oracle/train_ref.py, at the existing allowance (tests/test_gpu_train_edges.py: _check) with the two named differences of
_check and LONG_SUM_BETA below.

Inputs are drawn until no pooling window holds a near-tie (oracle/train_ref.py::pool_gaps): with hundreds of thousands
of pooling windows per batch a random input has one now and then, and there a float32 kernel may legitimately route a
gradient to the neighbouring position."""
import collections
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
from tskd_b200.autograd import B200TrainableMyCNN
from tskd_b200.trainer import B200Trainer
from oracle import mycnn_torch as O
from oracle.train_ref import MaskDropout, pool_gaps, train_reference
from conftest import rel_err
from test_gpu_train_edges import TIE_GAP, _arch, _check as _check_per_tensor, _device, _inputs, _refs

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
T = 128                    # final features per tile (kT)
POS_WEIGHT = 13.5
CONV_KEYS = BLOB_KEYS[:4]
# The grant tests/test_gpu_train_edges.py gives the conv gradients from B = 257 on (BIG_B_BETA: long cancelling sums), for
# the same reason: a conv weight gradient of a long window is a sum over B * L1 >= 45 000 positions (257 windows of 120
# samples are 28 000) and d x passes d f's error on to every sample of the window.  Observed need: up to 1.8e-6.
LONG_SUM_BETA = {k: 4e-6 for k in ("conv1.weight", "conv2.weight", "dx")}


def _check(got, truth, ref32, head, beta=None):
    """tests/test_gpu_train_edges.py::_check with one difference, the only allowance this file adds: a conv layer's bias
    gradient is judged together with its weight gradient, as one tensor.  Both are sums of the same d c terms over
    ~B * W / 2 positions (the bias with factor 1, a weight with an input sample), so they carry the same absolute
    rounding error; but a bias is one number per channel, and when that sum happens to cancel (conv2.bias comes out
    at under 1 % of conv2.weight's gradient for some upstream gradients) a floor taken from the bias alone leaves an
    honest float32 sum no room -- the float32 reference itself misses it by more, or less, depending on the CPU's
    summation order.  Judged at the layer's scale the bias keeps the element-wise bound of every weight."""
    def fold(d):
        g = dict(d["grads"])
        for n in ("conv1", "conv2"):
            w, b = g[n + ".weight"], g[n + ".bias"]
            g[n + ".weight"] = torch.cat([w.reshape(-1).cpu(), b.reshape(-1).cpu()])
            g[n + ".bias"] = torch.zeros(0)
        return {**d, "grads": g}
    _check_per_tensor(fold(got), {**truth, head: fold(truth[head])}, {**ref32, head: fold(ref32[head])}, head, {**LONG_SUM_BETA, **(beta or {})})


def _window_for(kind, L):
    """the shortest window of a preset's geometry with L final features"""
    a = tskd_b200.ARCH_PRESETS[kind]
    for W in range(a.pool_s * a.pool_s * L, a.pool_s * a.pool_s * L + 64):
        if a.with_shape(3, W).l_out == L:
            return W
    raise AssertionError(L)


def _clean_inputs(oarch, ref, B, seed, p):
    for s in range(seed, seed + 20000, 1000):
        x, age, y, dz, m1, m2 = _inputs(oarch, B, s, p)
        g1, g2 = pool_gaps(ref, x, m1)
        if float(g1.min()) > TIE_GAP and float(g2.min()) > TIE_GAP:
            return x, age, y, dz, m1, m2
    raise AssertionError("no input without near-ties")


def _fused(ref, oarch, x, age, y, mode, p, m1, m2, pos_weight=None):
    model = tskd_b200.B200MyCNN(_arch(oarch), has_out12=oarch.has_out12).to(DEV)
    model.load_state_dict(ref.state_dict())
    tr = B200Trainer(model, mode=mode, dropout=p, pos_weight=pos_weight)
    loss = tr.step(x, age, y, masks=(m1, m2), update=False)
    return {"loss": loss.cpu(), "grads": {k: v.cpu() for k, v in tr.grads().items()}}


# ------------------------------------------------------------------ the fused step and autograd against float64
CASES = [
    # kind, C, W, B, mode, p, pos_weight
    ("mycnn5", 3, 7504, 6, "sequence", 0.1, None),
    ("mycnn5", 3, 7504, 33, "sequence", 0.1, POS_WEIGHT),
    ("mycnn5", 3, 7504, 33, "independent", 0.0, None),
    ("mycnn5", 1, 7504, 6, "independent", 0.1, POS_WEIGHT),
    ("mycnn5", 1, 7504, 33, "sequence", 0.0, None),
    ("mycnn3", 3, 7502, 6, "sequence", 0.0, POS_WEIGHT),       # pool (2, 2): one c2 position after the last pooling window
    ("mycnn3", 3, 7502, 33, "independent", 0.1, None),
    ("mycnn5", 3, 75000, 3, "sequence", 0.1, None),            # the waveform window, 147 tiles
]


@pytest.mark.parametrize("kind,C,W,B,mode,p,pos_weight", CASES)
def test_fused_step_and_autograd_match_float64(kind, C, W, B, mode, p, pos_weight):
    oarch = O.stretched(O.ARCHS[kind], C, W)
    ref = O.make_ref(oarch, seed=B + W)
    x, age, y, dz, m1, m2 = _clean_inputs(oarch, ref, B, B + W, p)
    truth, ref32 = _refs(ref, x, age, mode, m1, m2, dz=dz, target=y, pos_weight=pos_weight)
    got = _fused(ref, oarch, x, age, y, mode, p, m1, m2, pos_weight)
    _check(got, truth, ref32, "bce" if pos_weight is None else "bce_pw")
    _check(_device(ref, _arch(oarch), x, age, mode, m1, m2, dz), truth, ref32, "dz")


# ------------------------------------------------------------------ tile seams
@pytest.mark.parametrize("L", [1023, 1024, 1025, 1152, 1157])
def test_tile_seams_and_the_plan_boundary(L):
    """L = 1023 ends on a last tile of 127 features, 1024 and 1152 are whole tiles, 1025 leaves a last tile of one
    feature, and 1024 / 1025 straddle the point where the pre-activation GEMM takes a second slice of 1024 positions;
    every one against float64, d x included"""
    oarch = O.stretched(O.ARCH_MYCNN5, 3, _window_for("mycnn5", L))
    assert oarch.l_out == L
    ref = O.make_ref(oarch, seed=L)
    x, age, _, dz, m1, m2 = _clean_inputs(oarch, ref, 5, L, 0.1)
    truth, ref32 = _refs(ref, x, age, "sequence", m1, m2, dz=dz)
    _check(_device(ref, _arch(oarch), x, age, "sequence", m1, m2, dz), truth, ref32, "dz")


def test_input_gradient_at_the_samples_two_tiles_share():
    oarch = O.stretched(O.ARCH_MYCNN5, 3, 7504)
    ref = O.make_ref(oarch, seed=3)
    x, age, _, dz, m1, m2 = _clean_inputs(oarch, ref, 4, 3, 0.1)
    truth, ref32 = _refs(ref, x, age, "independent", m1, m2, dz=dz)
    got = _device(ref, _arch(oarch), x, age, "independent", m1, m2, dz)
    a = tskd_b200.ARCH_PRESETS["mycnn5"]
    stride = a.pool_s * a.pool_s * T
    n2 = a.pool_s * (T - 1) + a.pool_k
    span = a.pool_s * (n2 + a.k2 - 2) + a.pool_k + a.k1 - 1
    assert stride < span < 2 * stride
    shared = torch.cat([torch.arange(k * stride, k * stride + span - stride) for k in range(1, oarch.l_out // T)])
    from oracle.train_ref import BETA, assert_close_elem
    assert (got["dx"][:, :, shared] != 0).any()
    assert_close_elem("dx at seams", got["dx"][:, :, shared], truth["dz"]["dx"][:, :, shared], ref32["dz"]["dx"][:, :, shared], beta=BETA)
    _check(got, truth, ref32, "dz")


def _tie_case(B, seed, W):
    """tests/test_gpu_train_edges.py::_tie_case at a long window: exact conv1 arithmetic, and constant runs laid across
    the seams between tiles 0 | 1 and 7 | 8 (x samples 512 and 4096), so pooling windows on both sides of a seam tie"""
    oarch = O.stretched(O.ARCH_MYCNN5, 3, W)
    ref = O.make_ref(oarch, seed=seed)
    g = torch.Generator().manual_seed(seed)
    with torch.no_grad():
        ref.conv1.weight.copy_(torch.randint(-2, 3, ref.conv1.weight.shape, generator=g) / 128.0)
        ref.conv1.bias.copy_(torch.randint(-8, 9, ref.conv1.bias.shape, generator=g) / 128.0)
    x = torch.randint(-8, 9, (B, 3, W), generator=g).float()
    for lo in (480, 4060):
        x[:, :, lo:lo + 80] = torch.randint(-8, 9, (B, 3, 1), generator=g).float()
    age = torch.rand(B, generator=g) * 60 + 20
    dz = torch.randn(B, generator=g)
    return oarch, ref, x, age, dz


def test_exact_pool_ties_across_a_tile_seam_route_to_the_first_maximum():
    oarch, ref, x, age, dz = _tie_case(4, seed=41, W=7504)
    g1, g2 = pool_gaps(ref, x)
    g1_32, g2_32 = pool_gaps(ref, x, dtype=torch.float32)
    for g64, g32 in ((g1, g1_32), (g2, g2_32)):
        ties = g64 == 0
        assert ties.any() and torch.equal(ties, g32 == 0)
        assert float(g64[~ties].min()) > TIE_GAP
    assert (g2[:, T - 4:T + 4] == 0).all()                               # the features either side of the first seam
    truth, ref32 = _refs(ref, x, age, "sequence", None, None, dz=dz)
    _check(_device(ref, _arch(oarch), x, age, "sequence", None, None, dz), truth, ref32, "dz")


def test_saturated_input_and_dropped_positions_at_a_seam():
    oarch = O.stretched(O.ARCH_MYCNN5, 3, 7504)
    ref = O.make_ref(oarch, seed=23)
    for s in range(23, 20023, 1000):
        x, age, _, dz, m1, m2 = _inputs(oarch, 6, s, 0.1)
        x = x * 40.0                                                      # conv1's tanh saturates
        m2[:, T - 1:T + 1] = 0.0                                          # the features either side of a seam are dropped
        m1[:, :, 2 * T - 2:2 * T + 6] = 0.0                               # and the p1 positions around it
        m2[5] = 0.0                                                       # one window loses every feature
        g1, g2 = pool_gaps(ref, x, m1)
        if float(g1.min()) > TIE_GAP and float(g2.min()) > TIE_GAP:
            break
    with torch.no_grad():
        assert (torch.tanh(ref.conv1(x)).abs() == 1.0).any()
    truth, ref32 = _refs(ref, x, age, "sequence", m1, m2, dz=dz)
    # out.weight's gradient is d lin x h1: with the features saturated it carries the sigmoid / tanh error the lstm tensors
    # are granted 4e-6 for (tests/test_gpu_train_edges.py: LSTM_BETA); observed need 1.2e-6
    _check(_device(ref, _arch(oarch), x, age, "sequence", m1, m2, dz), truth, ref32, "dz", {"out.weight": 4e-6})


# ------------------------------------------------------------------ NaN and inf
@pytest.mark.parametrize("mode", ["sequence", "independent"])
@pytest.mark.parametrize("where", ["first", "last", "seam", "+inf", "-inf"])
def test_nan_and_inf_follow_the_reference(where, mode):
    oarch = O.stretched(O.ARCH_MYCNN5, 3, 7504)
    ref = O.make_ref(oarch, seed=71)
    x, age, y, _, m1, m2 = _inputs(oarch, 5, 71, 0.1)
    dz = torch.randn(5, generator=torch.Generator().manual_seed(71))
    pos = {"first": 0, "last": oarch.window - 1, "seam": 4 * T + 3, "+inf": 3700, "-inf": 9}[where]
    x[2, 1, pos] = {"+inf": float("inf"), "-inf": float("-inf")}.get(where, float("nan"))
    truth, ref32 = _refs(ref, x, age, mode, m1, m2, dz=dz, target=y)
    if where in ("first", "last", "seam"):
        assert torch.isnan(truth["z"][2]) and torch.isnan(truth["bce"]["loss"])
    got = _device(ref, _arch(oarch), x, age, mode, m1, m2, dz)
    _check(got, truth, ref32, "dz")
    if mode == "independent":
        clean = [0, 1, 3, 4]
        assert torch.isfinite(got["dx"][clean]).all() and torch.isfinite(got["z"][clean]).all()
    _check(_fused(ref, oarch, x, age, y, mode, 0.1, m1, m2), truth, ref32, "bce")


# ------------------------------------------------------------------ the module under autograd; the frozen front end
def _module(oarch, ref, p):
    m = B200TrainableMyCNN(_arch(oarch), has_out12=oarch.has_out12).to(DEV)
    m.load_state_dict(ref.state_dict())
    m.dropout.p = p
    m.train()
    return m


def _module_grads(m, x, age, y, frozen):
    for k, prm in m.named_parameters():
        prm.grad = None
        prm.requires_grad_(not (frozen and k.startswith("conv")))
    torch.manual_seed(9)                                                  # the same dropout masks in both runs
    loss = nn.BCEWithLogitsLoss()(m(x, age), y)
    loss.backward()
    return loss.detach(), {k: (None if prm.grad is None else prm.grad.clone()) for k, prm in m.named_parameters() if k in BLOB_KEYS}


@pytest.mark.parametrize("C,W", [(3, 7504), (10, 120)])
def test_frozen_conv_gives_the_same_head_gradients(C, W):
    oarch = O.stretched(O.ARCH_MYCNN5, C, W)
    ref = O.make_ref(oarch, seed=5)
    x, age, y, _, _, _ = _inputs(oarch, 12, 5, 0.0)
    x, age, y = x.to(DEV), age.to(DEV), y.to(DEV)
    m = _module(oarch, ref, 0.1)
    loss_a, full = _module_grads(m, x, age, y, frozen=False)
    loss_b, head = _module_grads(m, x, age, y, frozen=True)
    assert torch.equal(loss_a, loss_b)
    for k in BLOB_KEYS:
        if k in CONV_KEYS:
            assert head[k] is None and full[k] is not None and bool((full[k] != 0).any()), k
        else:
            assert torch.equal(head[k], full[k]), k


# torch.profiler runs in a process of its own, as in tests/test_gpu_record.py
_LAUNCH_LIST = r"""
import collections, json, sys
import torch
from torch import nn
import tskd_b200
from tskd_b200.autograd import B200TrainableMyCNN
from torch.profiler import ProfilerActivity, profile

def kernels(fn):
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        torch.ones(1, device=dev).add_(1)
        torch.cuda.synchronize()
        fn()
        torch.cuda.synchronize()
    return collections.Counter(e.name for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA and "b2cnn::" in e.name)

C, W = int(sys.argv[1]), int(sys.argv[2])
dev = torch.device("cuda", 0)
m = B200TrainableMyCNN(tskd_b200.ARCH_PRESETS["mycnn5"].with_shape(C, W)).to(dev)
m.train()
x = torch.randn(9, C, W, device=dev)
age = torch.full((9,), 50.0, device=dev)
y = torch.ones(9, device=dev)
def step():
    m.zero_grad(set_to_none=True)
    nn.BCEWithLogitsLoss()(m(x, age), y).backward()
kernels(lambda: torch.ones(1, device=dev).add_(1))
lists = []
for frozen in (False, True):
    m.conv1.requires_grad_(not frozen); m.conv2.requires_grad_(not frozen)
    step()
    lists.append(kernels(step))
print(json.dumps(lists))
"""


@pytest.mark.parametrize("C,W", [(3, 7504), (10, 120)])
def test_frozen_conv_launches_no_conv_backward(C, W):
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    env = dict(os.environ, PYTHONPATH=os.pathsep.join([root] + [p for p in [os.environ.get("PYTHONPATH")] if p]))
    cmd = [sys.executable] + (["-s"] if sys.flags.no_user_site else []) + ["-c", _LAUNCH_LIST, str(C), str(W)]
    r = subprocess.run(cmd, capture_output=True, text=True, env=env, cwd=root, timeout=600)
    assert r.returncode == 0, r.stderr[-3000:]
    full, frozen = [collections.Counter(d) for d in json.loads(r.stdout.strip().splitlines()[-1])]
    has = lambda c, name: any(name in k for k in c)
    assert has(full, "train_conv_bwd(") and has(full, "train_dfeat(") and has(full, "grad_reduce"), full
    assert has(full, "train_conv_fwd(") and has(full, "train_pre0_partial") and not has(full, "train_dx"), full
    assert not has(frozen, "train_conv_bwd") and not has(frozen, "train_dfeat") and not has(frozen, "grad_reduce"), frozen
    assert has(frozen, "train_lstm_bwd") and has(frozen, "train_wih0_grad"), frozen


# ------------------------------------------------------------------ run-to-run, the eval path, Adam
def _two_runs(C, W, B):
    """two fused sequence steps with dropout, then autograd with d x and d age, twice from the same state: equal bits"""
    oarch = O.stretched(O.ARCH_MYCNN5, C, W)
    ref = O.make_ref(oarch, seed=7)
    x, age, y, dz, m1, m2 = _inputs(oarch, B, 7, 0.1)
    runs = []
    for _ in range(2):
        model = tskd_b200.B200MyCNN(_arch(oarch), has_out12=oarch.has_out12).to(DEV)
        model.load_state_dict(ref.state_dict())
        tr = B200Trainer(model, mode="sequence", dropout=0.1)
        losses = [tr.step(x, age, y, masks=(m1, m2)).cpu() for _ in range(2)]
        runs.append((losses, {k: v.cpu().clone() for k, v in tr.grads().items()}, {k: v.cpu().clone() for k, v in model.state_dict().items()},
                     _device(ref, _arch(oarch), x, age, "sequence", m1, m2, dz)))
    (la, ga, pa, da), (lb, gb, pb, db) = runs
    assert all(torch.equal(a, b) for a, b in zip(la, lb))
    for k in BLOB_KEYS:
        assert torch.equal(ga[k], gb[k]) and torch.equal(pa[k], pb[k]) and torch.equal(da["grads"][k], db["grads"][k]), k
    assert torch.equal(da["dx"], db["dx"]) and torch.equal(da["dage"], db["dage"])


def test_two_runs_give_the_same_bits():
    _two_runs(3, 7504, 40)


@pytest.mark.parametrize("B", [257, 2048])
def test_two_runs_give_the_same_bits_at_the_training_shape(B):
    """[B,10,120]: one tile per window, 257 / 1024 conv-backward CTAs"""
    _two_runs(10, 120, B)


@pytest.mark.parametrize("mode", ["sequence", "independent"])
def test_train_mode_without_dropout_agrees_with_the_generic_path(mode):
    oarch = O.stretched(O.ARCH_MYCNN5, 3, 7504)
    ref = O.make_ref(oarch, seed=81)
    x, age, _, _, _, _ = _inputs(oarch, 9, 81, 0.0)
    sd = ref.state_dict()
    with torch.no_grad():
        train = tskd_b200.mycnn_train_forward(x.to(DEV), age.to(DEV), [sd[k].to(DEV) for k in BLOB_KEYS], _arch(oarch), mode).cpu().numpy()
    model = tskd_b200.B200MyCNN(_arch(oarch), has_out12=oarch.has_out12).to(DEV)
    model.load_state_dict(sd)
    model.set_path("generic")
    ev = model.predict(x.to(DEV), age.to(DEV), mode=mode).cpu().numpy()
    assert rel_err(train, ev) <= 1e-5


def test_three_adam_steps_follow_torch_optim():
    oarch = O.stretched(O.ARCH_MYCNN5, 3, 7504)
    ref = O.make_ref(oarch, seed=0)
    ref.dropout = MaskDropout()
    ref.train()
    m = tskd_b200.B200MyCNN(_arch(oarch), has_out12=oarch.has_out12).to(DEV)
    m.load_state_dict({k: v for k, v in ref.state_dict().items() if not k.startswith("dropout")})
    tr = B200Trainer(m, lr=1e-3, mode="sequence", dropout=0.1)
    opt = torch.optim.Adam(ref.parameters(), lr=1e-3)
    for step in range(3):
        x, age, y, _, m1, m2 = _inputs(oarch, 20, 100 + step, 0.1)
        loss = tr.step(x, age, y, masks=(m1, m2))
        ref.dropout.set(m1, m2)
        opt.zero_grad()
        want = nn.BCEWithLogitsLoss()(ref(x, age), y)
        want.backward()
        opt.step()
        assert abs(float(loss) - float(want)) <= 2e-5 * max(1.0, abs(float(want))), (step, float(loss), float(want))
    sd, named = m.state_dict(), dict(ref.named_parameters())
    for k in BLOB_KEYS:                                                   # as tests/test_gpu_train.py judges it at W = 120
        a, b = sd[k].cpu().numpy().ravel(), named[k].detach().numpy().ravel()
        g = np.abs(named[k].grad.numpy().ravel())
        sel = g > 1e-4 * g.max()
        assert np.abs(a[sel] - b[sel]).max() <= 2e-5, (k, np.abs(a[sel] - b[sel]).max())
        assert np.abs(a - b).max() <= 6.1e-3


# ------------------------------------------------------------------ the workspace
def test_workspace_is_checked_and_not_overrun():
    oarch = O.stretched(O.ARCH_MYCNN5, 3, 7504)
    ref = O.make_ref(oarch, seed=2)
    B = 10
    x, age, y, _, m1, m2 = (t.to(DEV) for t in _inputs(oarch, B, 2, 0.1))
    lib = capi.load_library()
    cfg = capi.make_config(_arch(oarch), 0)
    need = int(lib.b2cnn_train_workspace_bytes(ctypes.byref(cfg), B))
    assert need > 0
    model = tskd_b200.B200MyCNN(_arch(oarch), has_out12=oarch.has_out12).to(DEV)
    model.load_state_dict(ref.state_dict())
    params = model.packed_weights().to(DEV).contiguous()
    grads, m_, v_ = torch.zeros_like(params), torch.zeros_like(params), torch.zeros_like(params)
    loss = torch.zeros(1, device=DEV)
    guard = 1 << 20
    buf = torch.full((need + guard,), 0xA5, dtype=torch.uint8, device=DEV)
    opt = capi.Adam(1e-3, 0.9, 0.999, 1e-8)
    ptr = lambda t: ctypes.c_void_p(t.data_ptr())
    st = ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)
    call = lambda nbytes: lib.b2cnn_train_step(ctypes.byref(cfg), ptr(params), ptr(m_), ptr(v_), ptr(grads), 1, ctypes.byref(opt), 0, ptr(x), B,
                                               ptr(age), ptr(y), capi.MODE_SEQUENCE, ptr(m1), ptr(m2), ptr(loss), ptr(buf), nbytes, st)
    assert call(need - 1) != 0 and "workspace" in lib.b2cnn_last_error().decode()
    assert (grads == 0).all() and float(loss) == 0.0                      # refused before any launch
    assert call(need) == 0
    torch.cuda.synchronize()
    assert bool(torch.isfinite(loss).all()) and bool((grads != 0).any())
    assert bool((buf[need:] == 0xA5).all())
