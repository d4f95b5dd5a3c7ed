"""GPU: the generic path of the sliding-window scorer (SlidingScorer(..., path="generic" / "auto"),
b2cnn_slide_create_path, csrc/b2cnn_slide.cu): exact fp32 CUDA-core kernels for every model the library accepts.

Every patient's stream is simulated on the host (Ward, as in tests/test_gpu_slide_lifecycle.py).  After each push every
patient with samples_seen >= W is judged element by element against the float64 reference of oracle/infer_ref.py
(check_elems: logits at beta = 2^-20, features at the generic-features grant 2e-6 of tests/test_gpu_infer_elem.py; NaN
and infinities exactly where the reference has them), every other patient must be NaN.  The logits and features must
also be bit-identical to predict(window, mode="independent") and features(window) of a model with path="generic" and
small_kernel=0 on the same windows: the scorer runs the same front-end kernel and the same projection order."""
import ctypes
import os
from collections import namedtuple
from dataclasses import replace

import numpy as np
import pytest
import torch

import tskd_b200
from conftest import GOLDEN, load_golden
from oracle import mycnn_torch as O
from oracle.infer_ref import centre_affine, infer_reference, random_affine
from oracle.train_ref import BETA, check_elems
from tskd_b200 import capi

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
BF, F32 = torch.bfloat16, torch.float32
BETA_LOGITS = BETA
BETA_FEATURES = 2e-6                      # BETA_GENERIC_FEATURES of tests/test_gpu_infer_elem.py
# Two grants, each for named cases only.  The scorer's values there are bit-identical to predict() / features() on
# the same windows (asserted before the bound), so they measure the generic front end's own fp32 rounding on these
# inputs, not the sliding.  Measured on one H100 80GB HBM3:
#   * MyCNN4 golden on physiological streams with S = W: one feature per window group at up to 3.1e-6, and one logit
#     at 1.01e-6 of a batch whose logits are all below 1.7e-2;
#   * m5-c10-tanh-aff-s8: one logit at 1.00e-6 of a batch whose logits are all below 4.6e-3.
BETA_LOGITS_SMALL_SCALE = 2e-6
BETA_FEATURES_PHYSIO = 4e-6
COEF = 1e-4


def _same(a, b):
    """bit-identical, NaN for NaN (None for None)"""
    if a is None or b is None:
        return a is None and b is None
    na, nb = torch.isnan(a), torch.isnan(b)
    return torch.equal(na, nb) and torch.equal(a[~na], b[~nb])


def _lattice(arch):
    """(F, R): feature stride and receptive field of one feature"""
    F = arch.pool_s ** 2
    return F, arch.pool_s * (arch.pool_k + arch.k2 - 2) + arch.pool_k + arch.k1 - 1


def _pair(geo, act="tanh", aff_seed=None, seed=0, path="generic"):
    """(ref, model, affine): a random float64-able reference and the library model with its weights"""
    C, k1, k2, pk, ps, W = geo
    ref = O.make_ref(O.RefArch(in_channels=C, k1=k1, k2=k2, pool_k=pk, pool_s=ps, window=W, age_coef=COEF, has_out12=False),
                     seed=seed)
    aff = None
    if aff_seed is not None:
        clean = tskd_b200.synth.make_windows(4, C, W, "normal", seed=seed)
        aff = centre_affine(ref, clean, act, random_affine(aff_seed))
    arch = tskd_b200.ArchConfig(in_channels=C, k1=k1, k2=k2, pool_k=pk, pool_s=ps, window=W, age_coef=COEF, act=act,
                                affine=aff is not None)
    m = tskd_b200.B200MyCNN(arch, has_out12=False, path=path).to(DEV)
    sd = dict(ref.state_dict())
    if aff is not None:
        sd.update(zip(("affine1_scale", "affine1_shift", "affine2_scale", "affine2_shift"), aff))
    m.load_state_dict(sd)
    m.set_option("small_kernel", 0)
    return ref, m, aff


def _golden(n):
    """(ref, model) of the MyCNN{n} golden checkpoint at W = 120, age_coef 1e-8 as its goldens"""
    g, sd = load_golden("mycnn5_xtestinput.npz" if n == 5 else f"mycnn{n}_ckpt.npz")
    m = tskd_b200.B200MyCNN.from_reference(sd, age_coef=1e-8, path="generic").to(DEV)
    m.set_option("small_kernel", 0)
    ref = O.RefMyCNN(replace(O.ARCHS[f"mycnn{n}"], age_coef=1e-8))
    ref.load_state_dict(sd)
    return ref.eval(), m


class Ward:
    """A generic-path scorer and the host-side truth of its P streams: own[p] holds the last W samples of p's stream."""

    def __init__(self, ref, m, P, S, dtype, seed, act="tanh", aff=None, path="generic", beta_z=BETA_LOGITS, beta_f=BETA_FEATURES):
        self.ref, self.m, self.P, self.S, self.dtype, self.act, self.aff = ref, m, P, S, dtype, act, aff
        self.beta_z, self.beta_f = beta_z, beta_f
        self.W, self.C = m.arch.window, m.arch.in_channels
        self.sc = tskd_b200.SlidingScorer(m, P, S, dtype, path=path)
        assert self.sc.path == "generic"
        self.own = [torch.empty(self.C, 0, dtype=dtype) for _ in range(P)]
        self.seen = np.zeros(P, dtype=np.int64)
        self.age = tskd_b200.synth.make_ages(P, seed=seed)
        self.age_dev = self.age.to(DEV)
        self.n = 0
        self.pairs = []
        self.judged = 0

    def admit(self, idx, hist=None):
        """hist: CPU [k, C, H] or None"""
        self.sc.admit(idx, hist.to(DEV) if hist is not None else None)
        for j, p in enumerate(idx):
            self.own[p] = hist[j].clone() if hist is not None else torch.empty(self.C, 0, dtype=self.dtype)
            self.seen[p] = hist.shape[2] if hist is not None else 0

    def discharge(self, idx):
        self.sc.discharge(idx)
        self.seen[list(idx)] = -1

    def reset(self):
        self.sc.reset()
        self.own = [torch.empty(self.C, 0, dtype=self.dtype) for _ in range(self.P)]
        self.seen[:] = 0

    def push(self, seg, judge=True, features=True):
        """seg: [P, C, S] on the device (any view); judges every valid patient; returns the push's output"""
        out = self.sc.push(seg, self.age_dev)
        self.n += 1
        segc = seg.cpu()
        for p in range(self.P):
            if self.seen[p] >= 0:
                self.own[p] = torch.cat([self.own[p], segc[p]], dim=1)[:, -self.W:]
                self.seen[p] += self.S
        valid = self.seen >= self.W
        assert np.array_equal(self.sc.samples_seen.cpu().numpy(), self.seen), self.n
        if not valid.any():
            assert out is None, self.n
            return out
        assert out is not None, self.n
        assert torch.isnan(out[torch.from_numpy(~valid).to(DEV)]).all(), self.n
        if judge:
            self.judge(out, np.flatnonzero(valid), self.n, features)
        return out

    def judge(self, out, rows, tag, features=True):
        rows = sorted(int(r) for r in rows)
        win = torch.stack([self.own[p] for p in rows])
        assert win.shape[2] == self.W
        age = self.age[rows]
        kw = dict(act=self.act, affine=self.aff)
        truth, ref32 = infer_reference(self.ref, win, age, **kw), infer_reference(self.ref, win, age, dtype=torch.float32, **kw)
        wd, rd = win.to(DEV), torch.tensor(rows, device=DEV)
        if out is not None:
            assert _same(out[rd], self.m.predict(wd, age.to(DEV))), tag            # predict(path=generic, small_kernel=0)
            self.pairs.append((f"z[{tag}]", out[rd].clone(), truth["z"], ref32["z"], self.beta_z))
        if features:
            f = self.sc.features()
            bad = torch.from_numpy(self.seen < self.W).to(DEV)
            assert torch.isnan(f[bad]).all(), tag
            assert _same(f[rd], self.m.features(wd)), tag
            self.pairs.append((f"features[{tag}]", f[rd].clone(), truth["features"], ref32["features"], self.beta_f))
        self.judged += len(rows)

    def check(self):
        assert self.judged > 0
        check_elems(self.pairs, os.environ.get("PYTEST_CURRENT_TEST", "").split(" ")[0])


def _stream(P, C, n, dtype, seed, dist="normal"):
    return tskd_b200.synth.make_windows(P, C, n, dist, seed=seed, dtype=dtype)


def _inject(x, S, R):
    """NaN at the first stream sample and at the last; +-inf in a tail (the last samples of a push), a seam (the
    first samples of the next push) and main features (mid-push), in different patients and pushes"""
    P, C, N = x.shape
    n_push = N // S
    x[0, 0, 0] = float("nan")
    x[1 % P, C - 1, N - 1] = float("nan")
    k = max(1, n_push // 2)
    x[2 % P, 0, k * S - 1] = float("inf")                          # last sample of push k: the tail of push k + 1
    x[3 % P, C - 1, k * S + min(R // 2, S - 1)] = float("-inf")     # inside the seam of push k + 1
    x[4 % P, C // 2, (k + 1) * S - 1 - S // 2] = float("inf")       # mid-push
    x[5 % P, 0, min(N - 1, (k + 1) * S + S // 2)] = float("nan")    # mid-push, a later window


def _views(x, view):
    """the stream on the device as a contiguous, row-padded or one-sample-offset buffer; segments are sliced from it"""
    P, C, N = x.shape
    if view == "padded":
        buf = torch.full((P, C, N + 13), float("nan"), dtype=x.dtype, device=DEV)
        buf[:, :, :N] = x
        return buf[:, :, :N]
    if view == "offset":
        buf = torch.full((P, C, N + 8), float("nan"), dtype=x.dtype, device=DEV)
        buf[:, :, 1:N + 1] = x
        return buf[:, :, 1:N + 1]
    return x.to(DEV)


def _segment(xd, n, S, view):
    seg = xd[:, :, n * S:(n + 1) * S]
    return seg.contiguous() if view == "contiguous" else seg


# ------------------------------------------------------------------ the reference's own checkpoints
def test_known_answer_mycnn5_pth(golden5):
    """MyCNN5.pth, X.TESTINPUT pushed as 10 segments of 12 samples at age 50: the notebook's probability; an admission
    with X.TESTINPUT as history has the golden features at once"""
    g, _ = golden5
    m = tskd_b200.B200MyCNN.from_reference(tskd_b200.load_reference_checkpoint(os.path.join(GOLDEN, "MyCNN5.pth"))).to(DEV)
    x = torch.from_numpy(g["x"]).to(DEV)                                # [1, 10, 120] float32
    sc = tskd_b200.SlidingScorer(m, 1, 12, F32, path="auto")
    assert sc.path == "generic"
    outs = [sc.push(x[:, :, 12 * i:12 * (i + 1)], age=50.0, return_prob=True) for i in range(10)]
    assert all(o is None for o in outs[:9])
    prob = float(outs[9][0])
    print(f"slid probability {prob!r}")
    assert abs(prob - 0.5668570399284363) < 2e-7                        # explore_torch.ipynb:4271
    assert np.abs(sc.features().cpu().numpy() - g["features"]).max() < 2e-6
    sc2 = tskd_b200.SlidingScorer(m, 3, 12, F32, path="generic")
    sc2.admit([1], x)
    f = sc2.features()
    assert torch.isnan(f[[0, 2]]).all()
    assert np.abs(f[1:2].cpu().numpy() - g["features"]).max() < 2e-6


@pytest.mark.parametrize("S", [12, 120])
@pytest.mark.parametrize("dtype", [BF, F32], ids=["bf16", "f32"])
@pytest.mark.parametrize("n", [2, 3, 4, 5])
def test_golden_checkpoints_w120(n, dtype, S):
    """MyCNN2/3/4/5 at their window of 120, the reference's trigger (S = 12: 60 s on the 5 s grid) and S = W; 130
    physiological streams (a 128-window projection tile and two more), NaN / inf samples in six of them"""
    ref, m = _golden(n)
    P, W = 130, 120
    F, R = _lattice(m.arch)
    n_push = W // S + 3
    x = _stream(P, m.arch.in_channels, n_push * S, dtype, seed=40 + n, dist="physio")
    _inject(x, S, R)
    xd = x.to(DEV)
    grant = dict(beta_z=BETA_LOGITS_SMALL_SCALE, beta_f=BETA_FEATURES_PHYSIO) if n == 4 else {}
    wd = Ward(ref, m, P, S, dtype, seed=40 + n, **grant)
    for k in range(n_push):
        wd.push(xd[:, :, k * S:(k + 1) * S])
    wd.check()


# ------------------------------------------------------------------ activations, affine, geometries, lattices, views
Case = namedtuple("Case", "geo S dtype act aff view P beta_z", defaults=(BETA_LOGITS,))
M5, M3 = (10, 5, 3, 2), (5, 5, 2, 2)                             # (k1, k2, pool_k, pool_s) of MyCNN5 and MyCNN2/3/4
CASES = {
    "m5-c10-relu-aff-s100": Case((10,) + M5 + (600,), 100, F32, "relu", 1, "padded", 40),
    "m5-c10-identity-s20-w602": Case((10,) + M5 + (602,), 20, BF, "identity", None, "offset", 40),   # W % 4 != 0
    "m5-c10-tanh-aff-s8": Case((10,) + M5 + (240,), 8, BF, "tanh", 2, "contiguous", 40, BETA_LOGITS_SMALL_SCALE),  # S < R
    "m5-c3-relu-s60": Case((3,) + M5 + (300,), 60, BF, "relu", None, "padded", 40),
    "m5-c4-tanh-s48": Case((4,) + M5 + (500,), 48, F32, "tanh", None, "offset", 40),                # S does not divide W
    "m3-c7-identity-aff-s44-w501": Case((7,) + M3 + (501,), 44, F32, "identity", 3, "contiguous", 40),
    "m3-c10-relu-s120": Case((10,) + M3 + (120,), 120, BF, "relu", None, "padded", 40),              # S = W
    "p11-s5": Case((2, 4, 3, 1, 1, 300), 5, F32, "relu", 4, "offset", 24),                           # F = 1, S < R = 6
    "p23-s45-w600": Case((3, 4, 3, 2, 3, 600), 45, BF, "tanh", 5, "padded", 24),                     # F = 9, R = 14
    "p43-s63-w700": Case((4, 6, 4, 4, 3, 700), 63, F32, "identity", None, "contiguous", 24),         # F = 9, R = 27
    "p43-s9-w200": Case((4, 6, 4, 4, 3, 200), 9, BF, "relu", 6, "offset", 24),                       # S < R
    "c16-p44-s32-w1470": Case((16, 3, 8, 4, 4, 1470), 32, F32, "relu", 7, "padded", 20),             # F = 16, R = 46 > S
    "c16-p44-s160-w1470": Case((16, 3, 8, 4, 4, 1470), 160, BF, "tanh", None, "contiguous", 20),
}


@pytest.mark.parametrize("name", list(CASES))
def test_configurations(name):
    c = CASES[name]
    ref, m, aff = _pair(c.geo, c.act, c.aff, seed=10 + list(CASES).index(name))
    F, R = _lattice(m.arch)
    assert m.arch.l_out == (c.geo[-1] - R) // F + 1
    W = c.geo[-1]
    n_push = -(-W // c.S) + 3
    x = _stream(c.P, c.geo[0], n_push * c.S, c.dtype, seed=7)
    _inject(x, c.S, R)
    xd = _views(x, c.view)
    wd = Ward(ref, m, c.P, c.S, c.dtype, 7, act=c.act, aff=aff, beta_z=c.beta_z)
    for k in range(n_push):
        wd.push(_segment(xd, k, c.S, c.view), features=k % 2 == 0)
    print(f"{name}: F = {F}, R = {R}, L = {m.arch.l_out}, judged {wd.judged} windows")
    wd.check()


# ------------------------------------------------------------------ lifecycle
def _hist(k, C, H, dtype, seed):
    return tskd_b200.synth.make_windows(k, C, H, "normal", seed=seed, dtype=dtype)


@pytest.mark.parametrize("geo,S,dtype", [((10,) + M5 + (600,), 60, BF), ((4, 6, 4, 4, 3, 702), 54, F32)],
                         ids=["m5-c10-bf16", "p43-c4-f32"])
def test_admissions(geo, S, dtype):
    """histories of W, W - S, R - 1, W - 1 and 0 samples before any push, before the first global window and after it;
    NaN / inf in histories; every patient scores from the push at which samples_seen reaches W, on its own stream;
    patients never touched stay bit-identical to a scorer without the lifecycle"""
    ref, m, _ = _pair(geo, seed=21)
    C, W = geo[0], geo[-1]
    F, R = _lattice(m.arch)
    P = 60
    n0 = -(-W // S)
    n_push = n0 + 4
    x = _stream(P, C, n_push * S, dtype, seed=21)
    xd = x.to(DEV)
    wd = Ward(ref, m, P, S, dtype, 21)
    ctl = tskd_b200.SlidingScorer(m, P, S, dtype, path="generic")
    perm = torch.randperm(P, generator=torch.Generator().manual_seed(21)).tolist()
    Hs = [W, W - S, R - 1, W - 1, 0]
    plan = {0: Hs, 2: Hs, n0 + 1: Hs}                                    # before any push, before and after the first window
    at, touched = 0, set()
    for k in range(n_push):
        for i, H in enumerate(plan.get(k, [])):
            idx = perm[at:at + 3]
            at += 3
            touched |= set(idx)
            h = _hist(3, C, H, dtype, 100 * k + i) if H else None
            if h is not None and i == 0:
                h[0, 0, 0] = float("nan")
                h[1, C - 1, H - 2] = float("inf")
            wd.admit(idx, h)
            if H == W:
                wd.judge(None, idx, f"admitted {k}", features=True)          # features() right after a full admission
        seg = xd[:, :, k * S:(k + 1) * S]
        got, want = wd.push(seg), ctl.push(seg, wd.age_dev)
        keep = torch.tensor([p for p in range(P) if p not in touched], device=DEV)
        if want is not None:
            assert torch.equal(got[keep], want[keep]), k
    wd.check()


def test_discharge_readmit_reset_replay_and_determinism():
    geo, S, P = (10,) + M5 + (240,), 24, 40
    ref, m, _ = _pair(geo, seed=31)
    C, W = geo[0], geo[-1]
    x = _stream(1000, C, 14 * S, F32, seed=31)
    xd = x[:P].to(DEV)
    hist = _hist(6, C, W, F32, 31)

    def scenario(wd):
        outs = []
        for k in range(14):
            if k == 3:
                wd.discharge([3, 17, 30])
            if k == 5:
                wd.admit([17, 4, 30, 9, 22, 0], hist)
            out = wd.push(xd[:, :, k * S:(k + 1) * S])
            outs.append(None if out is None else out.clone())
            assert wd.seen[3] == -1 or k < 3
        return outs

    wd = Ward(ref, m, P, S, F32, 31)
    first = scenario(wd)
    wd.check()
    wd.reset()
    assert torch.equal(wd.sc.samples_seen, torch.zeros(P, dtype=torch.int64, device=DEV))
    fresh = tskd_b200.SlidingScorer(m, P, S, F32, path="generic")
    for k in range(12):
        seg = xd[:, :, k * S:(k + 1) * S]
        assert _same(wd.sc.push(seg, wd.age_dev), fresh.push(seg, wd.age_dev)), k
    wd.reset()
    again = scenario(wd)
    assert all(_same(a, b) for a, b in zip(first, again))
    # the first P patients of a 1000-patient scorer, scalar age: bit-identical to the P-patient scorer
    big = tskd_b200.SlidingScorer(m, 1000, S, F32, path="generic")
    small = tskd_b200.SlidingScorer(m, P, S, F32, path="generic")
    xb = x.to(DEV)
    for k in range(12):
        a = big.push(xb[:, :, k * S:(k + 1) * S], age=50.0)
        b = small.push(xb[:P, :, k * S:(k + 1) * S], age=torch.full((P,), 50.0, device=DEV))
        assert _same(None if a is None else a[:P], b), k


def test_full_size_c10():
    """C = 10, W = 75000, S = 7500, P = 200, bf16: the first two windows of every patient"""
    geo, S, P = (10,) + M5 + (75000,), 7500, 200
    ref, m, _ = _pair(geo, seed=41)
    n_push = 11
    xd = _stream(P, 10, n_push * S, BF, seed=41).to(DEV)
    wd = Ward(ref, m, P, S, BF, 41)
    for k in range(n_push):
        wd.push(xd[:, :, k * S:(k + 1) * S], features=k == n_push - 1)
    wd.check()


# ------------------------------------------------------------------ path selection
def test_auto_path():
    """auto on a tensor-core model is the default scorer bit for bit; generic on that model passes the generic bounds;
    auto on C = 10 goes generic"""
    W, S, P = 7504, 1876, 130
    oarch = O.stretched(O.ARCHS["mycnn5"], 3, W)
    ref = O.make_ref(oarch, seed=51)
    arch = replace(tskd_b200.ARCH_PRESETS["mycnn5"].with_shape(3, W), age_coef=oarch.age_coef)
    m = tskd_b200.B200MyCNN(arch, has_out12=oarch.has_out12).to(DEV)
    m.load_state_dict(ref.state_dict())
    x = _stream(P, 3, 6 * S, BF, seed=51)
    _inject(x, S, 24)
    xd = x.to(DEV)
    age = tskd_b200.synth.make_ages(P, seed=51).to(DEV)
    tc, auto = tskd_b200.SlidingScorer(m, P, S), tskd_b200.SlidingScorer(m, P, S, path="auto")
    assert tc.path == "tensorcore" and auto.path == "tensorcore"
    for k in range(6):
        seg = xd[:, :, k * S:(k + 1) * S]
        assert _same(tc.push(seg, age), auto.push(seg, age)), k
    m.set_path("generic")
    m.set_option("small_kernel", 0)
    wd = Ward(ref, m, P, S, BF, 51)
    for k in range(6):
        wd.push(xd[:, :, k * S:(k + 1) * S], features=k == 5)
    wd.check()
    _, m10, _ = _pair((10,) + M5 + (1200,), seed=52, path="auto")
    assert tskd_b200.SlidingScorer(m10, 4, 120, path="auto").path == "generic"
    with pytest.raises(RuntimeError, match="error 2"):
        tskd_b200.SlidingScorer(m10, 4, 120)                           # the default stays the tensor-core path


def _rc_create(m, P, S, path, dtype=capi.DTYPE_F32):
    lib, h = m._ensure_handle()
    s = ctypes.c_void_p()
    rc = lib.b2cnn_slide_create_path(h, P, S, dtype, path, ctypes.byref(s))
    if rc == capi.OK:
        assert lib.b2cnn_slide_path(s) in (capi.PATH_GENERIC, capi.PATH_TENSORCORE)
        lib.b2cnn_slide_destroy(s)
    else:
        assert not s.value
    return rc


def test_errors():
    _, m, _ = _pair((3, 4, 3, 2, 3, 600), seed=61)                      # F = 9
    assert _rc_create(m, 4, 45, capi.PATH_GENERIC) == capi.OK
    assert _rc_create(m, 4, 45, capi.PATH_AUTO) == capi.OK
    assert _rc_create(m, 4, 48, capi.PATH_GENERIC) == capi.EINVAL       # not a multiple of F
    assert _rc_create(m, 4, 0, capi.PATH_GENERIC) == capi.EINVAL
    assert _rc_create(m, 4, 603, capi.PATH_GENERIC) == capi.EINVAL      # S > W
    assert _rc_create(m, 4, 45, 3) == capi.EINVAL                       # B2CNN_PATH_STREAM is not a scorer path
    assert _rc_create(m, 4, 45, 7) == capi.EINVAL
    assert _rc_create(m, 4, 36, capi.PATH_TENSORCORE) == capi.EARCH     # no tensor-core kernel for pool (2, 3)
    with pytest.raises(ValueError):
        tskd_b200.SlidingScorer(m, 4, 48, F32, path="generic")
    with pytest.raises(ValueError):
        tskd_b200.SlidingScorer(m, 4, 45, F32, path="cuda")
    # a window whose generic tile does not fit shared memory (b2cnn_forward refuses it too): EARCH, nothing allocated
    _, big, _ = _pair((16, 3, 8, 4, 4, 4830), seed=62)
    assert _rc_create(big, 4, 160, capi.PATH_GENERIC) == capi.EARCH
    assert "shared memory" in capi.last_error()
    assert _rc_create(big, 4, 160, capi.PATH_AUTO) == capi.EARCH
    # new weights without a reset: ESTATE, as on the tensor-core path
    ref, m3, _ = _pair((4, 6, 4, 4, 3, 700), seed=63)
    sc = tskd_b200.SlidingScorer(m3, 4, 63, F32, path="generic")
    seg = torch.zeros(4, 4, 63, device=DEV)
    sc.push(seg)
    m3.load_state_dict(O.make_ref(ref.arch, seed=64).state_dict())
    with pytest.raises(RuntimeError, match="error 5"):
        sc.push(seg)
    sc.reset()
    assert sc.push(seg) is None
