"""GPU: extra heads over one SlidingScorer's features (SlidingScorer.set_heads / push(heads=True),
b2cnn_slide_set_heads / _push_heads, csrc/b2cnn_slide.cu).

The criterion is bit identity.  Scorer A runs model M0 with heads M1..MK attached; twin scorers of M0..MK get the same
samples, ages and lifecycle calls.  At every push row 0 of A.push(heads=True) must be torch.equal to the M0 twin and row
i to twin i, NaN for NaN.  The heads share M0's conv weights; their LSTM, Linear and age_coef are seeded per head.  On
the generic path each row must also equal predict(window, path="generic", small_kernel=0) of its model."""
import copy
import ctypes
from dataclasses import replace

import pytest
import torch

import tskd_b200
from conftest import load_golden
from oracle import mycnn_torch as O
from oracle.infer_ref import centre_affine, random_affine
from tskd_b200 import capi

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
BF, F32 = torch.bfloat16, torch.float32
M5 = (10, 5, 3, 2)


def _same(a, b):
    """bit-identical, NaN for NaN"""
    na, nb = torch.isnan(a), torch.isnan(b)
    return torch.equal(na, nb) and torch.equal(a[~na], b[~nb])


def _seg(P, C, S, dtype, seed):
    return tskd_b200.synth.make_windows(P, C, S, "normal", seed=seed, dtype=dtype)


def _poison(seg, t):
    """NaN and +-inf samples in a few streams, at the segment's start, middle and end (tails, seams, main features)"""
    P, C, S = seg.shape
    rows = [(3 * t + j) % P for j in range(3)]
    seg[rows[0], 0, S - 2] = float("nan")
    seg[rows[1], C - 1, S // 2] = float("inf")
    seg[rows[2], 0, 1] = float("-inf")


# ------------------------------------------------------------------ models
def _head_sd(sd, seed):
    """the state dict with other LSTM, Linear and head weights and the same conv / affine weights"""
    g = torch.Generator().manual_seed(seed)
    return {k: (v if k.startswith(("conv", "affine")) else v + 0.05 * torch.randn(v.shape, generator=g, dtype=v.dtype))
            for k, v in sd.items()}


def _like(m0, sd, age_coef, generic):
    m = tskd_b200.B200MyCNN(replace(m0.arch, age_coef=age_coef), has_out12="out1.weight" in sd,
                            path="generic" if generic else "auto").to(DEV)
    m.load_state_dict(sd)
    if generic:
        m.set_option("small_kernel", 0)
    return m


def _tc_family(kind, C, W, K, seed):
    """M0 of a tensor-core geometry and K heads of the same conv weights"""
    ref = O.make_ref(O.stretched(O.ARCHS[kind], C, W), seed=seed)
    arch = replace(tskd_b200.ARCH_PRESETS[kind].with_shape(C, W), age_coef=ref.arch.age_coef)
    m0 = tskd_b200.B200MyCNN(arch, has_out12=ref.arch.has_out12).to(DEV)
    sd = dict(ref.state_dict())
    m0.load_state_dict(sd)
    return m0, sd, [_like(m0, _head_sd(sd, seed * 10 + i), 1e-3 * (i + 1), False) for i in range(K)]


def _gen_family(geo, K, seed, act="tanh", aff_seed=None):
    """M0 for the generic path: the MyCNN5.pth golden (geo None) or a seeded model, and K heads"""
    if geo is None:
        _, sd = load_golden("mycnn5_xtestinput.npz")
        m0 = tskd_b200.B200MyCNN.from_reference(sd, age_coef=1e-8, path="generic").to(DEV)
        sd = {k: v.cpu() for k, v in m0.state_dict().items()}
    else:
        C, k1, k2, pk, ps, W = geo
        ref = O.make_ref(O.RefArch(in_channels=C, k1=k1, k2=k2, pool_k=pk, pool_s=ps, window=W, age_coef=1e-4, has_out12=False),
                         seed=seed)
        sd = dict(ref.state_dict())
        if aff_seed is not None:
            aff = centre_affine(ref, tskd_b200.synth.make_windows(4, C, W, "normal", seed=seed), act, random_affine(aff_seed))
            sd.update(zip(("affine1_scale", "affine1_shift", "affine2_scale", "affine2_shift"), aff))
        arch = tskd_b200.ArchConfig(in_channels=C, k1=k1, k2=k2, pool_k=pk, pool_s=ps, window=W, age_coef=1e-4, act=act,
                                    affine=aff_seed is not None)
        m0 = tskd_b200.B200MyCNN(arch, has_out12=False, path="generic").to(DEV)
        m0.load_state_dict(sd)
    m0.set_option("small_kernel", 0)
    return m0, sd, [_like(m0, _head_sd(sd, seed * 10 + i), 1e-3 * (i + 1), True) for i in range(K)]


# ------------------------------------------------------------------ the ward: A with heads, twins of every model
class Ward:
    def __init__(self, m0, heads, P, S, dtype, path, seed, attach=True):
        self.models, self.P, self.S, self.dtype, self.path = [m0] + list(heads), P, S, dtype, path
        self.C, self.W = m0.arch.in_channels, m0.arch.window
        self.A = tskd_b200.SlidingScorer(m0, P, S, dtype, path=path)
        self.twins = [tskd_b200.SlidingScorer(m, P, S, dtype, path=path) for m in self.models]
        assert self.A.path == path
        if attach:
            self.A.set_heads(heads)
        self.age = tskd_b200.synth.make_ages(P, seed=seed).to(DEV)
        self.stream = None                       # host copy of the last W samples per patient (generic checks)

    def scorers(self):
        return [self.A] + self.twins

    def push(self, seg):
        seg_d = seg.to(DEV)
        out = self.A.push(seg_d, self.age, heads=True)
        tw = [t.push(seg_d, self.age) for t in self.twins]
        if self.path == "generic":
            s = seg.float()
            self.stream = s if self.stream is None else torch.cat([self.stream, s], dim=2)[:, :, -self.W:]
        assert (out is None) == (tw[0] is None)
        if out is None:
            return None
        K = len(self.A.heads)
        assert out.shape == (1 + K, self.P)
        assert _same(out[0], tw[0])
        nan0 = torch.isnan(out[0])
        for i in range(1, K + 1):
            twin = tw[self.models.index(self.A.heads[i - 1])]
            assert _same(out[i], twin), i
            assert torch.equal(torch.isnan(out[i]), nan0), i
        return out

    def check_predict(self, out):
        """generic path: every row equals predict() of its model on the true windows (patients with a full stream)"""
        if out is None or self.stream is None or self.stream.shape[2] < self.W:
            return
        win = self.stream.to(self.dtype).to(DEV)
        for i, m in enumerate([self.A.model] + list(self.A.heads)):
            assert _same(out[i], m.predict(win, self.age)), i


def _run(w, pushes, seed, poison=True):
    scored = 0
    for t in range(pushes):
        seg = _seg(w.P, w.C, w.S, w.dtype, seed * 1000 + t)
        if poison and t % 3 == 1:
            _poison(seg, t)
        out = w.push(seg)
        if w.path == "generic":
            w.check_predict(out)
        scored += 0 if out is None else 1
    assert scored > 0


TC_CASES = {
    #                  kind, C, W, S, dtype, P, K, pushes
    "m5-c3-bf16-k1": ("mycnn5", 3, 7504, 752, BF, 130, 1, 12),
    "m5-c3-bf16-k2-p1": ("mycnn5", 3, 7504, 752, BF, 1, 2, 11),
    "m5-c3-bf16-k3": ("mycnn5", 3, 7504, 752, BF, 130, 3, 12),
    "m5-c3-bf16-k8": ("mycnn5", 3, 7504, 752, BF, 130, 8, 11),
    "m3-c1-f32-w7502-k3": ("mycnn3", 1, 7502, 752, F32, 130, 3, 12),        # W % 4 != 0
    "m3-c1-f32-w7502-k1-p1": ("mycnn3", 1, 7502, 752, F32, 1, 1, 11),
    "m5-c3-bf16-w75000-p4096-k3": ("mycnn5", 3, 75000, 7500, BF, 4096, 3, 11),
}


@pytest.mark.parametrize("name", list(TC_CASES))
def test_heads_tensorcore(name):
    kind, C, W, S, dtype, P, K, pushes = TC_CASES[name]
    i = list(TC_CASES).index(name)
    m0, _, heads = _tc_family(kind, C, W, K, seed=3 + i)
    _run(Ward(m0, heads, P, S, dtype, "tensorcore", seed=i), pushes, seed=i)


GEN_CASES = {
    #                    geo (None: golden), act, aff, S, dtype, P, K, pushes
    "golden-w120-s12-k2": (None, "tanh", None, 12, F32, 130, 2, 12),
    "golden-w120-s12-k8-p1": (None, "tanh", None, 12, F32, 1, 8, 11),
    "c10-relu-negaff-k3": ((10,) + M5 + (600,), "relu", 1, 100, F32, 130, 3, 8),
    "c10-relu-negaff-k1-bf16": ((10,) + M5 + (600,), "relu", 1, 100, BF, 40, 1, 8),
}


@pytest.mark.parametrize("name", list(GEN_CASES))
def test_heads_generic(name):
    geo, act, aff, S, dtype, P, K, pushes = GEN_CASES[name]
    i = list(GEN_CASES).index(name)
    m0, _, heads = _gen_family(geo, K, seed=20 + i, act=act, aff_seed=aff)
    _run(Ward(m0, heads, P, S, dtype, "generic", seed=30 + i), pushes, seed=30 + i)


# ------------------------------------------------------------------ no cold start
@pytest.mark.parametrize("path", ["tensorcore", "generic"])
def test_heads_attached_late_score_at_once(path):
    if path == "tensorcore":
        m0, _, heads = _tc_family("mycnn5", 3, 7504, 3, seed=40)
        P, S, dtype, n_before = 130, 752, BF, 12
    else:
        m0, _, heads = _gen_family(None, 3, seed=41)
        P, S, dtype, n_before = 64, 12, F32, 13
    w = Ward(m0, heads, P, S, dtype, path, seed=42, attach=False)
    for t in range(n_before):                                   # n_before > W / S: windows are complete
        out = w.push(_seg(P, w.C, S, dtype, 4200 + t))
        assert t < 9 or out.shape == (1, P)
    w.A.set_heads(heads)
    for t in range(3):
        out = w.push(_seg(P, w.C, S, dtype, 4300 + t))
        assert out.shape == (4, P) and not torch.isnan(out).any()
        if path == "generic":
            w.check_predict(out)


# ------------------------------------------------------------------ lifecycle
@pytest.mark.parametrize("path", ["tensorcore", "generic"])
def test_heads_through_the_lifecycle(path):
    if path == "tensorcore":
        m0, _, heads = _tc_family("mycnn5", 3, 7504, 2, seed=50)
        P, S, dtype = 130, 752, BF
    else:
        m0, _, heads = _gen_family((10,) + M5 + (600,), 2, seed=51, act="relu", aff_seed=2)
        P, S, dtype = 130, 100, F32
    w = Ward(m0, heads, P, S, dtype, path, seed=52)
    C, W = w.C, w.W
    other = tskd_b200.SlidingScorer(m0, 8, S, dtype, path=path)
    seed = 5200

    def each(fn):
        for sc in w.scorers():
            fn(sc)

    def pushes(n):
        nonlocal seed
        for _ in range(n):
            seed += 1
            w.push(_seg(P, C, S, dtype, seed))
            assert torch.equal(w.A.samples_seen, w.twins[0].samples_seen)

    each(lambda sc: sc.admit([0, 5], _seg(2, C, W, dtype, 1)))          # before any push, H = W: scored at push 1
    pushes(2)
    each(lambda sc: sc.admit([7, 129], _seg(2, C, W - S - 8, dtype, 2)))   # H < W
    each(lambda sc: sc.discharge([1, 2, 64]))
    pushes(W // S + 1)
    for t in range(3):
        other.push(_seg(8, C, S, dtype, 5300 + t))
    for t in range(W // S):
        other.push(_seg(8, C, S, dtype, 5310 + t))
    state = other.export([0, 3, 6])
    each(lambda sc: sc.restore([2, 10, 11], state))                      # a restored patient is scored by every head
    each(lambda sc: sc.discharge([11]))
    pushes(2)
    each(lambda sc: sc.reset())                                          # heads stay attached
    assert len(w.A.heads) == 2
    pushes(W // S + 2)


# ------------------------------------------------------------------ snapshot and atomicity
@pytest.mark.parametrize("path", ["tensorcore", "generic"])
def test_heads_are_snapshots(path):
    if path == "tensorcore":
        m0, sd, heads = _tc_family("mycnn5", 3, 7504, 1, seed=60)
        P, S, dtype, n = 64, 752, BF, 10
    else:
        m0, sd, heads = _gen_family(None, 1, seed=61)
        P, S, dtype, n = 64, 12, F32, 10
    m1 = heads[0]
    frozen = copy.deepcopy(m1)                                           # M1's weights at set_heads
    new = _like(m1, _head_sd(sd, 6100), m1.arch.age_coef, path == "generic")   # what M1's weights will be changed to
    w = Ward(m0, [m1], P, S, dtype, path, seed=62)
    w.twins[1] = None                                                    # M1 changes below: its own twin would go stale
    w.models.append(frozen)
    w.twins.append(tskd_b200.SlidingScorer(frozen, P, S, dtype, path=path))
    w.models.append(new)
    w.twins.append(tskd_b200.SlidingScorer(new, P, S, dtype, path=path))
    plain = tskd_b200.SlidingScorer(m0, P, S, dtype, path=path)         # never has heads
    seed = 6200

    def push_rows():
        nonlocal seed
        seed += 1
        seg = _seg(P, w.C, S, dtype, seed).to(DEV)
        out = w.A.push(seg, w.age, heads=True)
        tw = [t.push(seg, w.age) if t is not None else None for t in w.twins]
        want0 = plain.push(seg, w.age)
        return out, tw, want0

    for _ in range(n):
        out, tw, want0 = push_rows()
    assert _same(out[0], want0) and _same(out[1], tw[2])
    m1.load_state_dict(new.state_dict())                                 # later weight changes do not reach the copy
    m1.sync_weights()
    out, tw, want0 = push_rows()
    assert _same(out[1], tw[2]) and not _same(out[1], tw[3])
    w.A.set_heads([m1])                                                  # until set_heads is called again
    out, tw, want0 = push_rows()
    assert _same(out[1], tw[3]) and _same(out[0], want0)
    w.A.set_heads([])
    assert w.A.heads == ()
    out, tw, want0 = push_rows()
    assert out.shape == (1, P) and _same(out[0], want0)
    seg = _seg(P, w.C, S, dtype, 6999).to(DEV)
    assert _same(w.A.push(seg, w.age), plain.push(seg, w.age))           # heads=False: as a scorer without heads


# ------------------------------------------------------------------ errors
def _set_heads_rc(sc, handles):
    arr = (ctypes.c_void_p * max(len(handles), 1))(*handles)
    rc = sc._lib.b2cnn_slide_set_heads(sc._s, arr, len(handles), torch.cuda.current_stream().cuda_stream)
    torch.cuda.synchronize()
    return rc


def test_set_heads_errors_change_nothing():
    m0, sd, heads = _tc_family("mycnn5", 3, 7504, 2, seed=70)
    P, S = 40, 752
    w = Ward(m0, heads, P, S, BF, "tensorcore", seed=71)
    for t in range(11):
        w.push(_seg(P, 3, S, BF, 7100 + t))
    lib, h = w.A._lib, [m._ensure_handle()[1].value for m in heads]
    EINVAL, EARCH, ESTATE = capi.EINVAL, capi.EARCH, capi.ESTATE
    assert lib.b2cnn_slide_set_heads(w.A._s, None, 1, None) == EINVAL                      # null array
    assert lib.b2cnn_slide_set_heads(None, None, 0, None) == EINVAL
    assert _set_heads_rc(w.A, h + [None]) == EINVAL                                       # null handle
    assert _set_heads_rc(w.A, h * 5) == EINVAL                                            # 10 > 8
    assert lib.b2cnn_slide_set_heads(w.A._s, (ctypes.c_void_p * 1)(h[0]), -1, None) == EINVAL
    bare = ctypes.c_void_p()                                                              # no weights
    cfg = capi.make_config(m0.arch, 0)
    assert lib.b2cnn_create(ctypes.byref(cfg), ctypes.byref(bare)) == capi.OK
    try:
        assert _set_heads_rc(w.A, [h[0], bare.value]) == EINVAL
    finally:
        lib.b2cnn_destroy(bare)
    other_arch = _tc_family("mycnn5", 3, 7500, 1, seed=72)[0]
    assert _set_heads_rc(w.A, [other_arch._ensure_handle()[1].value]) == EARCH
    sd_conv = dict(sd)
    sd_conv["conv2.bias"] = sd_conv["conv2.bias"] + 0.01
    other_conv = _like(m0, sd_conv, 1e-3, False)
    assert _set_heads_rc(w.A, [h[0], other_conv._ensure_handle()[1].value]) == ESTATE     # other front-end digest
    with pytest.raises(RuntimeError, match="b2cnn error 5"):
        w.A.set_heads([heads[0], other_conv])
    with pytest.raises(ValueError):
        w.A.set_heads([heads[0], other_arch])
    assert lib.b2cnn_slide_n_heads(w.A._s) == 2 and lib.b2cnn_slide_n_heads(None) == -1
    assert w.A.heads == tuple(heads)
    for t in range(3):                                                                    # outputs unchanged
        w.push(_seg(P, 3, S, BF, 7200 + t))
    w.A.set_heads([m0])                                                                   # the scorer's own handle
    out = w.A.push(_seg(P, 3, S, BF, 7300).to(DEV), w.age, heads=True)
    assert out.shape == (2, P) and _same(out[1], out[0])
    if torch.cuda.device_count() < 2:
        return                                                                            # another-device case: needs two GPUs
    far = _like(m0, sd, 1e-3, False).to("cuda:1")
    assert _set_heads_rc(w.A, [far._ensure_handle()[1].value]) == EINVAL


def test_head_on_another_gpu():
    if torch.cuda.device_count() < 2:
        pytest.skip("needs two GPUs: a head on another device than the scorer")
    m0, sd, _ = _tc_family("mycnn5", 3, 7504, 0, seed=73)
    sc = tskd_b200.SlidingScorer(m0, 8, 752)
    far = _like(m0, sd, 1e-3, False).to("cuda:1")
    with pytest.raises(ValueError):
        sc.set_heads([far])


def test_own_weights_changed_since_reset():
    m0, sd, heads = _tc_family("mycnn5", 3, 7504, 1, seed=74)
    sc = tskd_b200.SlidingScorer(m0, 8, 752)
    m0.load_state_dict(_head_sd(sd, 7400))                                # head-only change of the scorer's model
    with pytest.raises(RuntimeError, match="b2cnn error 5"):
        sc.set_heads(heads)
    assert sc.heads == ()
    sc.reset()
    sc.set_heads(heads)


@pytest.mark.parametrize("path", ["tensorcore", "generic"])
def test_conv_change_with_a_stale_head(path):
    """new conv weights of the scorer's model and reset(): push(heads=True) fails and names the head; push() runs"""
    if path == "tensorcore":
        m0, sd, heads = _tc_family("mycnn5", 3, 7504, 2, seed=75)
        P, S, dtype = 24, 752, BF
    else:
        m0, sd, heads = _gen_family(None, 2, seed=76)
        P, S, dtype = 24, 12, F32
    sc = tskd_b200.SlidingScorer(m0, P, S, dtype, path=path)
    sc.set_heads(heads)
    C = m0.arch.in_channels
    for t in range(3):
        sc.push(_seg(P, C, S, dtype, 7500 + t).to(DEV), heads=True)
    sd2 = dict(sd)
    sd2["conv1.weight"] = sd2["conv1.weight"] * 1.01
    m0.load_state_dict(sd2)
    sc.reset()
    twin = tskd_b200.SlidingScorer(m0, P, S, dtype, path=path)
    seg = _seg(P, C, S, dtype, 7600).to(DEV)
    with pytest.raises(RuntimeError, match=r"head 0 .*b2cnn error 5"):
        sc.push(seg, heads=True)
    for t in range(m0.arch.window // S + 2):                               # the failed push changed nothing
        seg = _seg(P, C, S, dtype, 7700 + t).to(DEV)
        a, b = sc.push(seg), twin.push(seg)
        assert (a is None) == (b is None) and (a is None or _same(a, b)), t
    sc.set_heads([m0])
    out = sc.push(seg, heads=True)
    assert _same(out[0], out[1]) and _same(out[0], twin.push(seg))


def test_trainable_candidate_as_head():
    """a B200TrainableMyCNN with frozen conv weights, trained a few steps, is a head like any model"""
    m0, sd, _ = _tc_family("mycnn5", 3, 7504, 0, seed=77)
    cand = tskd_b200.B200TrainableMyCNN(m0.arch, has_out12="out1.weight" in sd).to(DEV)
    cand.load_state_dict(sd)
    cand.conv1.requires_grad_(False)
    cand.conv2.requires_grad_(False)
    opt = torch.optim.Adam([p for p in cand.parameters() if p.requires_grad], lr=1e-2)
    x = _seg(8, 3, 7504, F32, 7800).to(DEV)
    y = (torch.arange(8, device=DEV) % 2).float()
    cand.train()
    for _ in range(3):
        opt.zero_grad()
        torch.nn.functional.binary_cross_entropy_with_logits(cand(x, torch.full((8,), 60.0, device=DEV)), y).backward()
        opt.step()
    cand.eval()
    assert torch.equal(cand.conv1.weight, m0.conv1.weight) and not torch.equal(cand.lstm.weight_ih_l0, m0.lstm.weight_ih_l0)
    _run(Ward(m0, [cand], 64, 752, BF, "tensorcore", seed=78), 11, seed=78)
