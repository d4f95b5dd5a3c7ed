"""GPU: heads with shorter windows over one SlidingScorer's feature ring (SlidingScorer.set_heads(..., shorter_windows=
True), b2cnn_slide_set_heads_ex, csrc/b2cnn_slide.cu).

Scorer A runs model M0 at window W with heads M1..MK at windows W_k <= W (W - W_k a multiple of the feature stride),
all with M0's conv weights and their own LSTM, Linear and age_coef.  Twin scorers of each model at its own window and
A's stride get the same segments, ages and lifecycle calls.  At every push row i of A.push(heads=True) must be
torch.equal to twin i, NaN for NaN (a twin that has not emitted yet: row i all NaN).  Every valid element is also judged
against the float64 reference of its model on its own window, at the grants the scorer already has (BETA for logits);
on the generic path every row must also equal predict(last W_k samples, path="generic", small_kernel=0)."""
import ctypes
import os
from dataclasses import replace

import pytest
import torch

import tskd_b200
from conftest import load_golden
from oracle import mycnn_torch as O
from oracle.infer_ref import centre_affine, infer_reference, random_affine
from oracle.train_ref import BETA, check_elems
from test_gpu_generic_elem import _model as _gen_model
from test_gpu_infer_elem import _model as _tc_model
from test_gpu_slide_heads import _poison, _same, _seg
from tskd_b200 import capi

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
BF, F32 = torch.bfloat16, torch.float32


def _check(pairs):
    check_elems(pairs, os.environ.get("PYTEST_CURRENT_TEST", "").split(" ")[0])


# ------------------------------------------------------------------ models: one front end, windows W and W_k
class Row:
    """a model of the family with its float64 reference (ref, act, affine)"""

    def __init__(self, ref, model, act="tanh", aff=None):
        self.ref, self.model, self.act, self.aff = ref, model, act, aff
        self.W = model.arch.window


def _with_conv(ref, conv):
    sd = dict(ref.state_dict())
    sd.update(conv)
    ref.load_state_dict(sd)
    return ref


def _tc_family(kind, C, W, Wks, seed):
    """M0 at W and one head per W_k of the same conv weights (a seeded reference each, age_coef 1e-3 (i + 1))"""
    base = O.stretched(O.ARCHS[kind], C, W)
    ref0 = O.make_ref(base, seed=seed)
    conv = {k: v for k, v in ref0.state_dict().items() if k.startswith("conv")}
    refs = [ref0] + [_with_conv(O.make_ref(replace(base, window=Wk, age_coef=1e-3 * (i + 1)), seed=seed * 10 + i), conv)
                     for i, Wk in enumerate(Wks)]
    return [Row(r, _tc_model(r)) for r in refs]


def _gen_family(geo, Wks, seed, act="tanh", aff_seed=None):
    """generic path: the MyCNN5.pth golden at W = 120 (geo None) or a seeded (C, k1, k2, pool_k, pool_s, W) model, and
    one head per W_k with its conv (and affine) weights"""
    if geo is None:
        _, sd = load_golden("mycnn5_xtestinput.npz")
        m0 = tskd_b200.B200MyCNN.from_reference(sd, age_coef=1e-8, path="generic").to(DEV)
        m0.set_option("small_kernel", 0)
        sd = {k: v.cpu() for k, v in m0.state_dict().items()}
        base = O.RefArch(window=120, age_coef=1e-8, has_out12="out1.weight" in sd)
        ref0 = O.RefMyCNN(base)
        ref0.load_state_dict(sd)
        ref0.eval()
        rows, aff = [Row(ref0, m0)], None
    else:
        C, k1, k2, pk, ps, W = geo
        base = O.RefArch(in_channels=C, k1=k1, k2=k2, pool_k=pk, pool_s=ps, window=W, age_coef=1e-4, has_out12=False)
        ref0 = O.make_ref(base, seed=seed)
        aff = None
        if aff_seed is not None:
            aff = centre_affine(ref0, tskd_b200.synth.make_windows(4, C, W, "normal", seed=seed), act, random_affine(aff_seed))
        rows = [Row(ref0, _gen_model(ref0, act, aff, path="generic", small=0), act, aff)]
    conv = {k: v for k, v in ref0.state_dict().items() if k.startswith("conv")}
    hbase = replace(base, has_out12=False)
    for i, Wk in enumerate(Wks):
        r = _with_conv(O.make_ref(replace(hbase, window=Wk, age_coef=1e-3 * (i + 1)), seed=seed * 10 + i), conv)
        rows.append(Row(r, _gen_model(r, act, aff, path="generic", small=0), act, aff))
    return rows


# ------------------------------------------------------------------ A with shorter heads, a twin per row
class Ward:
    def __init__(self, rows, P, S, dtype, path, seed, judge=True):
        self.rows, self.P, self.S, self.dtype, self.path = rows, P, S, dtype, path
        self.C, self.W = rows[0].model.arch.in_channels, rows[0].W
        self.A = tskd_b200.SlidingScorer(rows[0].model, P, S, dtype, path=path)
        assert self.A.path == path
        self.A.set_heads([r.model for r in rows[1:]], shorter_windows=True)
        assert self.A.head_windows == tuple(r.W for r in rows)
        # no twin can exist for a window shorter than the stride: that row is judged against float64 only
        self.twins = [tskd_b200.SlidingScorer(r.model, P, S, dtype, path=path) if r.W >= S else None for r in rows]
        self.age = tskd_b200.synth.make_ages(P, seed=seed)
        self.stream = torch.empty(P, self.C, 0)              # fp32 host copy of every stream (no lifecycle calls)
        self.judge, self.pairs, self.n = judge, [], 0

    def push(self, seg):
        self.n += 1
        n = self.n
        seg_d, age_d = seg.to(DEV), self.age.to(DEV)
        out = self.A.push(seg_d, age_d, heads=True)
        tw = [t.push(seg_d, age_d) if t is not None else None for t in self.twins]
        if self.judge:
            self.stream = torch.cat([self.stream, seg.float()], dim=2)
            complete = [n * self.S >= r.W for r in self.rows]
            assert (out is not None) == any(complete), n
            if out is not None:
                assert self.A.window_index == n - -(-self.W // self.S)
        if out is None:
            assert all(t is None for t in tw)
            return None
        assert out.shape == (len(self.rows), self.P)
        for i, t in enumerate(tw):
            if self.twins[i] is None:
                continue
            if t is None:
                assert torch.isnan(out[i]).all(), (n, i)
            else:
                assert _same(out[i], t), (n, i)
        if self.judge:
            self._judge(out, n)
        return out

    def _judge(self, out, n):
        for i, r in enumerate(self.rows):
            if n * self.S < r.W:
                assert torch.isnan(out[i]).all(), (n, i)
                continue
            win = self.stream[:, :, n * self.S - r.W:n * self.S]
            t = infer_reference(r.ref, win, self.age, act=r.act, affine=r.aff)
            t32 = infer_reference(r.ref, win, self.age, dtype=torch.float32, act=r.act, affine=r.aff)
            self.pairs.append((f"z{i}[W={r.W}, push {n}]", out[i].clone(), t["z"], t32["z"], BETA))
            if self.path == "generic":
                assert _same(out[i], r.model.predict(win.to(self.dtype).to(DEV), self.age.to(DEV))), (n, i)


def _run(w, pushes, seed, poison=True):
    emitted = 0
    for t in range(pushes):
        seg = _seg(w.P, w.C, w.S, w.dtype, seed * 1000 + t)
        if poison and t % 3 == 1:
            _poison(seg, t)
        emitted += w.push(seg) is not None
    assert emitted > 0
    _check(w.pairs)


# ------------------------------------------------------------------ tensor-core path
TC_CASES = {
    #                       kind, C, W, head windows, S, dtype, P, pushes
    "m5-c3-bf16-mixed-p130": ("mycnn5", 3, 7504, (3008, 1504, 752, 7504), 752, BF, 130, 12),
    "m5-c3-bf16-mixed-p1": ("mycnn5", 3, 7504, (3008, 1504, 752, 7504), 752, BF, 1, 11),
    "m5-c3-bf16-mixed-p257": ("mycnn5", 3, 7504, (3008, 1504, 752, 7504), 752, BF, 257, 11),
    "m3-c1-f32-w7502": ("mycnn3", 1, 7502, (3002, 1502), 752, F32, 130, 12),           # phi = 2
    "m5-c3-bf16-w7501-phi3": ("mycnn5", 3, 7501, (3001,), 752, BF, 130, 12),            # phi = 3
    "m5-c2-bf16-short-500": ("mycnn5", 2, 7504, (500, 3008), 752, BF, 130, 11),         # W_k < S: no twin
}


@pytest.mark.parametrize("name", list(TC_CASES))
def test_horizons_tensorcore(name):
    kind, C, W, Wks, S, dtype, P, pushes = TC_CASES[name]
    i = list(TC_CASES).index(name)
    rows = _tc_family(kind, C, W, Wks, seed=100 + i)
    _run(Ward(rows, P, S, dtype, "tensorcore", seed=110 + i), pushes, seed=120 + i)


# ------------------------------------------------------------------ generic path
GEN_CASES = {
    #                      geo (None: golden), head windows, act, affine seed, S, dtype, P, pushes
    "golden-w120-s12-k64": (None, (64,), "tanh", None, 12, F32, 130, 12),                # F = 4, L_k = 11
    "c10-relu-negaff-s100": ((10, 10, 5, 3, 2, 600), (300, 200), "relu", 1, 100, F32, 64, 8),
    "c16-p44-s160-w1470": ((16, 3, 8, 4, 4, 1470), (670,), "tanh", None, 160, BF, 64, 11),   # F = 16
}


@pytest.mark.parametrize("name", list(GEN_CASES))
def test_horizons_generic(name):
    geo, Wks, act, aff, S, dtype, P, pushes = GEN_CASES[name]
    i = list(GEN_CASES).index(name)
    rows = _gen_family(geo, Wks, seed=200 + i, act=act, aff_seed=aff)
    _run(Ward(rows, P, S, dtype, "generic", seed=210 + i), pushes, seed=220 + i)


# ------------------------------------------------------------------ early emission
def test_early_emission_before_the_scorers_window():
    """pushes before n S >= W return the rows whose windows are complete, row 0 all NaN, window_index negative"""
    rows = _tc_family("mycnn5", 3, 7504, (1504, 752), seed=300)
    w = Ward(rows, 64, 752, BF, "tensorcore", seed=301)
    for t in range(11):
        out = w.push(_seg(64, 3, 752, BF, 3000 + t))
        n = t + 1
        if n * 752 < 7504:
            assert out is not None and torch.isnan(out[0]).all() and w.A.window_index < 0
            assert not torch.isnan(out[2]).any() and bool(torch.isnan(out[1]).all()) == (n < 2)
    _check(w.pairs)


# ------------------------------------------------------------------ lifecycle
@pytest.mark.parametrize("path", ["tensorcore", "generic"])
def test_horizons_through_the_lifecycle(path):
    """admit (H >= W_k but < W, and H < W_k), discharge and re-admit, export / restore into another scorer with the
    same heads, reset: every row against a twin put through the same calls (a twin admits the last min(H, W_k) samples,
    all its window can hold; H - W_k is a multiple of 8 samples, two features)"""
    if path == "tensorcore":
        rows = _tc_family("mycnn5", 3, 7504, (3008, 1504), seed=400)
        P, S, dtype, H_long, H_short = 130, 752, BF, 3008 + 800, 1000
    else:
        rows = _gen_family(None, (64,), seed=401)
        P, S, dtype, H_long, H_short = 130, 12, F32, 64 + 16, 40
    w = Ward(rows, P, S, dtype, path, seed=402, judge=False)
    C, W = w.C, w.W
    seed = 4000

    def each(fn):
        fn(w.A, W)
        for t, r in zip(w.twins, w.rows):
            fn(t, r.W)

    def admit(idx, H, s):
        hist = _seg(len(idx), C, H, dtype, s).to(DEV)
        each(lambda sc, Wr: sc.admit(idx, hist[:, :, -min(H, Wr):]))

    def pushes(k):
        nonlocal seed
        outs = []
        for _ in range(k):
            seed += 1
            outs.append(w.push(_seg(P, C, S, dtype, seed)))
        return outs

    pushes(2)
    admit([0, 5], H_long, 1)                                   # H >= W_1 > W_2, H < W
    admit([7, 129], H_short, 2)                                # W_2 > H ... < W_1
    out = pushes(1)[0]
    assert torch.isnan(out[0, [0, 5]]).all() and not torch.isnan(out[1:, [0, 5]]).any()
    assert torch.isnan(out[:2, [7, 129]]).all()
    each(lambda sc, Wr: sc.discharge([1, 2, 64]))
    pushes(3)
    admit([1, 64], H_long, 3)                                  # re-admitted
    pushes(W // S + 1)
    # export from every scorer and restore into a scorer of another P with the same heads
    idx = [3, 5, 64, 100]
    A2 = tskd_b200.SlidingScorer(w.rows[0].model, 8, S, dtype, path=path)
    A2.set_heads([r.model for r in w.rows[1:]], shorter_windows=True)
    tw2 = [tskd_b200.SlidingScorer(r.model, 8, S, dtype, path=path) for r in w.rows]
    A2.restore([0, 2, 4, 6], w.A.export(idx))
    for t, t2 in zip(w.twins, tw2):
        t2.restore([0, 2, 4, 6], t.export(idx))
    for k in range(3):
        seg = _seg(8, C, S, dtype, 4900 + k).to(DEV)
        out = A2.push(seg, heads=True)
        for i, t2 in enumerate(tw2):
            want = t2.push(seg)
            assert want is None and torch.isnan(out[i]).all() or _same(out[i], want), (k, i)
    each(lambda sc, Wr: sc.reset())
    assert w.A.head_windows == tuple(r.W for r in w.rows)
    pushes(W // S + 2)


# ------------------------------------------------------------------ heads at W only: today's launches, today's bits
def _kernels(fn):
    """the kernels fn launches, by name and count (the first profiler session of a process may miss its first kernel:
    the test warms the profiler up before it compares)"""
    from collections import Counter
    from torch.profiler import ProfilerActivity, profile
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    return Counter(e.name for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA)


@pytest.mark.parametrize("path", ["tensorcore", "generic"])
def test_heads_at_W_only_run_todays_launches(path):
    if path == "tensorcore":
        rows = _tc_family("mycnn5", 3, 7504, (7504, 7504, 7504), seed=500)
        P, S, dtype = 130, 752, BF
    else:
        rows = _gen_family(None, (120, 120), seed=501)
        P, S, dtype = 130, 12, F32
    heads = [r.model for r in rows[1:]]
    old = tskd_b200.SlidingScorer(rows[0].model, P, S, dtype, path=path)
    new = tskd_b200.SlidingScorer(rows[0].model, P, S, dtype, path=path)
    old.set_heads(heads)
    new.set_heads(heads, shorter_windows=True)
    age = tskd_b200.synth.make_ages(P, seed=502).to(DEV)
    for t in range(rows[0].W // S + 3):
        seg = _seg(P, rows[0].model.arch.in_channels, S, dtype, 5000 + t).to(DEV)
        if t == rows[0].W // S + 2:
            _kernels(lambda: torch.ones(1, device=DEV).add_(1))                # profiler warm-up
            outs = {}
            k_old = _kernels(lambda: outs.__setitem__("old", old.push(seg, age, heads=True)))
            k_new = _kernels(lambda: outs.__setitem__("new", new.push(seg, age, heads=True)))
            assert k_old == k_new and sum(k_old.values()) > 0, (k_old, k_new)
            a, b = outs["old"], outs["new"]
        else:
            a, b = old.push(seg, age, heads=True), new.push(seg, age, heads=True)
        assert (a is None) == (b is None) and (a is None or torch.equal(a, b)), t


# ------------------------------------------------------------------ errors change nothing
def test_set_heads_ex_errors_change_nothing():
    rows = _tc_family("mycnn5", 3, 7504, (3008, 1504), seed=600)
    P, S = 40, 752
    w = Ward(rows, P, S, BF, "tensorcore", seed=601, judge=False)
    for t in range(4):
        w.push(_seg(P, 3, S, BF, 6000 + t))
    lib = w.A._lib
    conv = {k: v for k, v in rows[0].ref.state_dict().items() if k.startswith("conv")}
    base = rows[0].ref.arch

    def handle_of(Wk, conv_sd=conv, seed=610):
        m = _tc_model(_with_conv(O.make_ref(replace(base, window=Wk), seed=seed), conv_sd))
        return m, m._ensure_handle()[1].value

    def rc(handles, flags=capi.SLIDE_HEADS_SHORTER_WINDOWS):
        arr = (ctypes.c_void_p * max(len(handles), 1))(*handles)
        r = lib.b2cnn_slide_set_heads_ex(w.A._s, arr, len(handles), flags, torch.cuda.current_stream().cuda_stream)
        torch.cuda.synchronize()
        return r

    good = [r.model._ensure_handle()[1].value for r in rows[1:]]
    longer, h_longer = handle_of(7508)                                   # a longer window
    offl, h_offl = handle_of(3006)                                       # W - W_k = 4498: not a multiple of 4
    conv_b = dict(conv)
    conv_b["conv2.bias"] = conv_b["conv2.bias"] + 0.01
    other, h_other = handle_of(3008, conv_b)                             # other conv weights
    assert rc([good[0], h_longer]) == capi.EARCH
    assert rc([h_offl]) == capi.EARCH
    assert rc([good[0], h_other]) == capi.ESTATE
    assert rc(good, flags=2) == capi.EINVAL and rc(good, flags=3) == capi.EINVAL
    assert lib.b2cnn_slide_set_heads(w.A._s, (ctypes.c_void_p * 1)(good[0]), 1,
                                     torch.cuda.current_stream().cuda_stream) == capi.EARCH   # flags 0: windows must match
    # lstm_input == L_out(window) holds for every handle b2cnn_create accepts: the Python check of a model whose l_out
    # does not fit its window is in tests/test_slide_horizons_host.py
    for bad in ([rows[1].model, longer], [offl]):
        with pytest.raises(ValueError):
            w.A.set_heads(bad, shorter_windows=True)
    with pytest.raises(RuntimeError, match="b2cnn error 5"):
        w.A.set_heads([rows[1].model, other], shorter_windows=True)
    with pytest.raises(ValueError, match="differs"):
        w.A.set_heads([rows[1].model])                                   # shorter_windows=False: today's message
    assert lib.b2cnn_slide_n_heads(w.A._s) == 2 and w.A.heads == tuple(r.model for r in rows[1:])
    assert w.A.head_windows == (7504, 3008, 1504)
    for t in range(8):                                                   # every later output unchanged
        w.push(_seg(P, 3, S, BF, 6100 + t))
