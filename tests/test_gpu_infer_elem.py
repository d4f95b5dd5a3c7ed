"""GPU: every inference path element by element against the float64 reference of oracle/infer_ref.py -- logits, and the
features where a path exposes them -- at the shapes and values where a scale-relative bar is blind: logits that
straddle 0, small-amplitude windows (pre-activations near tanh's zero), saturated windows, the age-scale kink, NaN ages,
NaN and inf samples, window-tile and range seams, and the full [4096, 3, 75000] batch.

Every comparison is oracle/train_ref.py::assert_close_elem: |got - truth| <= 8 |ref32 - truth| + beta max|truth| per
element, where ref32 is the same reference in float32 (the existing oracle, bit for bit).  beta is 2^-20 unless a
named grant below says otherwise, with its reason.  Every test asserts which path ran (last_path, gpu_launches).

Finite samples stay small (|x| <= 1e4 here): far beyond that a float32 conv sum may overflow where float64 does not,
and the float32 reference then legitimately disagrees with the truth."""
import os
from collections import namedtuple
from dataclasses import replace

import numpy as np
import pytest
import torch

import tskd_b200
from oracle import mycnn_torch as O
from oracle.infer_ref import TC_FEATURES_BETA, infer_reference
from oracle.train_ref import BETA, assert_close_elem, check_elems

pytestmark = pytest.mark.gpu
DEV = "cuda:0"

# ------------------------------------------------------------------ cases
# kind, C, W, B, dtype, dist: the windows; amp scales them; zero: shift out.bias so the logits straddle 0; age: "rand",
# "kink" (relu(age * coef + 1) at and beyond its zero), "nan" (one NaN age), "scalar" (one age for the batch);
# bad: NaN / +-inf samples in a few windows; padded: rows from empty_windows
Case = namedtuple("Case", "kind C W B dtype dist seed amp zero age bad padded", defaults=(1.0, False, "rand", False, False))
BF, F32 = torch.bfloat16, torch.float32
CASES = {
    "m5-c3-w7504-b129": Case("mycnn5", 3, 7504, 129, BF, "normal", 1),
    "m5-c3-w7500-b128-staged": Case("mycnn5", 3, 7500, 128, BF, "normal", 2, zero=True),
    "m5-c3-w7500-b127-padded": Case("mycnn5", 3, 7500, 127, BF, "normal", 3, padded=True, age="kink"),
    "m5-c2-w1533-b257-odd": Case("mycnn5", 2, 1533, 257, BF, "normal", 4, bad=True),
    "m5-c1-w1528-b1": Case("mycnn5", 1, 1528, 1, BF, "normal", 5, age="scalar"),
    "m5-c3-w75000-b9": Case("mycnn5", 3, 75000, 9, BF, "normal", 6, zero=True),
    "m5-c3-w7504-b128-small-amp": Case("mycnn5", 3, 7504, 128, BF, "normal", 7, amp=1e-3),
    "m5-c3-w7504-b130-physio": Case("mycnn5", 3, 7504, 130, BF, "physio", 8, age="nan"),
    "m3-c3-w7504-b129": Case("mycnn3", 3, 7504, 129, BF, "normal", 9, zero=True, age="kink"),
    "m3-c3-w7502-b64-physio": Case("mycnn3", 3, 7502, 64, BF, "physio", 10, bad=True),
    "m3-c2-w1533-b257-small-amp": Case("mycnn3", 2, 1533, 257, BF, "normal", 11, amp=1e-3),
    "m5-c4-w3000-b130": Case("mycnn5", 4, 3000, 130, BF, "normal", 12),
    # fp32 windows
    "m5-c3-w7504-b129-f32": Case("mycnn5", 3, 7504, 129, F32, "normal", 21, zero=True),
    "m5-c3-w7500-b128-f32": Case("mycnn5", 3, 7500, 128, F32, "normal", 22, bad=True),
    "m5-c3-w7502-b127-f32-padded": Case("mycnn5", 3, 7502, 127, F32, "normal", 23, padded=True, age="nan"),
    "m5-c2-w1528-b257-f32-small-amp": Case("mycnn5", 2, 1528, 257, F32, "normal", 24, amp=1e-3, age="kink"),
    "m3-c3-w7504-b130-f32-physio": Case("mycnn3", 3, 7504, 130, F32, "physio", 25, age="scalar"),
    "m3-c1-w1528-b1-f32": Case("mycnn3", 1, 1528, 1, F32, "normal", 26, zero=True),
    "m5-c3-w75000-b9-f32": Case("mycnn5", 3, 75000, 9, F32, "normal", 6, zero=True),   # the bf16 case's weights
}


def _oarch(kind, C, W):
    return O.stretched(O.ARCHS[kind], C, W)


def _model(ref, path="auto", tc_splits=3):
    oarch = ref.arch
    arch = replace(tskd_b200.ARCH_PRESETS[oarch_kind(oarch)].with_shape(oarch.in_channels, oarch.window),
                   age_coef=oarch.age_coef)
    m = tskd_b200.B200MyCNN(arch, has_out12=oarch.has_out12, path=path, tc_splits=tc_splits).to(DEV)
    m.load_state_dict(ref.state_dict())
    return m


def oarch_kind(oarch):
    return "mycnn5" if oarch.k1 == 10 else "mycnn3"


def _ages(c, B, g):
    coef = O.ARCHS[c.kind].age_coef                       # 1e-8 for MyCNN5, 1e-4 for MyCNN2/3/4
    if c.age == "scalar":
        return torch.tensor([57.0])
    age = torch.rand(B, generator=g) * 65 + 15
    if c.age == "kink":                                   # age * coef + 1 == 0 (in float64), then negative
        age[::3] = -1.0 / coef
        age[1::3] = -3.0 / coef
    elif c.age == "nan":
        age[B // 2] = float("nan")
    return age


def _inject(x):
    """NaN at the first / last sample, +inf mid-window, -inf in the last window"""
    B, C, W = x.shape
    x[0, 0, 0] = float("nan")
    x[min(2, B - 1), C - 1, W - 1] = float("nan")
    x[min(3, B - 1), 0, W // 2] = float("inf")
    x[B - 1, C - 1, W // 3] = float("-inf")


def _windows(c, mix=False):
    """mix: every other window "normal" (saturated physio windows alone give nearly equal logits, which centring
    would shrink to the rounding error of the uncentred ones)"""
    g = torch.Generator().manual_seed(c.seed)
    x = tskd_b200.synth.make_windows(c.B, c.C, c.W, c.dist, seed=c.seed) * c.amp
    if mix:
        x[1::2] = tskd_b200.synth.make_windows(c.B // 2, c.C, c.W, "normal", seed=c.seed + 1)
    if c.bad:
        _inject(x)
    return x.to(c.dtype), _ages(c, c.B, g)


def _center(ref, x):
    """shift out.bias by the median float64 logit (at age scale 1) so that the logits straddle 0"""
    z = infer_reference(ref, x, 0.0)["z"]
    with torch.no_grad():
        ref.out.bias -= float(np.nanmedian(z.numpy()))


def _build_case(name):
    """(ref, x, age, truth, ref32) of a case; truth and ref32 for both batch modes"""
    c = CASES[name]
    ref = O.make_ref(_oarch(c.kind, c.C, c.W), seed=c.seed)
    x, age = _windows(c)
    if c.zero:
        _center(ref, x[:16])
    truth = {m: infer_reference(ref, x, age, m) for m in ("independent", "sequence")}
    ref32 = {m: infer_reference(ref, x, age, m, dtype=torch.float32) for m in ("independent", "sequence")}
    if c.zero and c.B > 1:
        zt = truth["independent"]["z"]
        assert (zt > 0).any() and (zt < 0).any(), name
    return ref, x, age, truth, ref32


@pytest.fixture(scope="module")
def case_data():
    """the float64 truth of a case is computed once and shared by every path of the case (the tests of one case run
    one after another, so one case's windows are kept at a time)"""
    cache = {}

    def get(name):
        if name not in cache:
            cache.clear()
            cache[name] = _build_case(name)
        return cache[name]
    yield get
    cache.clear()


def _to_dev(c, m, x):
    if not c.padded:
        return x.to(DEV)
    xp = m.empty_windows(x.shape[0], dtype=x.dtype)
    xp.copy_(x)
    assert not xp.is_contiguous()
    return xp


def _check(pairs):
    """(name, got, truth, ref32, beta) per element; all failures reported together; prints each comparison's smallest
    passing beta and how many elements it judged (oracle/train_ref.py::check_elems)"""
    check_elems(pairs, os.environ.get("PYTEST_CURRENT_TEST", "").split(" ")[0])


# ------------------------------------------------------------------ per-path grants (beta per path and output)
# Tensor-core logits: the features' own error (TC_FEATURES_BETA, oracle/infer_ref.py) summed by the projection over up
# to 18745 features.  Measured worst on an H100: 4.5e-6 at W = 75000 with centred logits (max|z| 1.6e-2), 2.8e-6
# through the CUDA-core projection (tc_fused=0) on the same windows, so the wgmma projection is not the cause.
BETA_TC_LOGITS = 6e-6
# fp32 windows through the streaming kernel: exact fp32 conv1, but the same MUFU tanh epilogue and wgmma projection as
# the bf16 kernel.  Measured 6.0e-6 on the W = 75000 centred case where the exact generic kernel needs 5.4e-7: the
# epilogue's error, summed over 18745 features, not the bf16 conv1, is what the tensor-core logits carry.
BETA_STREAM_LOGITS = 8e-6
# Exact float32 kernels in another summation order than torch's.  Saturated physio windows: conv1 sums terms of ~20
# into partial sums of ~1e2, whose float32 rounding reaches ~1e-6 of the feature scale where the float32 reference
# happens to be exact (measured 1.2e-6).  The [P, C, 120] batch kernel: centred logits, out.bias cancels an LSTM
# output of ~0.1 down to ~5e-3, leaving its float32 rounding at ~1e-6 of the largest (measured 1.2e-6).
BETA_GENERIC_FEATURES = 2e-6
BETA_BATCH_LOGITS = 2e-6


def _paths(c):
    """the (label, path, options, expected last_path) a case goes through"""
    out = []
    if c.dtype == BF and c.C <= 3:
        out.append(("tc-fused", "tensorcore", {}, "tensorcore"))
        if c.kind == "mycnn5":
            out.append(("tc-unfused", "tensorcore", {"tc_fused": 0}, "tensorcore"))
    if c.dtype == F32 and c.C <= 3 and (c.W % 4 == 0 or c.padded):
        out.append(("stream", "tensorcore", {}, "stream"))
    out.append(("generic", "generic", {}, "generic"))
    return out


PATH_CASES = [(n, p[0]) for n, c in CASES.items() for p in _paths(c)]


@pytest.mark.parametrize("name,label", PATH_CASES, ids=[f"{n}-{p}" for n, p in PATH_CASES])
def test_logits_independent(case_data, name, label):
    c = CASES[name]
    ref, x, age, truth, ref32 = case_data(name)
    _, path, opts, want_path = next(p for p in _paths(c) if p[0] == label)
    m = _model(ref, path)
    for k, v in opts.items():
        m.set_option(k, v)
    xd = _to_dev(c, m, x)
    got = m.predict(xd, age.to(DEV) if c.age != "scalar" else float(age))
    assert m.last_path == want_path, (m.last_path, want_path)
    beta = {"tc-fused": BETA_TC_LOGITS, "tc-unfused": BETA_TC_LOGITS, "stream": BETA_STREAM_LOGITS}.get(label, BETA)
    _check([("z", got, truth["independent"]["z"], ref32["independent"]["z"], beta)])


FEATURE_CASES = [(n, p) for n, c in CASES.items() for p in (["tensorcore"] if c.dtype == BF and c.kind == "mycnn5" else [])
                 + ["generic"]]


@pytest.mark.parametrize("name,path", FEATURE_CASES, ids=[f"{n}-{p}" for n, p in FEATURE_CASES])
def test_features(case_data, name, path):
    ref, x, _, truth, ref32 = case_data(name)
    m = _model(ref, path)
    got = m.features(x.to(DEV))
    assert m.last_path == path
    beta = TC_FEATURES_BETA if path == "tensorcore" else BETA_GENERIC_FEATURES
    _check([("features", got, truth["independent"]["features"], ref32["independent"]["features"], beta)])


# (a NaN window would turn every later logit of the scan NaN: these cases have none)
SEQ_CASES = [("m5-c3-w7504-b129", "tensorcore", "tensorcore"), ("m3-c3-w7504-b129", "tensorcore", "tensorcore"),
             ("m5-c2-w1528-b257-f32-small-amp", "tensorcore", "stream"), ("m5-c3-w7504-b129-f32", "tensorcore", "stream"),
             ("m3-c2-w1533-b257-small-amp", "generic", "generic"), ("m5-c3-w7500-b127-padded", "generic", "generic")]


@pytest.mark.parametrize("name,path,want_path", SEQ_CASES, ids=[f"{n}-{p}" for n, p, _ in SEQ_CASES])
def test_logits_sequence(case_data, name, path, want_path):
    """model(x, age): the LSTM scans the batch axis, on the fused, stream and generic front ends"""
    c = CASES[name]
    ref, x, age, truth, ref32 = case_data(name)
    m = _model(ref, path)
    got = m(_to_dev(c, m, x), age.to(DEV))
    assert m.last_path == want_path
    beta = {"tensorcore": BETA_TC_LOGITS, "stream": BETA_STREAM_LOGITS}.get(want_path, BETA)
    _check([("z", got, truth["sequence"]["z"], ref32["sequence"]["z"], beta)])


@pytest.mark.parametrize("kind,dtype", [("mycnn5", BF), ("mycnn3", F32)])
def test_sequence_over_thousands_of_steps(kind, dtype):
    """B = 4096 short windows in sequence mode: head_sequence_kernel carries the LSTM state over 4096 steps"""
    B, W = 4096, 1528
    ref = O.make_ref(_oarch(kind, 3, W), seed=31)
    x = tskd_b200.synth.make_windows(B, 3, W, "normal", seed=31, dtype=dtype)
    age = tskd_b200.synth.make_ages(B, seed=31)
    truth, ref32 = infer_reference(ref, x, age, "sequence"), infer_reference(ref, x, age, "sequence", torch.float32)
    m = _model(ref, "tensorcore")
    got = m(x.to(DEV), age.to(DEV))
    assert m.last_path == ("tensorcore" if dtype == BF else "stream")
    _check([("z", got, truth["z"], ref32["z"], BETA_TC_LOGITS if dtype == BF else BETA_STREAM_LOGITS)])


# ------------------------------------------------------------------ single-launch kernels
@pytest.mark.parametrize("kind,C,W,B,dtype,dist,age_kind", [
    ("mycnn5", 10, 120, 1, F32, "normal", "rand"),        # the production call [1, 10, 120]
    ("mycnn5", 10, 120, 7, BF, "physio", "kink"),
    ("mycnn3", 3, 1500, 40, BF, "physio", "nan"),
    ("mycnn5", 3, 2048, 256, F32, "normal", "scalar"),    # C * W == 6144 <= 8192, B == 256: the largest small call
    ("mycnn3", 1, 1533, 3, F32, "normal", "rand"),
])
def test_small_single_launch(kind, C, W, B, dtype, dist, age_kind):
    c = Case(kind, C, W, B, dtype, dist, 41 + B, age=age_kind, bad=B >= 4, zero=B >= 7)
    ref = O.make_ref(_oarch(kind, C, W), seed=c.seed)
    x, age = _windows(c, mix=c.zero)
    m = _model(ref)
    if c.zero:
        _center(ref, x)
        m.load_state_dict(ref.state_dict())
    truth, ref32 = infer_reference(ref, x, age), infer_reference(ref, x, age, dtype=torch.float32)
    a = age.to(DEV) if age_kind != "scalar" else float(age)
    got = m.predict(x.to(DEV), a)
    assert m.gpu_launches == 1 and m.last_path == "generic"
    prob = m.predict(x.to(DEV), a, return_prob=True)
    assert m.gpu_launches == 1
    _check([("z", got, truth["z"], ref32["z"], BETA),
            ("prob", prob, torch.sigmoid(truth["z"]), torch.sigmoid(ref32["z"]), BETA)])


@pytest.mark.parametrize("n,P,dtype,age_kind", [(5, 1000, F32, "rand"), (5, 37, BF, "kink"), (4, 300, F32, "nan"),
                                                (3, 600, F32, "scalar"), (2, 8, F32, "rand")])
def test_batch_kernel_production_shape(n, P, dtype, age_kind):
    """[P, 10 or 7, 120]: all patients of a trigger in one launch, one warp per window"""
    kind = "mycnn5" if n == 5 else ("mycnn4" if n == 4 else "mycnn3")
    C = 7 if n in (2, 3) else 10
    c = Case(kind, C, 120, P, dtype, "physio", 50 + n, age=age_kind, bad=True, zero=True)
    ref = O.make_ref(_oarch(kind, C, 120), seed=c.seed)
    x, age = _windows(c, mix=True)
    _center(ref, x)
    m = _model(ref)
    truth, ref32 = infer_reference(ref, x, age), infer_reference(ref, x, age, dtype=torch.float32)
    a = age.to(DEV) if age_kind != "scalar" else float(age)
    got = m.predict(x.to(DEV), a)
    assert m.gpu_launches == 1 and m.last_path == "generic"
    prob = m.predict(x.to(DEV), a, return_prob=True)
    _check([("z", got, truth["z"], ref32["z"], BETA_BATCH_LOGITS),
            ("prob", prob, torch.sigmoid(truth["z"]), torch.sigmoid(ref32["z"]), BETA)])


# ------------------------------------------------------------------ seams: window tiles, position ranges, persistent CTAs
@pytest.mark.parametrize("tiles", [4, 5])
@pytest.mark.parametrize("kind,W,B,dtype", [("mycnn5", 7504, 257, BF), ("mycnn3", 7500, 129, BF),
                                            ("mycnn5", 7504, 130, F32)])
def test_range_seams(monkeypatch, tiles, kind, W, B, dtype):
    """B2CNN_TC_TILES = 4 / 5: a 7504-sample window in about 90 position ranges, so every range-start halo is compared
    position by position (through the features of the projection)"""
    monkeypatch.setenv("B2CNN_TC_TILES", str(tiles))       # read by tc_prepare when the weights are set
    ref = O.make_ref(_oarch(kind, 3, W), seed=60 + tiles)
    x = tskd_b200.synth.make_windows(B, 3, W, "normal", seed=60 + tiles, dtype=dtype)
    age = tskd_b200.synth.make_ages(B, seed=60 + tiles)
    truth = infer_reference(ref, x, age)
    ref32 = infer_reference(ref, x, age, dtype=torch.float32)
    m = _model(ref, "tensorcore")
    got = m.predict(x.to(DEV), age.to(DEV))
    assert m.last_path == ("tensorcore" if dtype == BF else "stream")
    pairs = [("z", got, truth["z"], ref32["z"], BETA_TC_LOGITS if dtype == BF else BETA_STREAM_LOGITS)]
    if kind == "mycnn5" and dtype == BF:
        f = m.features(x.to(DEV))
        assert m.last_path == "tensorcore"
        pairs.append(("features", f, truth["features"], ref32["features"], TC_FEATURES_BETA))
        m.set_option("tc_fused", 0)
        pairs.append(("z unfused", m.predict(x.to(DEV), age.to(DEV)), truth["z"], ref32["z"], BETA_TC_LOGITS))
        assert m.last_path == "tensorcore"
    _check(pairs)


def test_persistent_ctas_walk_several_items():
    """B = 2100 at W = 7504: more (window tile, range) items than resident CTAs"""
    B, W = 2100, 7504
    ref = O.make_ref(_oarch("mycnn5", 3, W), seed=71)
    x = tskd_b200.synth.make_windows(B, 3, W, "physio", seed=71, dtype=BF)
    age = tskd_b200.synth.make_ages(B, seed=71)
    truth, ref32 = infer_reference(ref, x, age), infer_reference(ref, x, age, dtype=torch.float32)
    m = _model(ref, "tensorcore")
    got = m.predict(x.to(DEV), age.to(DEV))
    assert m.last_path == "tensorcore"
    _check([("z", got, truth["z"], ref32["z"], BETA_TC_LOGITS)])


def test_full_size_first_and_last_window_tiles():
    """[4096, 3, 75000] bf16 on the fused path; the first and the last window tile (b < 128, b >= 3968) judged"""
    B, W = 4096, 75000
    ref = O.make_ref(_oarch("mycnn5", 3, W), seed=81)
    x = tskd_b200.synth.make_windows(B, 3, W, "normal", seed=81, dtype=BF, device=DEV)
    age = tskd_b200.synth.make_ages(B, seed=81, device=DEV)
    m = _model(ref)
    got = m.predict(x, age)
    assert m.last_path == "tensorcore"
    sel = torch.cat([torch.arange(0, 128), torch.arange(B - 128, B)]).to(DEV)
    xs, ags = x[sel].cpu(), age[sel].cpu()
    del x
    truth, ref32 = infer_reference(ref, xs, ags), infer_reference(ref, xs, ags, dtype=torch.float32)
    _check([("z", got[sel], truth["z"], ref32["z"], BETA_TC_LOGITS)])


# ------------------------------------------------------------------ the two-piece weights must be visible
def test_two_piece_weights_fail_the_tensor_core_logit_bound():
    """tc_splits=2 keeps 16 mantissa bits of every conv1 weight in the fused kernel: its logits must miss the bound the
    default tensor-core logits meet (the same windows pass with tc_splits=3).  features() runs the unfused front end,
    which always uses the three pieces; tests/test_oracle_infer.py shows the feature bound rejects two-piece weights."""
    ref = O.make_ref(_oarch("mycnn5", 3, 7504), seed=0)
    x = tskd_b200.synth.make_windows(64, 3, 7504, "physio", seed=3, dtype=BF)
    truth, ref32 = infer_reference(ref, x, 65.0)["z"], infer_reference(ref, x, 65.0, dtype=torch.float32)["z"]
    m3, m2 = _model(ref, "tensorcore"), _model(ref, "tensorcore", tc_splits=2)
    z3, z2 = m3.predict(x.to(DEV), 65.0), m2.predict(x.to(DEV), 65.0)
    assert m3.last_path == m2.last_path == "tensorcore"
    assert_close_elem("z", z3, truth, ref32, beta=BETA_TC_LOGITS)
    with pytest.raises(AssertionError, match="elements off"):
        assert_close_elem("z", z2, truth, ref32, beta=BETA_TC_LOGITS)


# ------------------------------------------------------------------ the sliding scorer
BETA_SLIDE_LOGITS = BETA
BETA_SLIDE_FEATURES = TC_FEATURES_BETA


@pytest.mark.parametrize("kind,dtype,W,S,bad", [
    ("mycnn5", BF, 7504, 1876, False), ("mycnn5", F32, 7500, 740, False), ("mycnn3", BF, 7502, 1876, True),
    ("mycnn3", F32, 7504, 1876, False), ("mycnn5", BF, 200, 8, False), ("mycnn5", F32, 200, 8, True),
    ("mycnn3", BF, 200, 100, False),
])
def test_sliding_scorer(kind, dtype, W, S, bad):
    """logits and features() of every emitted window against the float64 truth of the explicit window"""
    P = 130
    ref = O.make_ref(_oarch(kind, 3, W), seed=91)
    n0 = -(-W // S)
    n_push = n0 + 2
    stream = tskd_b200.synth.make_windows(P, 3, n_push * S, "normal", seed=91, dtype=dtype)
    if bad:                                                 # a seam sample, a mid-segment sample, a tail sample
        stream[1, 0, S + S // 2] = float("nan")
        stream[2, 1, 2 * S + 3] = float("inf")
        stream[3, 2, n_push * S - 2] = float("-inf")
    age = tskd_b200.synth.make_ages(P, seed=91)
    m = _model(ref)
    sc = tskd_b200.SlidingScorer(m, P, S, dtype)
    sd = stream.to(DEV)
    pairs, emitted = [], 0
    for n in range(1, n_push + 1):
        got = sc.push(sd[:, :, (n - 1) * S:n * S], age.to(DEV))
        if n * S < W:
            assert got is None
            continue
        win = stream[:, :, n * S - W:n * S]
        truth, ref32 = infer_reference(ref, win, age), infer_reference(ref, win, age, dtype=torch.float32)
        pairs.append((f"z[{n}]", got.clone(), truth["z"], ref32["z"], BETA_SLIDE_LOGITS))
        pairs.append((f"features[{n}]", sc.features(), truth["features"], ref32["features"], BETA_SLIDE_FEATURES))
        emitted += 1
    assert emitted == n_push - n0 + 1
    sc.close()
    _check(pairs)
