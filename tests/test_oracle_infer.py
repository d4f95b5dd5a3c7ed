"""CPU: the inference reference (oracle/infer_ref.py) -- in float64 against the independent plain-C float64 restatement
(oracle/mycnn_ref.c) for every activation and against torch.nn's Conv1d -> BatchNorm1d(eval) -> act -> MaxPool1d for
the folded affine, in float32 against the existing oracle bit for bit -- and negative controls showing that the
per-element comparator the GPU inference tests use (oracle/train_ref.py::assert_close_elem) sees conv1 weights that
lost their third bf16 piece, and features that pool before a negative affine scale."""
import copy
from dataclasses import replace

import numpy as np
import pytest
import torch

import tskd_b200
from oracle import mycnn_c
from oracle import mycnn_torch as O
from oracle.infer_ref import ACTS, TC_FEATURES_BETA, centre_affine, infer_reference, random_affine
from oracle.train_ref import BETA, assert_close_elem

# a conv/pool geometry off the reference's two: overlapping pools (4 > 3) with an uncovered conv1 tail
OFF_REF = O.RefArch(in_channels=4, k1=6, k2=4, pool_k=4, pool_s=3, window=700, age_coef=1e-4, has_out12=False)
C_ACT = {"tanh": 0, "relu": 1, "identity": 2}                     # b2cnn_config.act, oracle/mycnn_ref.c


def _case(kind, C, W, B, seed, bad=True):
    oarch = O.stretched(O.ARCHS[kind], C, W)
    ref = O.make_ref(oarch, seed=seed)
    x = tskd_b200.synth.make_windows(B, C, W, "normal", seed=seed)
    if bad:
        x[1, 0, W // 3] = float("nan")
        x[2, C - 1, W // 2] = float("inf")
        x[3, 0, 5] = float("-inf")
    ages = tskd_b200.synth.make_ages(B, seed=seed)
    return ref, x, ages


def _close_1e12(name, got, want):
    got, want = np.asarray(got, dtype=np.float64), np.asarray(want, dtype=np.float64)
    assert np.array_equal(np.isnan(got), np.isnan(want)), name
    fin = np.isfinite(want)
    assert np.array_equal(got[~fin], want[~fin], equal_nan=True), name
    scale = np.abs(want[fin]).max()
    err = np.abs(got[fin] - want[fin]).max()
    assert err <= 1e-12 * scale, (name, err, scale)


@pytest.mark.parametrize("mode", ["independent", "sequence"])
@pytest.mark.parametrize("kind,C,W", [("mycnn5", 3, 1500), ("mycnn5", 10, 120), ("mycnn3", 3, 1502), ("mycnn3", 7, 120)])
def test_float64_reference_matches_plain_c(kind, C, W, mode):
    ref, x, ages = _case(kind, C, W, 6, seed=3)
    got = infer_reference(ref, x, ages, mode)
    assert got["z"].dtype == got["features"].dtype == torch.float64
    z, f = mycnn_c.forward(ref.arch, mycnn_c.pack_blob(ref.state_dict()), x.numpy(), ages.numpy(), mode=mode,
                           precision="f64", want_features=True)
    _close_1e12("features", got["features"].numpy(), f)
    _close_1e12("z", got["z"].numpy(), z)
    assert np.isnan(z[1]) and np.isfinite(z[2]) and np.isfinite(z[3]) if mode == "independent" else np.isnan(z[1:]).all()


@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16])
@pytest.mark.parametrize("kind,C,W", [("mycnn5", 3, 1500), ("mycnn3", 3, 1502)])
def test_float32_reference_is_the_oracle(kind, C, W, dtype):
    ref, x, ages = _case(kind, C, W, 5, seed=4)
    x = x.to(dtype)
    ind = infer_reference(ref, x, ages, "independent", dtype=torch.float32)
    seq = infer_reference(ref, x, ages, "sequence", dtype=torch.float32)
    eq = dict(rtol=0, atol=0, equal_nan=True)
    torch.testing.assert_close(ind["z"], O.ref_independent(ref, x, ages), **eq)
    torch.testing.assert_close(seq["z"], O.ref_sequence(ref, x, ages), **eq)
    torch.testing.assert_close(ind["features"], O.ref_features(ref, x), **eq)
    # one age for the whole batch, as predict(x, 65.0) passes it
    torch.testing.assert_close(infer_reference(ref, x, 65.0, "independent", dtype=torch.float32)["z"],
                               O.ref_independent(ref, x, torch.tensor([65.0])), **eq)
    # the reference's own activation, spelled out, is the default
    explicit = infer_reference(ref, x, ages, "sequence", dtype=torch.float32, act="tanh", affine=None)
    torch.testing.assert_close(explicit["z"], seq["z"], **eq)


@pytest.mark.parametrize("mode", ["independent", "sequence"])
@pytest.mark.parametrize("act", ["relu", "identity"])
@pytest.mark.parametrize("geom", ["mycnn5", "mycnn3", "off-ref"])
def test_float64_reference_matches_plain_c_for_each_activation(geom, act, mode):
    """relu / identity, NaN and +-inf samples included: the patterns (relu(-inf) = 0; inf - inf = NaN under identity)
    and the finite values agree with the plain-C restatement"""
    if geom == "off-ref":
        ref = O.make_ref(OFF_REF, seed=6)
        x = tskd_b200.synth.make_windows(6, OFF_REF.in_channels, OFF_REF.window, "normal", seed=6)
        x[1, 0, 100] = float("nan"); x[2, 3, 350] = float("inf"); x[3, 0, 5] = float("-inf")
        ages = tskd_b200.synth.make_ages(6, seed=6)
    else:
        ref, x, ages = _case(geom, 3, 1500 if geom == "mycnn5" else 1502, 6, seed=7)
    got = infer_reference(ref, x, ages, mode, act=act)
    z, f = mycnn_c.forward(ref.arch, mycnn_c.pack_blob(ref.state_dict()), x.numpy(), ages.numpy(), mode=mode,
                           precision="f64", act=C_ACT[act], want_features=True)
    _close_1e12("features", got["features"].numpy(), f)
    _close_1e12("z", got["z"].numpy(), z)
    assert np.isfinite(z).any() or mode == "sequence"


def _batchnorm_pair(seed, c_mid=4):
    """two eval-mode BatchNorm1d in float64 with random statistics and affine parameters (some weights negative), and
    their fold (scale = weight / sqrt(var + eps), shift = bias - mean * scale) in float32, as the model stores it"""
    g = torch.Generator().manual_seed(seed)
    bns, fold = [], []
    for n in (c_mid, 1):
        bn = torch.nn.BatchNorm1d(n).double().eval()
        with torch.no_grad():
            bn.running_mean.copy_(torch.randn(n, generator=g, dtype=torch.float64))
            bn.running_var.copy_(0.5 + 1.5 * torch.rand(n, generator=g, dtype=torch.float64))
            bn.weight.copy_(torch.randn(n, generator=g, dtype=torch.float64))
            bn.bias.copy_(torch.randn(n, generator=g, dtype=torch.float64))
        s = (bn.weight / torch.sqrt(bn.running_var + bn.eps)).float()
        # the fold is rounded to float32 (what the C ABI takes); the BatchNorm is set to match it exactly
        with torch.no_grad():
            bn.weight.copy_(s.double() * torch.sqrt(bn.running_var + bn.eps))
        t = (bn.bias.double() - bn.running_mean * s.double()).float()
        with torch.no_grad():
            bn.bias.copy_(t.double() + bn.running_mean * s.double())
        bns.append(bn)
        fold += [s, t]
    assert (fold[0] < 0).any(), "the fold must include a negative scale"
    return bns, tuple(fold)


@pytest.mark.parametrize("act", ["tanh", "relu", "identity"])
@pytest.mark.parametrize("arch", [OFF_REF, replace(O.ARCH_MYCNN5, in_channels=3, window=1500)], ids=["off-ref", "mycnn5"])
def test_affine_reference_matches_torch_batchnorm(arch, act):
    """conv -> +bias -> * scale + shift -> act -> MaxPool, with the scale and shift folded from an eval BatchNorm1d,
    is torch.nn's Conv1d -> BatchNorm1d -> act -> MaxPool1d in float64"""
    ref = O.make_ref(arch, seed=8)
    (bn1, bn2), fold = _batchnorm_pair(8)
    x = tskd_b200.synth.make_windows(5, arch.in_channels, arch.window, "normal", seed=8)
    x[1, 0, 40] = float("nan"); x[2, arch.in_channels - 1, 77] = float("inf")
    got = infer_reference(ref, x, 65.0, act=act, affine=fold)["features"]
    m = copy.deepcopy(ref).double()
    f = ACTS[act]
    with torch.no_grad():
        want = m.pool(f(bn2(m.conv2(m.pool(f(bn1(m.conv1(x.double())))))))).view(-1, m.MAGICNUM)
    _close_1e12("features", got.numpy(), want.numpy())


def _pool_then_affine(ref, x, act, aff):
    """float32 features with each max pool taken BEFORE the affine and the activation (wrong for a negative scale)"""
    f = ACTS[act]
    s1, t1, s2, t2 = aff
    with torch.no_grad():
        v = f(ref.pool(ref.conv1(x.float())) * s1.view(1, -1, 1) + t1.view(1, -1, 1))
        v = f(ref.pool(ref.conv2(v)) * s2 + t2)
    return v.view(-1, ref.MAGICNUM)


@pytest.mark.parametrize("act", ["tanh", "relu", "identity"])
def test_comparator_rejects_pooling_before_a_negative_affine_scale(act):
    """Negative control without a GPU: features computed exactly in float32 but pooled before the affine (what the
    generic kernel's pooled-first branch would give if it ran with the affine on) fail the per-element bound at
    beta = 2^-20, while the float32 reference passes it."""
    ref = O.make_ref(OFF_REF, seed=9)
    x = tskd_b200.synth.make_windows(4, OFF_REF.in_channels, OFF_REF.window, "normal", seed=9)
    aff = centre_affine(ref, x, act, random_affine(9))
    assert (aff[0] < 0).any() and (aff[2] < 0).all()
    truth = infer_reference(ref, x, 65.0, act=act, affine=aff)["features"]
    ref32 = infer_reference(ref, x, 65.0, dtype=torch.float32, act=act, affine=aff)["features"]
    assert_close_elem("features", ref32, truth, ref32, beta=BETA)
    with pytest.raises(AssertionError, match="elements off"):
        assert_close_elem("features", _pool_then_affine(ref, x, act, aff), truth, ref32, beta=BETA)


def test_reference_leaves_the_module_untouched():
    ref, x, ages = _case("mycnn5", 3, 1500, 2, seed=5, bad=False)
    before = {k: v.clone() for k, v in ref.state_dict().items()}
    infer_reference(ref, x, ages)
    assert all(v.dtype == torch.float32 and torch.equal(v, before[k]) for k, v in ref.state_dict().items())


def _two_piece(ref):
    """conv1 weights as the sum of two bf16 pieces (16 mantissa bits): what the tc_splits=2 option feeds the MMAs"""
    r = copy.deepcopy(ref)
    with torch.no_grad():
        w = r.conv1.weight
        hi = w.bfloat16().float()
        w.copy_(hi + (w - hi).bfloat16().float())
    assert not torch.equal(r.conv1.weight, ref.conv1.weight)
    return r


@pytest.mark.parametrize("kind,dist", [("mycnn5", "physio"), ("mycnn5", "normal"), ("mycnn3", "normal")])
def test_comparator_rejects_two_piece_conv1_weights(kind, dist):
    """Negative control without a GPU: features computed exactly in float32 but from conv1 weights missing their third
    bf16 piece are rejected at the beta the tensor-core features are granted, while the float32 reference passes."""
    oarch = O.stretched(O.ARCHS[kind], 3, 7504)
    ref = O.make_ref(oarch, seed=0)
    x = tskd_b200.synth.make_windows(8, 3, 7504, dist, seed=3, dtype=torch.bfloat16)
    truth = infer_reference(ref, x, 65.0)["features"]
    ref32 = infer_reference(ref, x, 65.0, dtype=torch.float32)["features"]
    assert_close_elem("features", ref32, truth, ref32, beta=TC_FEATURES_BETA)
    two = infer_reference(_two_piece(ref), x, 65.0, dtype=torch.float32)["features"]
    with pytest.raises(AssertionError, match="elements off"):
        assert_close_elem("features", two, truth, ref32, beta=TC_FEATURES_BETA)
