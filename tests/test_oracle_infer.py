"""CPU: the inference reference (oracle/infer_ref.py) -- in float64 against the independent plain-C float64 restatement
(oracle/mycnn_ref.c), in float32 against the existing oracle bit for bit -- and a negative control showing that the
per-element comparator the GPU inference tests use (oracle/train_ref.py::assert_close_elem) sees conv1 weights that
lost their third bf16 piece."""
import copy

import numpy as np
import pytest
import torch

import tskd_b200
from oracle import mycnn_c
from oracle import mycnn_torch as O
from oracle.infer_ref import TC_FEATURES_BETA, infer_reference
from oracle.train_ref import assert_close_elem


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
