"""CPU: the float64 training reference (oracle/train_ref.py) against finite differences, and the per-element comparator
(oracle/train_ref.py::assert_close_elem) the GPU training tests use."""
from dataclasses import replace

import numpy as np
import pytest
import torch
from torch.func import functional_call

from oracle import mycnn_torch as O
from oracle.mycnn_c import BLOB_KEYS
from oracle.train_ref import MaskDropout, assert_close_elem, pool_gaps, train_reference

# tiny layer stacks (hidden 3 keeps gradcheck's finite differences cheap; the graph is the same)
TINY = {
    "tail": O.RefArch(in_channels=2, k1=3, k2=2, pool_k=3, pool_s=2, hidden=3, window=12, age_coef=0.01,
                      has_out12=False),                   # L1 = 10: position 9 is in no pool window
    "gapped": O.RefArch(in_channels=2, k1=3, k2=2, pool_k=2, pool_s=3, window=14, age_coef=0.01,
                        hidden=3, has_out12=False),       # pool (2, 3): every third position is in no window
    "overlap": O.RefArch(in_channels=2, k1=2, k2=2, pool_k=2, pool_s=1, window=7, age_coef=0.01,
                         hidden=3, has_out12=False),
}


def _case(arch, B, seed):
    g = torch.Generator().manual_seed(seed)
    ref = O.make_ref(arch, seed=seed).double()
    x = torch.randn(B, arch.in_channels, arch.window, generator=g, dtype=torch.float64)
    age = torch.rand(B, generator=g, dtype=torch.float64) * 60 + 20
    m1 = torch.bernoulli(torch.full((B, arch.c_mid, arch.p1), 0.7, dtype=torch.float64), generator=g) / 0.7
    m2 = torch.bernoulli(torch.full((B, arch.l_out), 0.7, dtype=torch.float64), generator=g) / 0.7
    dz = torch.randn(B, generator=g, dtype=torch.float64)
    return ref, x, age, m1, m2, dz


def _logits_fn(ref, mode, m1, m2):
    """z as a function of (x, age, the 14 BLOB_KEYS tensors): the graph train_reference differentiates"""
    ref = ref.double()
    ref.dropout = MaskDropout()
    ref.train()

    def f(x, age, *params):
        p = dict(zip(BLOB_KEYS, params))
        if mode == "sequence":
            ref.dropout.set(m1, m2)
            return functional_call(ref, p, (x, age))
        outs = []
        for i in range(x.shape[0]):
            ref.dropout.set(m1[i:i + 1], m2[i:i + 1])
            outs.append(functional_call(ref, p, (x[i:i + 1], age[i:i + 1])))
        return torch.cat(outs)
    return f


@pytest.mark.parametrize("mode", ["sequence", "independent"])
@pytest.mark.parametrize("geom", sorted(TINY))
def test_float64_reference_passes_gradcheck(geom, mode):
    arch = TINY[geom]
    ref, x, age, m1, m2, dz = _case(arch, 3, seed=5)
    g1, g2 = pool_gaps(ref, x, m1)
    assert float(g1.min()) > 1e-3 and float(g2.min()) > 1e-3        # no max-pool kink within the finite differences
    named = dict(ref.named_parameters())
    params = [named[k].detach().clone().requires_grad_() for k in BLOB_KEYS]
    inputs = (x.clone().requires_grad_(), age.clone().requires_grad_(), *params)
    f = _logits_fn(ref, mode, m1, m2)
    assert torch.autograd.gradcheck(f, inputs, eps=1e-6, atol=1e-7, rtol=1e-5)
    # train_reference's "dz" head is the vector-Jacobian product of that same function
    z = f(*inputs)
    want = torch.autograd.grad(z, inputs, dz)
    got = train_reference(ref, x, age, mode, m1, m2, dz=dz)
    assert torch.equal(got["z"], z.detach())
    for k, w in zip(BLOB_KEYS, want[2:]):
        assert torch.allclose(got["dz"]["grads"][k], w, rtol=1e-12, atol=1e-15), k
    assert torch.allclose(got["dz"]["dx"], want[0], rtol=1e-12, atol=1e-15)
    assert torch.allclose(got["dz"]["dage"], want[1], rtol=1e-12, atol=1e-15)


def test_reference_heads_follow_the_loss_definitions():
    arch = TINY["tail"]
    ref, x, age, m1, m2, _ = _case(arch, 4, seed=6)
    y = torch.tensor([1.0, 0.0, 0.0, 1.0], dtype=torch.float64)
    out = train_reference(ref, x, age, "sequence", m1, m2, target=y, pos_weight=13.5)
    z = out["z"]
    plain = (torch.clamp(z, min=0) - z * y + torch.log1p(torch.exp(-z.abs()))).mean()
    weighted = ((1 - y) * z + (1 + 12.5 * y) * (torch.log1p(torch.exp(-z.abs())) + torch.clamp(-z, min=0))).mean()
    assert torch.allclose(out["bce"]["loss"], plain, rtol=1e-14) and torch.allclose(out["bce_pw"]["loss"], weighted, rtol=1e-14)
    # d loss / d z = (sigmoid(z) - y) / B for the plain head: through the "dz" head with that upstream gradient
    via_dz = train_reference(ref, x, age, "sequence", m1, m2, dz=(torch.sigmoid(z) - y) / 4)["dz"]
    for k in BLOB_KEYS:
        assert torch.allclose(out["bce"]["grads"][k], via_dz["grads"][k], rtol=1e-10, atol=1e-16), k


def test_age_relu_kink_gives_zero_gradient():
    arch = replace(TINY["gapped"], age_coef=-1.0 / 64)
    ref, x, _, m1, m2, dz = _case(arch, 3, seed=7)
    age = torch.tensor([32.0, 64.0, 100.0], dtype=torch.float64)              # scale 0.5, exactly 0, negative
    out = train_reference(ref, x, age, "independent", m1, m2, dz=dz)
    assert out["z"][1] == 0 and out["z"][2] == 0 and out["z"][0] != 0
    assert out["dz"]["dage"][1] == 0 and out["dz"]["dage"][2] == 0 and out["dz"]["dage"][0] != 0


def test_comparator_flags_a_small_entry_the_max_norm_passes():
    """a 1 % error on an entry 1000x below the tensor's largest passes max|err| / max|truth| <= 2e-4, but not this"""
    g = torch.Generator().manual_seed(0)
    truth = torch.randn(500, generator=g, dtype=torch.float64)
    truth[7] = truth.abs().max() * 1e-3
    ref32 = truth.float()
    got = ref32.clone()
    got[7] *= 1.01
    relerr = float((got.double() - truth).abs().max() / truth.abs().max())
    assert relerr <= 2e-4
    with pytest.raises(AssertionError, match=r"t: 1 of 500 elements off; worst at \(np.int64\(7\),\)"):
        assert_close_elem("t", got, truth, ref32)
    assert_close_elem("t", ref32, truth, ref32)                             # the float32 reference itself passes


def test_comparator_checks_nan_and_inf_patterns_and_caps_beta():
    truth = torch.tensor([1.0, float("nan"), float("inf"), -2.0], dtype=torch.float64)
    ref32 = truth.float()
    assert_close_elem("t", ref32, truth, ref32)
    with pytest.raises(AssertionError, match="NaN pattern"):
        assert_close_elem("t", torch.tensor([1.0, 0.0, float("inf"), -2.0]), truth, ref32)
    with pytest.raises(AssertionError, match="NaN pattern"):
        assert_close_elem("t", torch.tensor([float("nan"), float("nan"), float("inf"), -2.0]), truth, ref32)
    with pytest.raises(AssertionError, match="infinity"):
        assert_close_elem("t", torch.tensor([1.0, float("nan"), float("-inf"), -2.0]), truth, ref32)
    with pytest.raises(AssertionError):
        assert_close_elem("t", ref32, truth, ref32, beta=1e-4)
