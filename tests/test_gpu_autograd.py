"""GPU: the model in train() mode under torch autograd (b2cnn_train_forward / b2cnn_train_backward) and the fused step with
pos_weight, against the oracle module (oracle/mycnn_torch.py) in train() mode with the same explicit dropout masks, the
way test_gpu_train.py checks the fused step: per element against that graph in float64 (oracle/train_ref.py).  The reference's training cell (bin/explore_torch.ipynb:3140-3240) is
nn.BCEWithLogitsLoss(pos_weight=13.5) with optim.Adam(lr=1e-5), optim.Adagrad commented out beside it."""
from dataclasses import replace

import numpy as np
import pytest
import torch
from torch import nn

import tskd_b200
from tskd_b200.arch import BLOB_KEYS, INERT_KEYS
from tskd_b200.trainer import B200Trainer
from oracle import mycnn_torch as O
from oracle.train_ref import MaskDropout, assert_close_elem, train_reference
from conftest import rel_err
from test_gpu_train import _batch

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
POS_WEIGHT = 13.5                       # bin/explore_torch.ipynb:2116


def _pair(kind, C, W, seed=0):
    oarch = O.stretched(O.ARCHS[kind], C, W)
    ref = O.make_ref(oarch, seed=seed)
    ref.dropout = MaskDropout()
    ref.train()
    arch = replace(tskd_b200.ARCH_PRESETS[kind].with_shape(C, W), age_coef=oarch.age_coef)
    m = tskd_b200.B200TrainableMyCNN(arch, has_out12=oarch.has_out12).to(DEV)
    m.load_state_dict({k: v for k, v in ref.state_dict().items() if not k.startswith("dropout")})
    m.dropout.p = oarch.dropout
    return oarch, ref, m


def _dev(t):
    return None if t is None else t.to(DEV)


def _logits(m, x, age, mode, m1, m2):
    named = dict(m.named_parameters())
    return tskd_b200.mycnn_train_forward(x, age, [named[k] for k in BLOB_KEYS], m.arch, mode, _dev(m1), _dev(m2))


def _assert_loss_close(got, want, rel, step=None):
    got, want = float(got.detach()), float(want.detach())
    assert abs(got - want) <= rel * max(1.0, abs(want)), (step, got, want)


def _refs(ref, x, age, mode, m1, m2, **heads):
    """the float64 truth and the float32 yardstick (oracle/train_ref.py)"""
    return (train_reference(ref, x, age, mode, m1, m2, **heads),
            train_reference(ref, x, age, mode, m1, m2, dtype=torch.float32, **heads))


def _check_grads(got, truth, ref32):
    """got: the 14 BLOB_KEYS gradients; truth / ref32: one head of train_reference"""
    for k in BLOB_KEYS:
        assert_close_elem(k, got[k], truth["grads"][k], ref32["grads"][k])


def _check_module_grads(m, truth, ref32):
    named = dict(m.named_parameters())
    _check_grads({k: named[k].grad for k in BLOB_KEYS}, truth, ref32)
    for k in INERT_KEYS:
        if k in named:
            assert named[k].grad is None, k


@pytest.mark.parametrize("kind,C,W,B,mode,p", [
    ("mycnn5", 10, 120, 32, "sequence", 0.1),        # the reference's training shape and semantics
    ("mycnn5", 10, 120, 32, "independent", 0.1),
    ("mycnn2", 7, 120, 16, "sequence", 0.5),         # older revision: k1 = 5, pool(2,2), dropout 0.5
    ("mycnn5", 3, 1528, 12, "sequence", 0.1),        # a stretched window (L_out = 377)
])
def test_logits_and_gradients_match_autograd(kind, C, W, B, mode, p):
    oarch, ref, m = _pair(kind, C, W)
    x, age, _, m1, m2 = _batch(oarch, B, seed=5, p=p)
    r = torch.randn(B, generator=torch.Generator().manual_seed(9))       # an arbitrary upstream gradient d loss / d z
    xd, ad = x.to(DEV).requires_grad_(), age.to(DEV).requires_grad_()
    z = _logits(m, xd, ad, mode, m1, m2)
    (z * r.to(DEV)).sum().backward()
    truth, ref32 = _refs(ref, x, age, mode, m1, m2, dz=r)
    assert_close_elem("z", z, truth["z"], ref32["z"])
    _check_module_grads(m, truth["dz"], ref32["dz"])
    assert_close_elem("dx", xd.grad, truth["dz"]["dx"], ref32["dz"]["dx"])
    assert_close_elem("dage", ad.grad, truth["dz"]["dage"], ref32["dz"]["dage"])


def test_pos_weight_loss_through_autograd_and_the_fused_step():
    oarch, ref, m = _pair("mycnn5", 10, 120)
    x, age, _, m1, m2 = _batch(oarch, 32, seed=21, p=0.1)
    y = (torch.rand(32, generator=torch.Generator().manual_seed(4)) < 0.2).float()     # imbalanced, hence the class weight
    truth, ref32 = _refs(ref, x, age, "sequence", m1, m2, target=y, pos_weight=POS_WEIGHT)
    truth, ref32 = truth["bce_pw"], ref32["bce_pw"]
    loss = nn.BCEWithLogitsLoss(pos_weight=torch.tensor(POS_WEIGHT, device=DEV))(
        _logits(m, x.to(DEV), age.to(DEV), "sequence", m1, m2), y.to(DEV))
    loss.backward()
    assert_close_elem("loss", loss.reshape(1), truth["loss"].reshape(1), ref32["loss"].reshape(1))
    _check_module_grads(m, truth, ref32)

    plain = tskd_b200.B200MyCNN(m.arch).to(DEV)
    plain.load_state_dict(m.state_dict())
    tr = B200Trainer(plain, dropout=0.1, pos_weight=POS_WEIGHT)
    fused = tr.step(x, age, y, masks=(m1, m2), update=False)
    assert_close_elem("fused loss", fused.reshape(1), truth["loss"].reshape(1), ref32["loss"].reshape(1))
    _check_grads(tr.grads(), truth, ref32)


def _check_params_after_steps(sd, ref, lr):
    # as in test_gpu_train.py::test_three_adam_steps_follow_torch_optim, with the bounds scaled by the learning rate: where a
    # gradient is numerically zero its sign is noise, so the tight bound is over the entries with a real gradient signal
    # (plus a few float32 ulps of the parameter itself), and every entry moves by at most the steps themselves
    named = dict(ref.named_parameters())
    for k in BLOB_KEYS:
        a, b = sd[k].cpu().numpy().ravel(), named[k].detach().numpy().ravel()
        g = np.abs(named[k].grad.numpy().ravel())
        sel = g > 1e-4 * g.max()
        assert np.abs(a[sel] - b[sel]).max() <= 2e-2 * lr + 4e-7, (k, np.abs(a[sel] - b[sel]).max())
        assert np.abs(a - b).max() <= 6.1 * lr, (k, np.abs(a - b).max())


def _check_eval_scores(m, ref, oarch):
    m.eval()
    ref.eval()
    ref.dropout.set(None, None)
    xs, ages, _, _, _ = _batch(oarch, 9, seed=7, p=0.0)
    with torch.no_grad():
        want = ref(xs, ages).numpy()
    got = m(xs.to(DEV), ages.to(DEV)).cpu().numpy()
    assert rel_err(got, want) <= 1e-4


@pytest.mark.parametrize("optim,lr", [(torch.optim.Adam, 1e-5), (torch.optim.Adagrad, 5e-3)])
def test_three_steps_of_the_reference_training_cell(optim, lr):
    oarch, ref, m = _pair("mycnn5", 10, 120)
    m.train()
    opt_d, opt_r = optim(m.parameters(), lr=lr), optim(ref.parameters(), lr=lr)
    crit_d = nn.BCEWithLogitsLoss(pos_weight=torch.tensor(POS_WEIGHT, device=DEV))
    crit_r = nn.BCEWithLogitsLoss(pos_weight=torch.tensor(POS_WEIGHT))
    for step in range(3):
        x, age, y, m1, m2 = _batch(oarch, 64, seed=100 + step, p=0.1)             # batch 64, like the reference's cell
        opt_d.zero_grad()
        loss = crit_d(_logits(m, x.to(DEV), age.to(DEV), "sequence", m1, m2), y.to(DEV))
        loss.backward()
        opt_d.step()
        ref.dropout.set(m1, m2)
        opt_r.zero_grad()
        want = crit_r(ref(x, age), y)
        want.backward()
        opt_r.step()
        _assert_loss_close(loss, want, 2e-5, step)
    _check_params_after_steps(m.state_dict(), ref, lr)
    _check_eval_scores(m, ref, oarch)                  # the inference path scores with the updated weights


def test_autograd_adam_tracks_the_fused_step():
    oarch, ref, m = _pair("mycnn5", 10, 120)
    fused = tskd_b200.B200MyCNN(m.arch).to(DEV)
    fused.load_state_dict(m.state_dict())
    tr = B200Trainer(fused, lr=1e-3, dropout=0.1)
    opt = torch.optim.Adam(m.parameters(), lr=1e-3)
    m.train()
    for step in range(3):
        x, age, y, m1, m2 = _batch(oarch, 20, seed=200 + step, p=0.1)
        want = tr.step(x, age, y, masks=(m1, m2))
        opt.zero_grad()
        loss = nn.BCEWithLogitsLoss()(_logits(m, x.to(DEV), age.to(DEV), "sequence", m1, m2), y.to(DEV))
        loss.backward()
        opt.step()
        _assert_loss_close(loss, want, 2e-5, step)
    sd, got = m.state_dict(), fused.state_dict()
    grads = tr.grads()
    for k in BLOB_KEYS:
        a, b = sd[k].cpu().numpy().ravel(), got[k].cpu().numpy().ravel()
        g = np.abs(grads[k].cpu().numpy().ravel())
        sel = g > 1e-4 * g.max()
        assert np.abs(a[sel] - b[sel]).max() <= 2e-5, (k, np.abs(a[sel] - b[sel]).max())
        assert np.abs(a - b).max() <= 6.1e-3, (k, np.abs(a - b).max())


def test_module_forward_in_train_mode():
    """model.train(); model(x, age) draws its own masks; with p = 0 it is the oracle without dropout."""
    oarch, ref, m = _pair("mycnn5", 10, 120)
    x, age, y, _, _ = _batch(oarch, 16, seed=3, p=0.0)
    m.train()
    m.dropout.p = 0.0
    z = m(x.to(DEV), age[:1].to(DEV))                                  # one age for the batch, broadcast like the reference
    nn.BCEWithLogitsLoss()(z, y.to(DEV)).backward()
    truth, ref32 = _refs(ref, x, age[:1], "sequence", None, None, target=y)
    assert_close_elem("z", z, truth["z"], ref32["z"])
    _check_module_grads(m, truth["bce"], ref32["bce"])

    m.dropout.p = 0.1
    xb = x.to(DEV, torch.bfloat16).requires_grad_()
    torch.manual_seed(1)
    z1 = m(xb, age.to(DEV))
    z1.sum().backward()
    assert xb.grad is not None and xb.grad.dtype == torch.bfloat16 and xb.grad.shape == xb.shape
    torch.manual_seed(1)
    z2 = m(xb, age.to(DEV))
    torch.manual_seed(2)
    z3 = m(xb, age.to(DEV))
    assert torch.equal(z1, z2) and not torch.equal(z1, z3) and torch.isfinite(z1).all()
