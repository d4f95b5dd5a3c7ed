"""GPU: one training step (row f4, csrc/b2cnn_train.cu) against torch autograd + torch.optim.Adam on the oracle module.

The oracle (oracle/mycnn_torch.py, the layer stack of bin/models.py:5-36) runs the reference's training-loop body
(bin/utils.py:200-208) on the CPU: zero_grad, model(input, age) in train() mode, nn.BCEWithLogitsLoss (bin/utils.py:663),
backward, torch.optim.Adam.step (bin/explore_torch.ipynb:3204-3205).  Dropout masks are explicit on both sides (torch's
Philox stream cannot be shared): the oracle's nn.Dropout is swapped for a module that multiplies by the same masks, in
call order, so its own forward() is what gets differentiated.  The loss and the gradients of one step are compared element by
element with that graph in float64 (oracle/train_ref.py: train_reference, assert_close_elem)."""
from dataclasses import replace

import numpy as np
import pytest
import torch
from torch import nn

import tskd_b200
from tskd_b200.trainer import B200Trainer
from oracle import mycnn_torch as O
from oracle.train_ref import MaskDropout, assert_close_elem, train_reference
from conftest import rel_err

pytestmark = pytest.mark.gpu
DEV = "cuda:0"


def _pair(kind, C, W, seed=0):
    oarch = O.stretched(O.ARCHS[kind], C, W)
    ref = O.make_ref(oarch, seed=seed)
    ref.dropout = MaskDropout()
    ref.train()
    arch = replace(tskd_b200.ARCH_PRESETS[kind].with_shape(C, W), age_coef=oarch.age_coef)
    m = tskd_b200.B200MyCNN(arch, has_out12=oarch.has_out12).to(DEV)
    m.load_state_dict({k: v for k, v in ref.state_dict().items() if not k.startswith("dropout")})
    return oarch, ref, m


def _batch(oarch, B, seed, p):
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(B, oarch.in_channels, oarch.window, generator=g)
    age = torch.rand(B, generator=g) * 60 + 20
    y = (torch.rand(B, generator=g) > 0.5).float()
    if p > 0:
        m1 = torch.bernoulli(torch.full((B, 4, oarch.p1), 1 - p), generator=g) / (1 - p)
        m2 = torch.bernoulli(torch.full((B, oarch.l_out), 1 - p), generator=g) / (1 - p)
    else:
        m1 = m2 = None
    return x, age, y, m1, m2


@pytest.mark.parametrize("kind,C,W,B,mode,p", [
    ("mycnn5", 10, 120, 32, "sequence", 0.1),        # the reference's training shape and semantics
    ("mycnn5", 10, 120, 7, "sequence", 0.0),
    ("mycnn5", 10, 120, 24, "independent", 0.1),
    ("mycnn2", 7, 120, 16, "sequence", 0.5),         # older revision: k1 = 5, pool(2,2), dropout 0.5
    ("mycnn5", 3, 1528, 12, "sequence", 0.1),        # a stretched window (L_out = 377)
])
def test_gradients_and_loss_match_autograd(kind, C, W, B, mode, p):
    oarch, ref, m = _pair(kind, C, W)
    x, age, y, m1, m2 = _batch(oarch, B, seed=5, p=p)
    tr = B200Trainer(m, mode=mode, dropout=p)
    loss = tr.step(x, age, y, masks=(m1, m2), update=False)
    truth = train_reference(ref, x, age, mode, m1, m2, target=y)["bce"]
    ref32 = train_reference(ref, x, age, mode, m1, m2, target=y, dtype=torch.float32)["bce"]
    assert_close_elem("loss", loss.cpu().reshape(1), truth["loss"].reshape(1), ref32["loss"].reshape(1))
    got = tr.grads()
    for k in tskd_b200.arch.BLOB_KEYS:
        assert_close_elem(k, got[k], truth["grads"][k], ref32["grads"][k])


def test_three_adam_steps_follow_torch_optim():
    oarch, ref, m = _pair("mycnn5", 10, 120)
    tr = B200Trainer(m, lr=1e-3, mode="sequence", dropout=0.1)
    opt = torch.optim.Adam(ref.parameters(), lr=1e-3)
    for step in range(3):
        x, age, y, m1, m2 = _batch(oarch, 20, seed=100 + step, p=0.1)
        loss = tr.step(x, age, y, masks=(m1, m2))
        ref.dropout.set(m1, m2)
        opt.zero_grad()
        want = nn.BCEWithLogitsLoss()(ref(x, age), y)
        want.backward()
        opt.step()
        assert abs(float(loss) - float(want)) <= 2e-5 * max(1.0, abs(float(want))), (step, float(loss), float(want))
    # Adam's update is lr * m / (sqrt(v) + eps): where a gradient is numerically zero its sign is noise, so the
    # comparison is over the entries with a real gradient signal and on the net movement of every tensor
    sd, named = m.state_dict(), dict(ref.named_parameters())
    for k in tskd_b200.arch.BLOB_KEYS:
        a, b = sd[k].cpu().numpy().ravel(), named[k].detach().numpy().ravel()
        g = np.abs(named[k].grad.numpy().ravel())
        sel = g > 1e-4 * g.max()
        assert np.abs(a[sel] - b[sel]).max() <= 2e-5, (k, np.abs(a[sel] - b[sel]).max())
        assert np.abs(a - b).max() <= 6.1e-3            # never more than the three steps themselves (3 x 2 lr)
    # the inference path scores with the updated weights
    ref.eval()
    ref.dropout.set(None, None)
    xs, ages, _, _, _ = _batch(oarch, 9, seed=7, p=0.0)
    with torch.no_grad():
        want = ref(xs, ages).numpy()
    got = m(xs.to(DEV), ages.to(DEV)).cpu().numpy()
    assert rel_err(got, want) <= 1e-4


def test_training_decreases_the_loss_with_its_own_masks():
    oarch, _, m = _pair("mycnn5", 10, 120, seed=3)
    tr = B200Trainer(m, lr=5e-3, mode="sequence", dropout=0.1, seed=1)
    x, age, y, _, _ = _batch(oarch, 48, seed=11, p=0.0)
    y = (x[:, 0, :].mean(dim=1) > 0).float()             # a learnable target
    first = float(tr.step(x, age, y))
    for _ in range(60):
        last = float(tr.step(x, age, y))
    assert np.isfinite(last) and last < 0.8 * first, (first, last)
