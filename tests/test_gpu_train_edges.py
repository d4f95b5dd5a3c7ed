"""GPU: the training kernels (csrc/b2cnn_train.cu) element by element against the float64 reference of oracle/train_ref.py,
at the geometries, batch sizes, dropout masks, inputs and edge values where they could be subtly wrong: pool windows
that leave positions uncovered, overlap or skip positions; B = 1 and the benchmarked B = 2048 BPTT chain; saturated
tanh; exact pool ties (first-maximum routing); the relu kink of the age scale; bf16 inputs; NaN and inf.

Every comparison is oracle/train_ref.py::assert_close_elem: |got - truth| <= 8 |ref32 - truth| + beta max|truth| per element,
where ref32 is the same reference in float32.  Random inputs are checked for accidental near-ties in the pool windows
first (oracle/train_ref.py::pool_gaps): there a float32 kernel may legitimately route a gradient elsewhere."""
from dataclasses import replace

import numpy as np
import pytest
import torch

import tskd_b200
from tskd_b200.arch import BLOB_KEYS, ArchConfig
from tskd_b200.trainer import B200Trainer
from oracle import mycnn_torch as O
from oracle.train_ref import BETA, assert_close_elem, pool_gaps, train_reference
from conftest import rel_err

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
TIE_GAP = 2e-6          # relative gap below which a pool window counts as a near-tie (float32 conv rounding is ~1e-7)
POS_WEIGHT = 13.5

# small geometries through the same layer stack: C = 3, k1 = 4, k2 = 3
CUSTOM = {
    "pool43": O.RefArch(in_channels=3, k1=4, k2=3, pool_k=4, pool_s=3, window=60, dropout=0.1, has_out12=False),  # L1 tail uncovered
    "pool21": O.RefArch(in_channels=3, k1=4, k2=3, pool_k=2, pool_s=1, window=40, dropout=0.1, has_out12=False),  # overlapping
    "pool11": O.RefArch(in_channels=3, k1=4, k2=3, pool_k=1, pool_s=1, window=40, dropout=0.5, has_out12=False),  # no pooling
    "pool23": O.RefArch(in_channels=3, k1=4, k2=3, pool_k=2, pool_s=3, window=60, dropout=0.1, has_out12=False),  # gapped
}


def _oarch(kind, C=None, W=None):
    if kind in CUSTOM:
        return CUSTOM[kind]
    return O.stretched(O.ARCHS[kind], C, W)


def _arch(oarch):
    return ArchConfig(in_channels=oarch.in_channels, k1=oarch.k1, k2=oarch.k2, pool_k=oarch.pool_k, pool_s=oarch.pool_s,
                      window=oarch.window, age_coef=oarch.age_coef)


def _dev(t):
    return None if t is None else t.to(DEV)


def _masks(oarch, B, p, g):
    if p == 0:
        return None, None
    m1 = torch.bernoulli(torch.full((B, oarch.c_mid, oarch.p1), 1 - p), generator=g) / (1 - p)
    m2 = torch.bernoulli(torch.full((B, oarch.l_out), 1 - p), generator=g) / (1 - p)
    return m1, m2


def _inputs(oarch, B, seed, p, kind="normal"):
    """x, age, target, an upstream gradient with exact zeros, and the two dropout masks"""
    g = torch.Generator().manual_seed(seed)
    if kind == "physio":
        x = tskd_b200.synth.make_windows(B, oarch.in_channels, oarch.window, "physio", seed=seed)
    else:
        x = torch.randn(B, oarch.in_channels, oarch.window, generator=g)
    age = torch.rand(B, generator=g) * 60 + 20
    y = (torch.rand(B, generator=g) > 0.5).float()
    dz = torch.randn(B, generator=g)
    dz[::3] = 0.0
    m1, m2 = _masks(oarch, B, p, g)
    return x, age, y, dz, m1, m2


def _assert_no_near_ties(ref, x, m1):
    g1, g2 = pool_gaps(ref, x, m1)
    assert float(g1.min()) > TIE_GAP and float(g2.min()) > TIE_GAP, (float(g1.min()), float(g2.min()))


def _device(ref, arch, x, age, mode, m1, m2, dz, x_dtype=torch.float32):
    """logits and d(z . dz) / d(params, x, age) through mycnn_train_forward / torch autograd on the device"""
    sd = ref.state_dict()
    params = [sd[k].detach().to(DEV).clone().requires_grad_() for k in BLOB_KEYS]
    xd = x.to(DEV, x_dtype).requires_grad_()
    ad = age.to(DEV).requires_grad_()
    z = tskd_b200.mycnn_train_forward(xd, ad, params, arch, mode, _dev(m1), _dev(m2))
    z.backward(dz.to(DEV))
    return {"z": z.detach().cpu(), "grads": {k: p.grad.cpu() for k, p in zip(BLOB_KEYS, params)},
            "dx": xd.grad.cpu(), "dage": ad.grad.cpu()}


# the kernels' sigmoid and tanh (expf / tanhf, up to 2 ulp) against the CPU's, amplified by a (1 - a) and 1 - a^2 near
# saturation and along the BPTT chain
LSTM_BETA = {k: 4e-6 for k in BLOB_KEYS if k.startswith("lstm.")}


def _check(got, truth, ref32, head, beta=None):
    """every tensor of `got` per element; all failures reported together"""
    beta = {**LSTM_BETA, **(beta or {})}
    t, r = truth[head], ref32[head]
    pairs = [("z", got["z"], truth["z"], ref32["z"])] if "z" in got else []
    if "loss" in got:
        pairs.append(("loss", got["loss"].reshape(1), t["loss"].reshape(1), r["loss"].reshape(1)))
    pairs += [(k, got["grads"][k], t["grads"][k], r["grads"][k]) for k in BLOB_KEYS]
    pairs += [(k, got[k], t[k], r[k]) for k in ("dx", "dage") if k in got]
    errors = []
    for name, a, b, c in pairs:
        try:
            assert_close_elem(name, a, b, c, beta=beta.get(name, BETA))
        except AssertionError as e:
            errors.append(str(e))
    assert not errors, "\n".join(errors)


def _refs(ref, x, age, mode, m1, m2, **heads):
    return (train_reference(ref, x, age, mode, m1, m2, **heads),
            train_reference(ref, x, age, mode, m1, m2, dtype=torch.float32, **heads))


# ------------------------------------------------------------------ geometry x batch x dropout, through autograd
CASES = [
    # id, kind, C, W, B, mode, p, seed
    ("mycnn5-b1-seq", "mycnn5", 10, 120, 1, "sequence", 0.1, 1),
    ("mycnn5-b1-ind", "mycnn5", 10, 120, 1, "independent", 0.0, 2),
    ("mycnn5-b2-seq", "mycnn5", 10, 120, 2, "sequence", 0.5, 3),
    ("mycnn4-b257-ind", "mycnn4", 10, 120, 257, "independent", 0.1, 4),
    ("mycnn3-w1500-b2-ind", "mycnn3", 3, 1500, 2, "independent", 0.5, 5),
    ("mycnn3-w1500-b3-seq", "mycnn3", 3, 1500, 3, "sequence", 0.1, 6),
    ("mycnn5-w123-b257-seq", "mycnn5", 10, 123, 257, "sequence", 0.1, 15),   # L1 = 114, L2 = 52: last positions uncovered
    ("mycnn5-w123-b3-ind", "mycnn5", 10, 123, 3, "independent", 0.0, 8),
    ("pool43-b5-seq", "pool43", None, None, 5, "sequence", 0.1, 9),
    ("pool21-b5-ind", "pool21", None, None, 5, "independent", 0.1, 10),
    ("pool11-b5-seq", "pool11", None, None, 5, "sequence", 0.5, 11),
    ("pool23-b5-ind", "pool23", None, None, 5, "independent", 0.1, 12),
    ("pool23-b5-seq", "pool23", None, None, 5, "sequence", 0.1, 13),
    ("mycnn5-b2048-seq", "mycnn5", 10, 120, 2048, "sequence", 0.1, 14),      # the benchmarked size, the long BPTT chain
]
# at B >= 257 the conv gradients are sums over B x L1 >= 28 000 positions, and those long sums cancel
BIG_B_BETA = {k: 4e-6 for k in ("conv1.weight", "conv1.bias", "conv2.weight", "conv2.bias")}


@pytest.mark.parametrize("kind,C,W,B,mode,p,seed", [c[1:] for c in CASES], ids=[c[0] for c in CASES])
def test_autograd_matches_float64(kind, C, W, B, mode, p, seed):
    oarch = _oarch(kind, C, W)
    ref = O.make_ref(oarch, seed=seed)
    x, age, _, dz, m1, m2 = _inputs(oarch, B, seed, p)
    _assert_no_near_ties(ref, x, m1)
    truth, ref32 = _refs(ref, x, age, mode, m1, m2, dz=dz)
    got = _device(ref, _arch(oarch), x, age, mode, m1, m2, dz)
    _check(got, truth, ref32, "dz", BIG_B_BETA if B >= 257 else None)


def test_saturated_tanh_and_an_all_zero_dropout_row():
    oarch = O.ARCH_MYCNN5
    ref = O.make_ref(oarch, seed=23)
    x, age, _, dz, m1, m2 = _inputs(oarch, 64, 23, 0.5, kind="physio")    # conv1's tanh saturates
    m2[5] = 0.0                                                             # one window loses every feature
    _assert_no_near_ties(ref, x, m1)
    with torch.no_grad():
        assert (torch.tanh(ref.conv1(x)).abs() == 1.0).any()
    for mode in ("sequence", "independent"):
        truth, ref32 = _refs(ref, x, age, mode, m1, m2, dz=dz)
        # d x inherits the LSTM gradients' error through d f, and saturation leaves few positions to set its scale
        _check(_device(ref, _arch(oarch), x, age, mode, m1, m2, dz), truth, ref32, "dz", {"dx": 4e-6})


# ------------------------------------------------------------------ the fused step (BCE, BCE with pos_weight)
@pytest.mark.parametrize("kind,B,mode,pos_weight,seed", [
    ("mycnn5", 2048, "sequence", None, 35),
    ("mycnn5", 2048, "sequence", POS_WEIGHT, 35),
    ("mycnn4", 257, "independent", POS_WEIGHT, 32),
    ("mycnn5", 1, "sequence", None, 31),
])
def test_fused_step_matches_float64(kind, B, mode, pos_weight, seed):
    oarch = O.ARCHS[kind]
    ref = O.make_ref(oarch, seed=seed)
    x, age, y, _, m1, m2 = _inputs(oarch, B, seed, 0.1)
    _assert_no_near_ties(ref, x, m1)
    truth, ref32 = _refs(ref, x, age, mode, m1, m2, target=y, pos_weight=pos_weight)
    model = tskd_b200.B200MyCNN(_arch(oarch), has_out12=oarch.has_out12).to(DEV)
    model.load_state_dict(ref.state_dict())
    tr = B200Trainer(model, mode=mode, dropout=0.1, pos_weight=pos_weight)
    loss = tr.step(x, age, y, masks=(m1, m2), update=False)
    got = {"loss": loss.cpu(), "grads": {k: v.cpu() for k, v in tr.grads().items()}}
    _check(got, truth, ref32, "bce" if pos_weight is None else "bce_pw", BIG_B_BETA if B >= 257 else None)


# ------------------------------------------------------------------ exact pool ties: the first maximum takes the gradient
def _tie_case(B, seed):
    """conv1 weights and bias on the 2^-7 grid, integer samples in [-8, 8] with two constant runs of 40 samples per
    channel: every conv1 output is exact in any summation order, so every implementation sees the same ties, and the
    constant runs make whole stretches of c1, p1 and c2 equal"""
    oarch = O.ARCH_MYCNN5
    ref = O.make_ref(oarch, seed=seed)
    g = torch.Generator().manual_seed(seed)
    with torch.no_grad():
        ref.conv1.weight.copy_(torch.randint(-2, 3, ref.conv1.weight.shape, generator=g) / 128.0)
        ref.conv1.bias.copy_(torch.randint(-8, 9, ref.conv1.bias.shape, generator=g) / 128.0)
    x = torch.randint(-8, 9, (B, oarch.in_channels, oarch.window), generator=g).float()
    for lo in (20, 80):
        x[:, :, lo:lo + 40] = torch.randint(-8, 9, (B, oarch.in_channels, 1), generator=g).float()
    age = torch.rand(B, generator=g) * 60 + 20
    dz = torch.randn(B, generator=g)
    return oarch, ref, x, age, dz


@pytest.mark.parametrize("mode", ["sequence", "independent"])
def test_exact_pool_ties_route_to_the_first_maximum(mode):
    oarch, ref, x, age, dz = _tie_case(8, seed=41)
    g1, g2 = pool_gaps(ref, x)
    g1_32, g2_32 = pool_gaps(ref, x, dtype=torch.float32)
    for g64, g32 in ((g1, g1_32), (g2, g2_32)):
        ties = g64 == 0
        assert ties.any()                                            # there are ties ...
        assert torch.equal(ties, g32 == 0)                           # ... exact in the float32 reference too
        assert float(g64[~ties].min()) > TIE_GAP                     # and no near-ties besides them
    truth, ref32 = _refs(ref, x, age, mode, None, None, dz=dz)
    _check(_device(ref, _arch(oarch), x, age, mode, None, None, dz), truth, ref32, "dz")


# ------------------------------------------------------------------ the age scale relu(age * coef + 1)
@pytest.mark.parametrize("mode", ["sequence", "independent"])
def test_age_scale_kink_follows_torch_relu_backward(mode):
    """coef = -1/64, ages spanning 64: the scale is negative for some windows and exactly 0 at age 64, where torch's
    relu backward gives zero"""
    oarch = replace(O.ARCH_MYCNN5, age_coef=-1.0 / 64)
    ref = O.make_ref(oarch, seed=51)
    x, _, _, dz, m1, m2 = _inputs(oarch, 16, 51, 0.1)
    dz[::3] = torch.randn(len(dz[::3]), generator=torch.Generator().manual_seed(1))   # non-zero at the kink
    age = torch.tensor([30., 64., 40., 50., 60., 64., 70., 80., 90., 100., 63., 65., 20., 128., 94., 10.])
    _assert_no_near_ties(ref, x, m1)
    truth, ref32 = _refs(ref, x, age, mode, m1, m2, dz=dz)
    got = _device(ref, _arch(oarch), x, age, mode, m1, m2, dz)
    _check(got, truth, ref32, "dz")
    off = age >= 64
    assert (got["z"][off] == 0).all() and (got["dage"][off] == 0).all()
    assert (got["dage"][~off] != 0).all()


def test_scalar_age_broadcast_over_the_batch():
    oarch = O.ARCH_MYCNN4                                              # age_coef 1e-4
    ref = O.make_ref(oarch, seed=52)
    x, _, _, dz, m1, m2 = _inputs(oarch, 6, 52, 0.5)
    age = torch.tensor([57.0])
    _assert_no_near_ties(ref, x, m1)
    truth, ref32 = _refs(ref, x, age, "sequence", m1, m2, dz=dz)
    got = _device(ref, _arch(oarch), x, age, "sequence", m1, m2, dz)
    assert got["dage"].shape == (1,)
    _check(got, truth, ref32, "dz")


# ------------------------------------------------------------------ bf16 input
def test_bf16_input_gradient_within_one_ulp():
    oarch = O.ARCH_MYCNN5
    ref = O.make_ref(oarch, seed=61)
    x, age, _, dz, m1, m2 = _inputs(oarch, 16, 61, 0.1)
    xb = x.to(torch.bfloat16)
    xr = xb.float()                                                    # the input the kernels see
    _assert_no_near_ties(ref, xr, m1)
    truth, ref32 = _refs(ref, xr, age, "sequence", m1, m2, dz=dz)
    got = _device(ref, _arch(oarch), xb, age, "sequence", m1, m2, dz, x_dtype=torch.bfloat16)
    assert got["dx"].dtype == torch.bfloat16
    gx, tx = got.pop("dx").double().numpy(), truth["dz"]["dx"].numpy()
    ulp = 2.0 ** (np.floor(np.log2(np.maximum(np.abs(tx), 1e-300))) - 7)          # one bf16 ulp at the true value
    err, bound = np.abs(gx - tx), ulp + BETA * np.abs(tx).max()
    i = np.unravel_index(np.argmax(err - bound), tx.shape)
    assert (err <= bound).all(), (i, gx[i], tx[i])
    _check(got, truth, ref32, "dz")


# ------------------------------------------------------------------ NaN and inf
def _bad_batch(B, where, seed):
    """window 2 of B carries the bad value: NaN at the first / last sample or mid-window, or +inf / -inf"""
    oarch = O.ARCH_MYCNN5
    x, age, y, dz, m1, m2 = _inputs(oarch, B, seed, 0.1)
    dz = torch.randn(B, generator=torch.Generator().manual_seed(seed))
    pos = {"first": 0, "last": oarch.window - 1, "mid": 61, "+inf": 37, "-inf": 90}[where]
    x[2, 4, pos] = {"+inf": float("inf"), "-inf": float("-inf")}.get(where, float("nan"))
    return oarch, x, age, y, dz, m1, m2


@pytest.mark.parametrize("mode", ["sequence", "independent"])
@pytest.mark.parametrize("where", ["first", "last", "mid", "+inf", "-inf"])
def test_nan_and_inf_follow_the_reference(where, mode):
    oarch, x, age, y, dz, m1, m2 = _bad_batch(5, where, seed=71)
    ref = O.make_ref(oarch, seed=71)
    truth, ref32 = _refs(ref, x, age, mode, m1, m2, dz=dz, target=y)
    if where in ("first", "last", "mid"):
        assert torch.isnan(truth["z"][2]) and torch.isnan(truth["bce"]["loss"])
    got = _device(ref, _arch(oarch), x, age, mode, m1, m2, dz)
    _check(got, truth, ref32, "dz")
    if mode == "independent":                                          # the clean windows keep a finite input gradient
        clean = [0, 1, 3, 4]
        assert torch.isfinite(got["dx"][clean]).all() and torch.isfinite(got["z"][clean]).all()
    # the fused step: loss and gradient NaN patterns of the float64 loss
    model = tskd_b200.B200MyCNN(_arch(oarch)).to(DEV)
    model.load_state_dict(ref.state_dict())
    tr = B200Trainer(model, mode=mode, dropout=0.1)
    loss = tr.step(x, age, y, masks=(m1, m2), update=False)
    _check({"loss": loss.cpu(), "grads": {k: v.cpu() for k, v in tr.grads().items()}}, truth, ref32, "bce")


@pytest.mark.parametrize("mode", ["sequence", "independent"])
def test_train_mode_without_dropout_agrees_with_the_eval_path(mode):
    oarch = O.ARCH_MYCNN5
    ref = O.make_ref(oarch, seed=81)
    x, age, _, _, _, _ = _inputs(oarch, 8, 81, 0.0)
    x[1, 0, 0] = float("nan")
    x[3, 9, oarch.window - 1] = float("nan")
    x[5, 4, 61] = float("nan")
    x[6, 2, 37] = float("inf")
    arch = _arch(oarch)
    sd = ref.state_dict()
    params = [sd[k].to(DEV) for k in BLOB_KEYS]
    with torch.no_grad():
        train = tskd_b200.mycnn_train_forward(x.to(DEV), age.to(DEV), params, arch, mode).cpu().numpy()
    model = tskd_b200.B200MyCNN(arch).to(DEV)
    model.load_state_dict(sd)
    model.eval()
    if mode == "sequence":
        ev = model(x.to(DEV), age.to(DEV)).cpu().numpy()
    else:
        ev = model.predict(x.to(DEV), age.to(DEV), mode="independent").cpu().numpy()
    assert np.array_equal(np.isnan(train), np.isnan(ev)), (train, ev)
    assert np.isnan(ev).any()
    ok = ~np.isnan(ev)
    if ok.any():
        assert rel_err(train[ok], ev[ok]) <= 1e-5
