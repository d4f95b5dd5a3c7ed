"""GPU: parity of the CUDA path (through the C ABI, via ctypes) against
  * the committed golden vectors produced by the unmodified reference, and
  * the PyTorch-CPU oracle on the same seeded inputs, at sizes the oracle finishes in seconds.
Tolerance: 1e-4 relative on logits (BASELINE.json north_star), i.e.
max|gpu - ref| / max(|ref|, 1e-6) <= 1e-4; intermediate features: 2e-5 absolute.
"""
from dataclasses import replace

import numpy as np
import pytest
import torch

import tskd_b200
from conftest import load_golden, rel_err, rel_err_elem
from oracle import mycnn_c
from oracle import mycnn_torch as O

pytestmark = pytest.mark.gpu
TOL = 1e-4
DEV = "cuda:0"


def _pair(kind, C, W, seed=0, age_coef=None, path="auto"):
    """(oracle module, B200 model) with identical seeded weights."""
    oarch = O.stretched(O.ARCHS[kind], C, W)
    if age_coef is not None:
        oarch = replace(oarch, age_coef=age_coef)
    ref = O.make_ref(oarch, seed=seed)
    arch = replace(tskd_b200.ARCH_PRESETS[kind].with_shape(C, W), age_coef=oarch.age_coef)
    m = tskd_b200.B200MyCNN(arch, has_out12=oarch.has_out12, path=path).to(DEV)
    m.load_state_dict(ref.state_dict())
    return ref, m


# ------------------------------------------------------------------ golden vectors
def test_known_answer_mycnn5(golden5):
    g, sd = golden5
    m = tskd_b200.B200MyCNN.from_reference(sd).to(DEV)
    x = torch.from_numpy(g["x"]).to(DEV)
    for age in (50, 65):
        y = m(x, torch.tensor([float(age)], device=DEV))
        assert y.shape == (1,) and y.device.type == "cuda"
        assert rel_err(y.cpu().numpy(), g[f"logit_age{age}"]) <= 2e-6
    prob = m.predict(x, 50.0, return_prob=True).cpu().numpy()
    assert abs(prob[0] - 0.5668570399284363) < 2e-7                 # explore_torch.ipynb:4271
    assert np.abs(m.features(x).cpu().numpy() - g["features"]).max() < 2e-6
    # float64 numpy input as predictStream.py:105,155 builds it, host tensors in and out
    y = m(torch.from_numpy(g["x_f64"]), torch.tensor([50.0]))
    assert y.device.type == "cpu" and rel_err(y.numpy(), g["logit_age50"]) <= 2e-6
    assert m.gpu_launches >= 1 and m.last_path in ("generic", "tensorcore")


def test_batch_semantics_mycnn5(golden5):
    g, sd = golden5
    m = tskd_b200.B200MyCNN.from_reference(sd).to(DEV)
    for tag in ("xb", "xn"):
        x, a = torch.from_numpy(g[tag]).to(DEV), torch.from_numpy(g["ab"]).to(DEV)
        assert rel_err(m(x, a).cpu().numpy(), g[f"{tag}_seq_logits"]) <= TOL            # model(x_batch)
        assert rel_err(m.predict(x, a).cpu().numpy(), g[f"{tag}_ind_logits"]) <= TOL     # per-window loop
        assert rel_err(m.predict(x, a, mode="sequence").cpu().numpy(), g[f"{tag}_seq_logits"]) <= TOL
    assert np.abs(m.features(torch.from_numpy(g["xn"]).to(DEV)).cpu().numpy() - g["xn_features"]).max() < 2e-5


@pytest.mark.parametrize("n", [2, 3, 4])
def test_older_checkpoints(n):
    g, sd = load_golden(f"mycnn{n}_ckpt.npz")
    m = tskd_b200.B200MyCNN.from_reference(sd, age_coef=1e-8).to(DEV)   # goldens: bin/models.py forward
    x, a = torch.from_numpy(g["xb"]).to(DEV), torch.from_numpy(g["ab"]).to(DEV)
    assert rel_err(m(x, a).cpu().numpy(), g["seq_logits_coef1e8"]) <= TOL
    assert rel_err(m.predict(x, a).cpu().numpy(), g["ind_logits_coef1e8"]) <= TOL
    assert np.abs(m.features(x).cpu().numpy() - g["features"]).max() < 2e-5


@pytest.mark.parametrize("name", ["stretched_mycnn5_c3_w1500_b4.npz", "stretched_mycnn3_c3_w1500_b4.npz",
                                  "stretched_mycnn3_c3_w7500_b1.npz", "stretched_mycnn5_c3_w7500_b2.npz"])
def test_stretched_goldens(name):
    g, sd = load_golden(name)
    W = g["x"].shape[2]
    m = tskd_b200.B200MyCNN.from_reference(sd, window=W, age_coef=1e-8).to(DEV)
    x, a = torch.from_numpy(g["x"]).to(DEV), torch.from_numpy(g["age"]).to(DEV)
    assert rel_err(m(x, a).cpu().numpy(), g["seq_logits"]) <= TOL
    assert rel_err(m.predict(x, a).cpu().numpy(), g["ind_logits"]) <= TOL
    assert rel_err(m.predict(x.to(torch.bfloat16), a).cpu().numpy(), g["bf16_ind_logits"]) <= TOL
    assert np.abs(m.features(x).cpu().numpy() - g["features"]).max() < 2e-5


# ------------------------------------------------------------------ oracle on seeded inputs
@pytest.mark.parametrize("kind,C,W,B,dist,dtype", [
    ("mycnn5", 3, 7500, 96, "normal", torch.bfloat16),
    ("mycnn5", 3, 7500, 96, "physio", torch.bfloat16),
    ("mycnn5", 3, 7500, 64, "normal", torch.float32),
    ("mycnn3", 3, 7500, 64, "normal", torch.bfloat16),
    ("mycnn3", 3, 7500, 64, "physio", torch.float32),
    ("mycnn4", 10, 120, 300, "physio", torch.float32),
    ("mycnn5", 10, 120, 300, "normal", torch.float32),
    ("mycnn5", 3, 37500, 16, "normal", torch.bfloat16),
    ("mycnn5", 3, 75000, 12, "normal", torch.bfloat16),
    ("mycnn5", 3, 75000, 8, "physio", torch.bfloat16),
    ("mycnn3", 3, 75000, 8, "normal", torch.bfloat16),
    ("mycnn5", 7, 1203, 33, "normal", torch.float32),     # odd window length, ragged tile tail
])
def test_independent_vs_oracle(kind, C, W, B, dist, dtype):
    ref, m = _pair(kind, C, W)
    x = tskd_b200.synth.make_windows(B, C, W, dist, seed=11, dtype=dtype)
    ages = tskd_b200.synth.make_ages(B, seed=11)
    want = O.ref_independent(ref, x.float(), ages).numpy()
    got = m.predict(x.to(DEV), ages.to(DEV)).cpu().numpy()
    assert rel_err(got, want) <= TOL, (m.last_path, rel_err(got, want))
    fw = O.ref_features(ref, x.float()).numpy()
    fg = m.features(x.to(DEV)).cpu().numpy()
    assert np.abs(fg - fw).max() < 2e-5


@pytest.mark.parametrize("kind,C,W,B", [("mycnn5", 10, 120, 64), ("mycnn5", 10, 120, 16), ("mycnn3", 3, 1500, 40)])
def test_sequence_vs_oracle(kind, C, W, B):
    """utils.evaluate() calls model(input, age) with B=16/64 (explore_torch.ipynb:932,3151)."""
    ref, m = _pair(kind, C, W)
    x = tskd_b200.synth.make_windows(B, C, W, "normal", seed=5)
    ages = tskd_b200.synth.make_ages(B, seed=5)
    want = O.ref_sequence(ref, x, ages).numpy()
    got = m(x.to(DEV), ages.to(DEV)).cpu().numpy()
    assert rel_err(got, want) <= TOL


def test_closer_to_fp64_truth_than_tolerance():
    """Against the plain-C fp64 restatement: the CUDA path is as close to the exact result as
    torch-CPU fp32 is (both ~1e-6), far inside the 1e-4 bar."""
    ref, m = _pair("mycnn5", 3, 7500)
    x = tskd_b200.synth.make_windows(6, 3, 7500, "normal", seed=2)
    ages = tskd_b200.synth.make_ages(6, seed=2)
    blob = mycnn_c.pack_blob(ref.state_dict())
    truth = mycnn_c.forward(ref.arch, blob, x.numpy(), ages.numpy(), precision="f64")
    got = m.predict(x.to(DEV), ages.to(DEV)).cpu().numpy()
    cpu = O.ref_independent(ref, x, ages).numpy()
    assert rel_err(got, truth) <= 2e-5 and rel_err(cpu, truth) <= 2e-5


def test_age_broadcast_quirk_of_run_model(golden5):
    """utils.run_model passes age as (1, n) (bin/utils.py:681): n>1 gives a (1, n, n) result."""
    g, sd = golden5
    m = tskd_b200.B200MyCNN.from_reference(sd).to(DEV)
    ref = O.RefMyCNN(O.ARCH_MYCNN5); ref.load_state_dict(sd); ref.eval()
    x = torch.from_numpy(g["xn"][:3])
    age = torch.tensor([[50.0, 60.0, 70.0]])
    want = O.ref_sequence(ref, x, age)
    got = m(x.to(DEV), age.to(DEV)).cpu()
    assert got.shape == want.shape == (1, 3, 3)
    assert rel_err(got.numpy(), want.numpy()) <= TOL
    one = m(x[:1].to(DEV), torch.tensor([[50.0]], device=DEV))     # n == 1: shape (1, 1)
    assert one.shape == (1, 1)


# ------------------------------------------------------------------ edge cases
def test_nan_inf_semantics_match_reference():
    ref, m = _pair("mycnn5", 3, 7500)
    x = tskd_b200.synth.make_windows(8, 3, 7500, "edge", seed=4, dtype=torch.bfloat16)
    ages = torch.full((8,), 65.0)
    want = O.ref_independent(ref, x.float(), ages).numpy()
    got = m.predict(x.to(DEV), ages.to(DEV)).cpu().numpy()
    assert np.array_equal(np.isnan(want), np.isnan(got))
    assert np.isnan(want[0]) and np.isfinite(want[1])        # NaN propagates; +inf saturates
    ok = ~np.isnan(want)
    assert rel_err(got[ok], want[ok]) <= TOL
    # a NaN exactly at a pool-window edge must not be dropped (fmaxf would)
    x2 = torch.randn(1, 10, 120)
    x2[0, 2, 119] = float("nan")
    ref5, m5 = _pair("mycnn5", 10, 120)
    assert torch.isnan(O.ref_independent(ref5, x2, torch.tensor([65.0]))).all()
    assert torch.isnan(m5.predict(x2.to(DEV), 65.0)).all()


def test_batch_of_one_and_ragged_sizes():
    ref, m = _pair("mycnn5", 3, 7500)
    for B in (1, 2, 63, 65, 129):
        x = tskd_b200.synth.make_windows(B, 3, 7500, "normal", seed=B, dtype=torch.bfloat16)
        ages = tskd_b200.synth.make_ages(B, seed=B)
        want = O.ref_independent(ref, x.float(), ages).numpy()
        assert rel_err(m.predict(x.to(DEV), ages.to(DEV)).cpu().numpy(), want) <= TOL, B


def test_error_behaviour():
    _, m = _pair("mycnn5", 10, 120)
    with pytest.raises(RuntimeError, match="expected input"):
        m(torch.zeros(1, 9, 120, device=DEV), torch.tensor([50.0], device=DEV))
    with pytest.raises(RuntimeError, match="expected input"):
        m(torch.zeros(1, 10, 121, device=DEV), torch.tensor([50.0], device=DEV))
    with pytest.raises(RuntimeError, match="age"):
        m.predict(torch.zeros(4, 10, 120, device=DEV), torch.tensor([1.0, 2.0]))
    m.set_path("tensorcore")
    with pytest.raises(RuntimeError, match="tensor"):
        m(torch.zeros(1, 10, 120, device=DEV), torch.tensor([50.0], device=DEV))


def test_empty_batch_matches_reference():
    """model(x, a) on zero windows raises in the reference (nn.LSTM rejects a zero-length sequence, bin/models.py:30);
    the per-row loop over zero rows scores nothing (bin/predictStream.py:70) -> predict() returns an empty tensor."""
    ref, m = _pair("mycnn5", 10, 120)
    x0 = torch.zeros(0, 10, 120)
    with pytest.raises(RuntimeError):
        ref(x0, torch.zeros(0))
    with pytest.raises(RuntimeError):
        m(x0.to(DEV), torch.zeros(0, device=DEV))
    with pytest.raises(RuntimeError):
        m.predict(x0.to(DEV), 65.0, mode="sequence")
    out = m.predict(x0.to(DEV), 65.0)
    assert tuple(out.shape) == (0,) and out.dtype == torch.float32 and out.device.type == "cuda"
    with pytest.raises(RuntimeError, match="expected input"):
        m.predict(torch.zeros(0, 9, 120, device=DEV), 65.0)


def test_host_path_equals_device_path():
    ref, m = _pair("mycnn5", 3, 7500)
    x = tskd_b200.synth.make_windows(700, 3, 7500, "normal", seed=9, dtype=torch.bfloat16)   # > 1 chunk of 64 MiB? (31 MB) -> single; force more below
    ages = tskd_b200.synth.make_ages(700, seed=9)
    dev = m.predict(x.to(DEV), ages.to(DEV)).cpu()
    host = m.predict(x.pin_memory(), ages)
    assert host.device.type == "cpu" and torch.equal(dev, host)
    xf = x.float()                                            # 63 MB fp32 -> still one chunk; 2100 windows -> 3 chunks
    big = xf.repeat(3, 1, 1)
    hostb = m.predict(big, ages.repeat(3))
    assert torch.equal(hostb[:700], hostb[700:1400]) and rel_err(hostb[:700].numpy(), dev.numpy()) <= 1e-6


# Conv1d + (folded eval-BatchNorm) + ReLU/identity/tanh + MaxPool1d at other kernel/pool geometries (SURVEY.md section 0,
# reconciliation 1) is checked element by element against float64 in tests/test_gpu_generic_elem.py; the fold itself
# against torch.nn's BatchNorm1d in tests/test_oracle_infer.py.


# ------------------------------------------------------------------ full BASELINE size: properties
def test_full_size_properties():
    """[4096, 3, 75000] bf16 (BASELINE.json configs[1]): size-independent properties --
    equivariance under a permutation of the windows, prefix consistency, duplicate windows give
    bit-identical logits -- plus the oracle on ALL 4096 windows (chunks of 128 through torch-CPU, ~10-40 s of host
    time), judged per element."""
    ref, m = _pair("mycnn5", 3, 75000)
    B = 4096
    x = tskd_b200.synth.make_windows(B, 3, 75000, "normal", seed=1234, dtype=torch.bfloat16, device=DEV)
    ages = tskd_b200.synth.make_ages(B, seed=1234, device=DEV)
    x[B - 1] = x[0]; ages[B - 1] = ages[0]
    y = m.predict(x, ages)
    assert torch.isfinite(y).all() and y[0] == y[B - 1]
    perm = torch.randperm(B, device=DEV)
    assert torch.equal(m.predict(x[perm], ages[perm]), y[perm])
    assert torch.equal(m.predict(x[:1000], ages[:1000]), y[:1000])
    yh = y.cpu().numpy()
    worst = 0.0
    for b0 in range(0, B, 128):
        want = O.ref_independent(ref, x[b0:b0 + 128].float().cpu(), ages[b0:b0 + 128].cpu()).numpy()
        worst = max(worst, rel_err_elem(yh[b0:b0 + 128], want))
    assert worst <= TOL, worst


def test_single_launch_small_window_kernel(golden5):
    """[1,10,120] (the production call, predictStream.py:157) runs as ONE kernel launch; it must
    agree with the multi-kernel general path and with the reference goldens."""
    g, sd = golden5
    m = tskd_b200.B200MyCNN.from_reference(sd).to(DEV)
    x = torch.from_numpy(g["xn"]).to(DEV)
    a = torch.from_numpy(g["ab"]).to(DEV)
    y_small = m.predict(x, a)
    assert m.gpu_launches == 1 and m.last_path == "generic"
    m.set_option("small_kernel", 0)
    y_general = m.predict(x, a)
    assert m.gpu_launches > 1
    assert rel_err(y_small.cpu().numpy(), g["xn_ind_logits"]) <= 2e-6
    assert rel_err(y_small.cpu().numpy(), y_general.cpu().numpy()) <= 2e-6
    m.set_option("small_kernel", 1)
    one = m(torch.from_numpy(g["x"]).to(DEV), torch.tensor([50.0], device=DEV))
    assert m.gpu_launches == 1 and rel_err(one.cpu().numpy(), g["logit_age50"]) <= 2e-6
    # bf16 input, other geometry, sigmoid epilogue
    ref, m3 = _pair("mycnn3", 3, 1500)
    xb = tskd_b200.synth.make_windows(40, 3, 1500, "physio", seed=2, dtype=torch.bfloat16)
    ages = tskd_b200.synth.make_ages(40, seed=2)
    want = torch.sigmoid(O.ref_independent(ref, xb.float(), ages)).numpy()
    got = m3.predict(xb.to(DEV), ages.to(DEV), return_prob=True).cpu().numpy()
    assert m3.gpu_launches == 1 and rel_err(got, want) <= TOL


# ------------------------------------------------------------------ production shape, batched: [P, 10, 120]
@pytest.mark.parametrize("n,P,dtype", [(5, 1000, torch.float32), (5, 37, torch.float32), (5, 4096, torch.bfloat16),
                                       (4, 600, torch.float32), (3, 300, torch.float32), (2, 9, torch.float32)])
def test_short_window_batch_kernel_production_shape(n, P, dtype):
    """All patients of a trigger in ONE launch (one warp per window): the shipped checkpoints MyCNN5 (10 ch, k1=10,
    pool(3,2)), MyCNN4 (10 ch, k1=5, pool(2,2)), MyCNN2/3 (7 ch) on [P, C, 120] -- vs the oracle's per-window loop
    and vs the per-window launch path."""
    g, sd = load_golden("mycnn5_xtestinput.npz" if n == 5 else f"mycnn{n}_ckpt.npz")
    m = tskd_b200.B200MyCNN.from_reference(sd, age_coef=1e-8).to(DEV)
    C = m.arch.in_channels
    x = tskd_b200.synth.make_windows(P, C, 120, "physio", seed=20 + n, dtype=dtype, device=DEV)
    x[1] = tskd_b200.synth.make_windows(1, C, 120, "normal", seed=5, dtype=dtype, device=DEV)[0]
    ages = tskd_b200.synth.make_ages(P, seed=20 + n, device=DEV)
    y = m.predict(x, ages)
    assert m.gpu_launches == 1 and m.last_path == "generic"
    oarch = replace(O.ARCH_MYCNN5 if n == 5 else O.ARCHS["mycnn3"], in_channels=C, age_coef=1e-8, has_out12=("out1.weight" in sd))
    ref = O.RefMyCNN(oarch); ref.load_state_dict(sd); ref.eval()
    k = min(P, 256)
    want = O.ref_independent(ref, x[:k].float().cpu(), ages[:k].cpu()).numpy()
    assert rel_err_elem(y[:k].cpu().numpy(), want) <= TOL
    # the same windows one launch each (B < 8 takes the single-window kernel): same numbers to fp32 noise
    one = torch.cat([m.predict(x[i:i + 1], ages[i:i + 1]) for i in range(0, k, max(1, k // 16))])
    assert rel_err(one.cpu().numpy(), y[:k:max(1, k // 16)].cpu().numpy()) <= 2e-6
    prob = m.predict(x[:k], ages[:k], return_prob=True).cpu().numpy()
    assert rel_err(prob, 1 / (1 + np.exp(-want.astype(np.float64)))) <= TOL
    # NaN / inf semantics of the reference (max_pool1d propagates NaN, tanh saturates inf)
    xe = x[:16].clone().float()
    xe[3, 2, 50] = float("nan"); xe[5, 0, 119] = float("inf"); xe[7, C - 1, 0] = float("-inf")
    we = O.ref_independent(ref, xe.cpu(), ages[:16].cpu()).numpy()
    ge = m.predict(xe, ages[:16]).cpu().numpy()
    assert np.array_equal(np.isnan(we), np.isnan(ge)) and np.isnan(we[3]) and np.isfinite(we[5])
    assert rel_err(ge[~np.isnan(we)], we[~np.isnan(we)]) <= TOL
