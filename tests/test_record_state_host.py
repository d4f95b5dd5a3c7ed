"""CPU: the LSTM state across calls without a GPU -- predict_record's and SlidingScorer.admit's state checks, which run
before any library call, the C symbols bound in capi, and the float64 oracle with an initial state
(oracle/record_state_ref.py): its layout against nn.LSTM's (h, c) tuple, the split identity, the zero state as today's
oracle, the gradient of the initial state, the golden of the reference's utils.run_model scored in two chained chunks,
and the training oracle chained over two chunks against one pass."""
import os
import re

import numpy as np
import pytest
import torch

import tskd_b200
from conftest import GOLDEN, ROOT, load_golden
from oracle import mycnn_torch as O
from oracle.infer_ref import infer_reference
from oracle.record_state_ref import from_lstm_tuple, sequence_with_state, to_lstm_tuple, train_record_state_reference
from oracle.train_ref import assert_close_elem
from tskd_b200 import capi
from tskd_b200.model import check_record_state
from test_slide_state_host import _scorer

NEW = ("b2cnn_score_record_state", "b2cnn_slide_admit_ex")


def test_symbols_declared_and_bound():
    header = open(os.path.join(ROOT, "include", "b2cnn.h")).read()
    for name in NEW:
        assert name in capi.SYMBOLS
        assert re.search(rf"\b{name}\s*\(", header), name


def _model():
    return tskd_b200.B200MyCNN(tskd_b200.ARCH_PRESETS["mycnn5"].with_shape(3, 7504))


def test_predict_record_state_checks():
    m = _model()
    x = torch.zeros(2, 3, 9000, dtype=torch.bfloat16)
    ok = torch.zeros(2, 2, 2, 16, dtype=torch.float64)
    for state, ret in ((ok, False), (None, True), (ok, True)):
        with pytest.raises(ValueError, match="sequence"):                # before any library call
            m.predict_record(x, 8, state=state, return_state=ret)
    for bad in (torch.zeros(3, 2, 2, 16), torch.zeros(2, 64), torch.zeros(2, 2, 16, 2), torch.zeros(2, 2, 2, 16, dtype=torch.int32),
                [[0.0] * 16] * 8, 0.0):
        with pytest.raises(ValueError, match="state"):
            m.predict_record(x, 8, mode="sequence", state=bad)
    with pytest.raises(ValueError, match="return_state"):
        m.predict_record(x, 8, mode="sequence", return_state=1)
    with pytest.raises(ValueError, match="mode"):                        # the mode is still checked first
        m.predict_record(x, 8, mode="seq", state=ok)


def test_admit_lstm_checks():
    ind = _scorer()
    seq = _scorer()
    seq.mode = "sequence"
    lstm = torch.zeros(1, 2, 2, 16)
    with pytest.raises(ValueError, match="sequence-mode"):
        ind.admit([1], lstm=lstm)
    assert ind.check_lstm(None, 1) is None and seq.check_lstm(lstm, 1) is lstm
    for bad in (torch.zeros(2, 2, 2, 16), torch.zeros(1, 64), torch.zeros(1, 2, 2, 16, dtype=torch.int64), "zeros"):
        with pytest.raises(ValueError, match="lstm"):
            seq.admit([1], lstm=bad)


# ------------------------------------------------------------------ the oracle
def _ref():
    return O.make_ref(O.ARCH_MYCNN5, seed=3)


def test_layout_is_nn_lstm_tuple():
    ref = _ref().double()
    s = torch.randn(3, 2, 2, 16, dtype=torch.float64)
    h, c = to_lstm_tuple(s)
    assert h.shape == c.shape == (2, 3, 16)
    for b in range(3):
        for layer in range(2):
            assert torch.equal(h[layer, b], s[b, layer, 0]) and torch.equal(c[layer, b], s[b, layer, 1])
    assert torch.equal(from_lstm_tuple(h, c), s)
    # one nn.LSTM step from (h, c) returns the tuple in the same layout
    f = torch.randn(1, 3, ref.MAGICNUM, dtype=torch.float64)
    _, (hn, cn) = ref.lstm(f, (h, c))
    assert from_lstm_tuple(hn, cn).shape == (3, 2, 2, 16)


def test_zero_state_is_the_sequence_oracle():
    ref = _ref()
    x = tskd_b200.synth.make_windows(7, 10, 120, "normal", seed=1)
    age = torch.tensor([58.0])
    want = infer_reference(ref, x, age, "sequence")["z"]
    for state in (None, torch.zeros(2, 2, 16)):
        got = sequence_with_state(ref, x, age, state)["z"]
        assert torch.allclose(got, want, rtol=0, atol=1e-15)


def test_split_identity_and_empty():
    ref = _ref()
    x = tskd_b200.synth.make_windows(9, 10, 120, "normal", seed=2)
    age = torch.tensor([71.0])
    s0 = 0.5 * torch.randn(2, 2, 16, dtype=torch.float64)
    whole = sequence_with_state(ref, x, age, s0)
    for k in (1, 4, 8):
        a = sequence_with_state(ref, x[:k], age, s0)
        b = sequence_with_state(ref, x[k:], age, a["state"])
        assert torch.allclose(torch.cat([a["z"], b["z"]]), whole["z"], rtol=0, atol=1e-14)
        assert torch.allclose(b["state"], whole["state"], rtol=0, atol=1e-14)
    e = sequence_with_state(ref, x[:0], age, s0)
    assert e["z"].shape == (0,) and torch.equal(e["state"], s0)


def test_initial_state_gradient():
    """autograd through (h0, c0) against a central difference"""
    ref = _ref()
    x = tskd_b200.synth.make_windows(4, 10, 120, "normal", seed=4)
    age = torch.tensor([60.0])
    s0 = (0.3 * torch.randn(2, 2, 16, dtype=torch.float64)).requires_grad_(True)
    sequence_with_state(ref, x, age, s0)["z"].sum().backward()
    g = s0.grad
    i = (1, 1, 7)                                                       # c of layer 1, unit 7
    eps = 1e-6
    with torch.no_grad():
        sp, sm = s0.detach().clone(), s0.detach().clone()
        sp[i] += eps
        sm[i] -= eps
        fd = (sequence_with_state(ref, x, age, sp)["z"].sum() - sequence_with_state(ref, x, age, sm)["z"].sum()) / (2 * eps)
    assert abs(float(g[i]) - float(fd)) <= 1e-7 * max(1.0, abs(float(fd)))


@pytest.mark.parametrize("tag", ["a", "b"])
def test_run_model_golden_in_two_chunks(tag):
    """utils.run_model's golden (tests/golden/run_model_record.npz) from two chained float64 calls"""
    g = np.load(os.path.join(GOLDEN, "run_model_record.npz"))
    _, sd = load_golden("mycnn5_xtestinput.npz")
    ref = O.RefMyCNN(O.ARCH_MYCNN5)
    ref.load_state_dict(sd)
    ref.eval()
    win = torch.from_numpy(g[f"frame_{tag}"]).T.contiguous().unfold(1, 120, 120).permute(1, 0, 2).contiguous()
    n_gold = g[f"prob_{tag}"].shape[1]
    k = n_gold // 2
    for i, age in enumerate(g["ages"]):
        a = torch.tensor([float(age)])
        zs = {}
        for dt in (torch.float64, torch.float32):
            first = sequence_with_state(ref, win[:k], a, dtype=dt)
            second = sequence_with_state(ref, win[k:n_gold], a, first["state"], dtype=dt)
            zs[dt] = torch.sigmoid(torch.cat([first["z"], second["z"]])).detach()
        assert_close_elem(f"run_model {tag} two chunks age {age}", torch.from_numpy(g[f"prob_{tag}"][i]), zs[torch.float64],
                          zs[torch.float32])


def test_training_state_checks():
    x = torch.zeros(2, 10, 300)
    check_record_state(x, "sequence", torch.zeros(2, 2, 2, 16), True)
    check_record_state(x, "sequence", None, False)
    for state, ret in ((torch.zeros(2, 2, 2, 16), False), (None, True)):
        with pytest.raises(ValueError, match="sequence"):
            check_record_state(x, "independent", state, ret)
    for bad in (torch.zeros(3, 2, 2, 16), torch.zeros(2, 64), torch.zeros(2, 2, 2, 16, dtype=torch.int16), "zeros"):
        with pytest.raises(ValueError, match="state"):
            check_record_state(x, "sequence", bad, False)
    with pytest.raises(ValueError, match="return_state"):
        check_record_state(x, "sequence", None, "yes")
    for name in ("b2cnn_train_step_record_state", "b2cnn_train_forward_record_state", "b2cnn_train_backward_record_state"):
        assert name in capi.SYMBOLS


def test_training_oracle_chain_identity():
    """two chained float64 chunks of the training oracle give one pass's logits, final state and gradients"""
    ref = _ref()
    S, n_w, B = 12, 7, 2
    N = 120 + (n_w - 1) * S
    g = torch.Generator().manual_seed(5)
    rec = torch.randn(B, 10, N, generator=g)
    s0 = 0.5 * torch.randn(B, 2, 2, 16, generator=g, dtype=torch.float64)
    r = torch.randn(B * n_w, generator=g, dtype=torch.float64)
    ds = torch.randn(B, 2, 2, 16, generator=g, dtype=torch.float64)
    whole = train_record_state_reference(ref, rec, S, 60.0, [n_w] * B, s0, dz=r, dstate=ds)
    k = 3
    rz = r.reshape(B, n_w)
    b = train_record_state_reference(ref, rec[:, :, k * S:], S, 60.0, [n_w - k] * B, _state_after(ref, rec, S, k, s0),
                                     dz=rz[:, k:].reshape(-1), dstate=ds)
    a = train_record_state_reference(ref, rec[:, :, :(k - 1) * S + 120], S, 60.0, [k] * B, s0, dz=rz[:, :k].reshape(-1), dstate=b["dstate"])
    z = torch.cat([a["z"].reshape(B, k), b["z"].reshape(B, n_w - k)], dim=1).reshape(-1)
    assert torch.allclose(z, whole["z"], rtol=0, atol=1e-13) and torch.allclose(b["state"], whole["state"], rtol=0, atol=1e-13)
    assert torch.allclose(a["dstate"], whole["dstate"], rtol=0, atol=1e-12)
    for key in whole["grads"]:
        assert torch.allclose(a["grads"][key] + b["grads"][key], whole["grads"][key], rtol=0, atol=1e-11), key


def _state_after(ref, rec, S, k, s0, W=120):
    """each recording's state after its first k windows"""
    out = []
    for b in range(rec.shape[0]):
        wins = rec[b].unfold(1, W, S).permute(1, 0, 2)[:k]
        out.append(sequence_with_state(ref, wins, torch.tensor([60.0]), s0[b])["state"].detach())
    return torch.stack(out)


def test_training_refuses_overlapping_states():
    """the _record_state training calls refuse overlapping state arrays before any CUDA call (the step's backward reads
    state_in after its forward wrote state_out); the pointers here are never dereferenced"""
    import ctypes
    lib = tskd_b200.load_library()
    cfg = capi.make_config(tskd_b200.ARCH_PRESETS["mycnn5"])
    B, S = 2, 72
    N = 120 + 3 * S
    cts = (ctypes.c_int64 * B)(4, 4)
    P = ctypes.c_void_p
    fake = P(1 << 40)                                                   # params, records, age, z, workspace, ...
    rows = 64 * 4 * B                                                   # bytes of one state array
    a, half, after = P(1 << 41), P((1 << 41) + rows // 2), P((1 << 41) + rows)
    seq = capi.MODE_SEQUENCE
    for sin, sout in ((a, a), (a, half), (half, a)):
        rc = lib.b2cnn_train_forward_record_state(ctypes.byref(cfg), fake, fake, B, N, S, cts, seq, fake, None, None, sin, sout, fake,
                                                  fake, 1 << 40, None)
        assert rc == capi.EINVAL and "overlap" in capi.last_error()
        adam = capi.Adam(1e-3, 0.9, 0.999, 1e-8)
        rc = lib.b2cnn_train_step_record_state(ctypes.byref(cfg), fake, fake, fake, fake, 1, ctypes.byref(adam), 1, fake, B, N, S, cts, seq,
                                               fake, fake, None, None, None, sin, sout, fake, fake, 1 << 40, None)
        assert rc == capi.EINVAL and "overlap" in capi.last_error()
    # the backward: d_state_out onto d_state_in, and state_in onto d_state_in
    for sin, dso, dsi in ((None, a, a), (a, None, half), (after, a, half)):
        rc = lib.b2cnn_train_backward_record_state(ctypes.byref(cfg), fake, fake, B, N, S, cts, seq, fake, None, None, sin, fake, dso, fake,
                                                   None, None, dsi, 0, fake, 1 << 40, None)
        assert rc == capi.EINVAL and "overlap" in capi.last_error()
