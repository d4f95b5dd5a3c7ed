"""GPU: export and import of SlidingScorer patients (SlidingScorer.export / restore, b2cnn_slide_export / _import,
csrc/b2cnn_slide.cu).

The main criterion is bit identity with an uninterrupted scorer.  Scorer A pushes n1 segments; some of its patients
are exported and imported into scorer B, which has another P, other slots, another push count and a ring rotated by
other streams.  From then on A and B get the same segments for those patients, and at every push their logits and
features() rows are torch.equal, NaN for NaN.  Twins that never export or import show that neither call disturbs
anything else: A against a twin that never exported, B's other patients against a twin that never imported."""
import ctypes
from dataclasses import replace

import numpy as np
import pytest
import torch

import tskd_b200
from conftest import load_golden
from oracle import mycnn_torch as O
from oracle.infer_ref import centre_affine, infer_reference, random_affine
from oracle.train_ref import BETA, check_elems
from tskd_b200 import capi

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
BF, F32 = torch.bfloat16, torch.float32
M5, M3 = (10, 5, 3, 2), (5, 5, 2, 2)          # (k1, k2, pool_k, pool_s) of MyCNN5 and MyCNN2/3/4


def _same(a, b):
    """bit-identical, NaN for NaN"""
    na, nb = torch.isnan(a), torch.isnan(b)
    return torch.equal(na, nb) and torch.equal(a[~na], b[~nb])


def _rows(t, idx, width=None):
    """rows idx of a push output / features, NaN rows for None (no complete window anywhere)"""
    if t is None:
        shape = (len(idx),) if width is None else (len(idx), width)
        return torch.full(shape, float("nan"))
    return t[torch.tensor(idx, device=t.device)].cpu()


def _feats(sc):
    """features(), None when no patient has a complete window"""
    try:
        return sc.features()
    except RuntimeError as e:
        assert "b2cnn error 5" in str(e)
        return None


# ------------------------------------------------------------------ models
def _tc_model(kind, C, W, seed):
    """(ref, model) of a tensor-core geometry"""
    ref = O.make_ref(O.stretched(O.ARCHS[kind], C, W), seed=seed)
    arch = replace(tskd_b200.ARCH_PRESETS[kind].with_shape(C, W), age_coef=ref.arch.age_coef)
    m = tskd_b200.B200MyCNN(arch, has_out12=ref.arch.has_out12).to(DEV)
    m.load_state_dict(ref.state_dict())
    return ref, m


def _gen_model(geo, act="tanh", aff_seed=None, seed=0):
    """(ref state dict, model) of any geometry for the generic path, predict() with path generic and small_kernel 0"""
    C, k1, k2, pk, ps, W = geo
    ref = O.make_ref(O.RefArch(in_channels=C, k1=k1, k2=k2, pool_k=pk, pool_s=ps, window=W, age_coef=1e-4, has_out12=False),
                     seed=seed)
    sd = dict(ref.state_dict())
    if aff_seed is not None:
        aff = centre_affine(ref, tskd_b200.synth.make_windows(4, C, W, "normal", seed=seed), act, random_affine(aff_seed))
        sd.update(zip(("affine1_scale", "affine1_shift", "affine2_scale", "affine2_shift"), aff))
    arch = tskd_b200.ArchConfig(in_channels=C, k1=k1, k2=k2, pool_k=pk, pool_s=ps, window=W, age_coef=1e-4, act=act,
                                affine=aff_seed is not None)
    m = tskd_b200.B200MyCNN(arch, has_out12=False, path="generic").to(DEV)
    m.load_state_dict(sd)
    m.set_option("small_kernel", 0)
    return sd, m


def _golden5():
    g, sd = load_golden("mycnn5_xtestinput.npz")
    m = tskd_b200.B200MyCNN.from_reference(sd, age_coef=1e-8, path="generic").to(DEV)
    m.set_option("small_kernel", 0)
    return sd, m


def _lattice(arch):
    """(F, R): feature stride and receptive field of one feature"""
    return arch.pool_s ** 2, arch.pool_s * (arch.pool_k + arch.k2 - 2) + arch.pool_k + arch.k1 - 1


def _seg(P, C, S, dtype, seed):
    return tskd_b200.synth.make_windows(P, C, S, "normal", seed=seed, dtype=dtype)


# ------------------------------------------------------------------ the main criterion
class Side:
    """A scorer and its twin: both get every push, admit and discharge, only the scorer exports or imports.  rec holds
    the last T samples of every stream as the scorer's tails hold them (zeros before the stream)."""

    def __init__(self, m, P, S, dtype, path, seed):
        self.m, self.P, self.S, self.C, self.W = m, P, S, m.arch.in_channels, m.arch.window
        self.sc = tskd_b200.SlidingScorer(m, P, S, dtype, path=path)
        self.tw = tskd_b200.SlidingScorer(m, P, S, dtype, path=path)
        assert self.sc.path == path
        self.T = self.sc._state_fields["tail_len"]
        self.rec = torch.zeros(P, self.C, self.T)
        self.age = tskd_b200.synth.make_ages(P, seed=seed).to(DEV)

    def push(self, seg):
        seg_d = seg.to(DEV)
        self.out, self.tout = self.sc.push(seg_d, self.age), self.tw.push(seg_d, self.age)
        self.rec = torch.cat([self.rec, seg.float()], dim=2)[:, :, -self.T:]
        return self.out

    def admit(self, idx, hist):
        for sc in (self.sc, self.tw):
            sc.admit(idx, hist.to(DEV))
        self.rec[idx] = torch.cat([torch.zeros(len(idx), self.C, self.T), hist.float()], dim=2)[:, :, -self.T:]

    def discharge(self, idx):
        for sc in (self.sc, self.tw):
            sc.discharge(idx)


def _poison(seg, rows, S, R):
    """NaN in the last samples (the tail), +inf inside the next push's seam, -inf and NaN further back (features)"""
    C = seg.shape[1]
    seg[rows[0], 0, S - 2] = float("nan")
    seg[rows[1], 1 % C, max(S - R // 2, 0)] = float("inf")
    seg[rows[2], 0, 0] = float("-inf")
    seg[rows[3], C - 1, S // 2] = float("nan")


def run_move(mA, mB, P_A, P_B, S, dtype, path, n1, n_b, n2, seed, states=True, bad=True, tmp_path=None):
    """A (model mA) pushes n1 segments -- with `states` a patient is admitted with a short history (seen < W at the
    export), one discharged (seen = -1) and one readmitted with a full window; with `bad` NaN / inf samples land in
    the last pushes -- and exports k patients.  B (model mB, P_B patients, n_b pushes of other streams first) restores
    them into shuffled slots.  Over n2 more pushes A and B must agree bit for bit on those patients, A with its twin
    on every patient, and B with its twin on every other patient."""
    rng = np.random.default_rng(seed)
    A, B = Side(mA, P_A, S, dtype, path, seed), Side(mB, P_B, S, dtype, path, seed + 1)
    C, W, L = A.C, A.W, mA.arch.l_out
    F, R = _lattice(mA.arch)
    k = min(P_A, P_B) // 2 + 3
    move = [int(v) for v in rng.permutation(P_A)[:k]]
    slots = [int(v) for v in rng.permutation(P_B)[:k]]
    others = sorted(set(range(P_B)) - set(slots))
    B.age[torch.tensor(slots, device=DEV)] = A.age[torch.tensor(move, device=DEV)]       # the same patients' ages
    for t in range(n1):
        seg = _seg(P_A, C, S, dtype, seed * 100 + t)
        if bad and t >= n1 - 2:
            _poison(seg, move[4:8], S, R)
        if states and t == n1 - 1:
            A.admit([move[0]], _seg(1, C, max(W - 2 * S, 0), dtype, seed * 100 + 50))
            A.discharge([move[1]])
            A.admit([move[2]], _seg(1, C, W, dtype, seed * 100 + 51))
        A.push(seg)
    for t in range(n_b):
        B.push(_seg(P_B, C, S, dtype, seed * 100 + 70 + t))

    fa = _feats(A.sc)
    state = A.sc.export(move)
    seen_a = A.sc.samples_seen.cpu()
    assert torch.equal(state["seen"], seen_a[move]) and state["seen"].device.type == "cpu"
    assert state["features"].device == A.sc.device and state["tail"].shape == (k, C, A.T)
    assert _same(state["tail"].cpu(), A.rec[move])                    # the last T samples, converted to fp32
    complete = [j for j, p in enumerate(move) if seen_a[p] >= W]
    assert complete
    if fa is not None:                                                 # bit-identical to features() rows
        assert _same(state["features"][complete].cpu(), _rows(fa, [move[j] for j in complete]))
    if tmp_path is not None:
        torch.save(state, tmp_path / "ward.pt")
        state = torch.load(tmp_path / "ward.pt")
    B.sc.restore(slots, state)
    assert torch.equal(B.sc.samples_seen.cpu()[slots], seen_a[move])
    fb = B.sc.features()                                               # at once, before the next push
    assert _same(_rows(fb, [slots[j] for j in complete]), state["features"][complete].cpu())

    scored = 0
    for t in range(n2):
        sa = _seg(P_A, C, S, dtype, seed * 100 + 200 + t)
        if bad and t == 0:
            _poison(sa, move[-4:], S, R)
        sb = _seg(P_B, C, S, dtype, seed * 100 + 300 + t)
        sb[slots] = sa[move]
        oa, ob = A.push(sa), B.push(sb)
        assert (oa is None) == (A.tout is None) and (oa is None or _same(oa, A.tout)), t      # export changed nothing
        assert _same(_rows(oa, move), _rows(ob, slots)), t
        assert _same(_rows(ob, others), _rows(B.tout, others)), t                             # nor did the import
        fa, fat, fb, fbt = _feats(A.sc), _feats(A.tw), _feats(B.sc), _feats(B.tw)
        assert (fa is None) == (fat is None) and (fa is None or _same(fa, fat)), t
        assert _same(_rows(fa, move, L), _rows(fb, slots, L)), t
        assert _same(_rows(fb, others, L), _rows(fbt, others, L)), t
        scored += 0 if oa is None else int((~torch.isnan(_rows(oa, move))).sum())
    assert scored > 0
    return A, B, move, slots


TC_CASES = {
    #          kind, C, W, S, dtype, P_A, P_B, n1, n_b, n2
    "m5-c3-bf16": ("mycnn5", 3, 7504, 1876, BF, 130, 200, 6, 2, 5),
    "m5-c3-bf16-fresh": ("mycnn5", 3, 7504, 1876, BF, 130, 70, 6, 0, 5),        # B never pushed: negative indices
    "m5-c2-f32": ("mycnn5", 2, 4000, 1000, F32, 40, 56, 5, 3, 4),
    "m3-c3-f32-w7502": ("mycnn3", 3, 7502, 1876, F32, 64, 40, 6, 1, 4),         # W % 4 != 0
    "m3-c1-bf16-fresh": ("mycnn3", 1, 4000, 1000, BF, 40, 36, 7, 0, 4),
}


@pytest.mark.parametrize("name", list(TC_CASES))
def test_move_tensorcore(name):
    kind, C, W, S, dtype, P_A, P_B, n1, n_b, n2 = TC_CASES[name]
    _, m = _tc_model(kind, C, W, seed=3 + list(TC_CASES).index(name))
    run_move(m, m, P_A, P_B, S, dtype, "tensorcore", n1, n_b, n2, seed=list(TC_CASES).index(name) + 1)


GEN_CASES = {
    #            geo or "golden", act, aff, S, dtype, P_A, P_B, n1, n_b, n2
    "golden-m5-w120-s12": ("golden", "tanh", None, 12, F32, 40, 56, 12, 3, 6),
    "golden-m5-w120-s12-bf16-fresh": ("golden", "tanh", None, 12, BF, 40, 24, 12, 0, 6),
    "c10-w75000": ((10,) + M5 + (75000,), "tanh", None, 7500, BF, 200, 160, 11, 2, 2),
    "c10-relu-negaff": ((10,) + M5 + (600,), "relu", 1, 100, F32, 40, 48, 8, 2, 5),
    "c16-pool44-f16": ((16, 3, 8, 4, 4, 1470), "tanh", None, 160, BF, 24, 30, 11, 1, 4),
    "c10-w602": ((10,) + M5 + (602,), "identity", None, 100, BF, 24, 30, 8, 2, 4),          # W % F != 0
    "c10-s8-lt-r": ((10,) + M5 + (240,), "tanh", 2, 8, BF, 24, 30, 32, 3, 5),               # S < R
}


def _gen(name, seed):
    geo, act, aff = GEN_CASES[name][:3]
    return _golden5()[1] if geo == "golden" else _gen_model(geo, act, aff, seed=seed)[1]


@pytest.mark.parametrize("name", list(GEN_CASES))
def test_move_generic(name):
    S, dtype, P_A, P_B, n1, n_b, n2 = GEN_CASES[name][3:]
    i = list(GEN_CASES).index(name)
    m = _gen(name, 20 + i)
    run_move(m, m, P_A, P_B, S, dtype, "generic", n1, n_b, n2, seed=30 + i)


@pytest.mark.parametrize("path", ["tensorcore", "generic"])
def test_restart_new_handle(path, tmp_path):
    """a new model object (its own library handle) and a new scorer continue from the state torch.save wrote"""
    if path == "tensorcore":
        mA, mB = _tc_model("mycnn5", 3, 7504, seed=5)[1], _tc_model("mycnn5", 3, 7504, seed=5)[1]
        run_move(mA, mB, 64, 64, 1876, BF, path, 6, 0, 4, seed=50, tmp_path=tmp_path)
    else:
        mA, mB = _golden5()[1], _golden5()[1]
        run_move(mA, mB, 32, 48, 12, F32, path, 12, 0, 5, seed=51, tmp_path=tmp_path)
    assert mA._handle.value != mB._handle.value


# ------------------------------------------------------------------ stride change, weight changes
def test_stride_change_generic():
    """into a scorer with another stride (both multiples of F): its logits are predict()'s on the true windows"""
    _, m = _golden5()
    W, C, P, S, S2 = 120, 10, 24, 12, 40
    a = tskd_b200.SlidingScorer(m, P, S, F32, path="generic")
    ages = tskd_b200.synth.make_ages(P, seed=3).to(DEV)
    stream = _seg(P, C, 11 * S, F32, 60)
    stream[3, 2, 11 * S - 3] = float("nan")                                   # in the tail
    stream[4, 1, 11 * S - 30] = float("inf")
    for t in range(11):
        a.push(stream[:, :, t * S:(t + 1) * S].to(DEV), ages)
    move = [5, 3, 4, 0, 17, 9]
    slots = [2, 7, 0, 11, 8, 1]
    state = a.export(move)
    b = tskd_b200.SlidingScorer(m, 12, S2, F32, path="generic")
    b.push(_seg(12, C, S2, F32, 61).to(DEV), ages[:12])
    b.restore(slots, state)
    own = stream[move]
    for t in range(4):
        seg = _seg(12, C, S2, F32, 62 + t)
        out = b.push(seg.to(DEV), ages[:12])
        own = torch.cat([own, seg[slots]], dim=2)[:, :, -W:]
        want = m.predict(own.to(DEV), ages[:12][torch.tensor(slots, device=DEV)])
        assert _same(out[torch.tensor(slots, device=DEV)].cpu(), want.cpu()), t
        if t == 0:
            assert torch.isnan(out[torch.tensor([3, 4, 5], device=DEV)]).all()  # their windows are not full yet


def _head_only(sd, seed):
    """the state dict with new LSTM, Linear and head weights and the same conv weights"""
    g = torch.Generator().manual_seed(seed)
    return {k: (v if k.startswith("conv") or k.startswith("affine") else v + 0.05 * torch.randn(v.shape, generator=g, dtype=v.dtype))
            for k, v in sd.items()}


@pytest.mark.parametrize("path", ["tensorcore", "generic"])
def test_head_only_weight_update(path):
    """export, new LSTM / Linear / head weights, reset(), restore: the logits are those of an uninterrupted scorer of the
    new model (bit for bit) and of predict() on the true windows (generic: bit for bit; tensor cores: within the
    scorer's grant against the float64 reference)"""
    if path == "tensorcore":
        ref, m = _tc_model("mycnn5", 3, 7504, seed=7)
        sd, W, C, S, dtype, n1 = ref.state_dict(), 7504, 3, 1876, BF, 6
    else:
        sd, m = _golden5()
        W, C, S, dtype, n1 = 120, 10, 12, F32, 12
    P = 40
    ages = tskd_b200.synth.make_ages(P, seed=8).to(DEV)
    a = tskd_b200.SlidingScorer(m, P, S, dtype, path=path)
    new_sd = _head_only(dict(sd), 9)
    m_new = _tc_model("mycnn5", 3, 7504, seed=7)[1] if path == "tensorcore" else _golden5()[1]
    m_new.load_state_dict(new_sd)
    uninterrupted = tskd_b200.SlidingScorer(m_new, P, S, dtype, path=path)
    stream = _seg(P, C, (n1 + 4) * S, dtype, 70)
    for t in range(n1):
        seg = stream[:, :, t * S:(t + 1) * S].to(DEV)
        a.push(seg, ages)
        uninterrupted.push(seg, ages)
    move = list(range(P))
    state = a.export(move)
    m.load_state_dict(new_sd)
    with pytest.raises(RuntimeError, match="b2cnn error 5"):
        a.push(stream[:, :, :S].to(DEV), ages)                                # stale until reset
    a.reset()
    a.restore(move, state)
    pairs = []
    for t in range(n1, n1 + 4):
        seg = stream[:, :, t * S:(t + 1) * S].to(DEV)
        out, want = a.push(seg, ages), uninterrupted.push(seg, ages)
        assert _same(out.cpu(), want.cpu()), t
        win = stream[:, :, (t + 1) * S - W:(t + 1) * S]
        if path == "generic":
            assert _same(out.cpu(), m.predict(win.to(DEV), ages).cpu()), t
        else:
            ref.load_state_dict(new_sd)
            truth = infer_reference(ref, win, ages.cpu())
            ref32 = infer_reference(ref, win, ages.cpu(), dtype=torch.float32)
            pairs.append((f"z[{t}]", out.clone(), truth["z"], ref32["z"], BETA))
    if pairs:
        check_elems(pairs, "test_head_only_weight_update[tensorcore]")


def test_conv_weights_changed():
    """new conv weights: the import is refused with B2CNN_ESTATE and the scorer is unchanged"""
    ref, m = _tc_model("mycnn5", 3, 7504, seed=11)
    P, S = 24, 1876
    ages = tskd_b200.synth.make_ages(P, seed=12).to(DEV)
    a = tskd_b200.SlidingScorer(m, P, S)
    for t in range(5):
        a.push(_seg(P, 3, S, BF, 80 + t).to(DEV), ages)
    state = a.export(range(P))
    sd = dict(ref.state_dict())
    sd["conv1.weight"] = sd["conv1.weight"] * 1.01
    m.load_state_dict(sd)
    a.reset()
    twin = tskd_b200.SlidingScorer(m, P, S)
    with pytest.raises(RuntimeError, match="b2cnn error 5"):
        a.restore(range(P), state)
    for t in range(5):
        seg = _seg(P, 3, S, BF, 90 + t).to(DEV)
        oa, ot = a.push(seg, ages), twin.push(seg, ages)
        assert (oa is None) == (ot is None) and (oa is None or _same(oa, ot)), t


# ------------------------------------------------------------------ errors
def _import_rc(sc, idx, state, feats=True, tails=True, seen=None, ws_bytes=None, **hdr_over):
    """b2cnn_slide_import through the C ABI: its return code"""
    lib = sc._lib
    hdr = capi.SlideStateHeader(**{n: int(state[n]) for n in sc.STATE_HEADER})
    for n, v in hdr_over.items():
        setattr(hdr, n, v)
    k = len(idx)
    arr = (ctypes.c_int32 * max(k, 1))(*idx)
    seen = (state["seen"] if seen is None else seen).contiguous()
    nb = int(lib.b2cnn_slide_state_workspace_bytes(sc._s, k))
    ws = torch.empty(max(nb, 1), dtype=torch.uint8, device=DEV)
    rc = lib.b2cnn_slide_import(sc._s, arr, k, ctypes.byref(hdr), state["features"].data_ptr() if feats else None,
                                state["tail"].data_ptr() if tails else None, seen.data_ptr(), ws.data_ptr(),
                                nb if ws_bytes is None else ws_bytes, torch.cuda.current_stream().cuda_stream)
    torch.cuda.synchronize()
    return rc


def test_errors_leave_the_scorer_unchanged():
    _, m = _tc_model("mycnn5", 3, 7504, seed=13)
    P, S = 20, 1876
    ages = tskd_b200.synth.make_ages(P, seed=14).to(DEV)
    a = tskd_b200.SlidingScorer(m, P, S)
    b, twin = tskd_b200.SlidingScorer(m, P, S), tskd_b200.SlidingScorer(m, P, S)
    for t in range(5):
        seg = _seg(P, 3, S, BF, 100 + t).to(DEV)
        a.push(seg, ages)
        b.push(seg.flip(0), ages)
        twin.push(seg.flip(0), ages)
    idx = [3, 1, 4]
    state = a.export(idx)
    f0, s0 = b.features(), b.samples_seen
    EINVAL, ESTATE = capi.EINVAL, capi.ESTATE
    cases = [
        (EINVAL, dict(magic=0x12345678)), (EINVAL, dict(version=2)), (EINVAL, dict(path=capi.PATH_GENERIC)),
        (EINVAL, dict(dtype=capi.DTYPE_F32)), (EINVAL, dict(in_channels=2)), (EINVAL, dict(window=7500)),
        (EINVAL, dict(lstm_input=1870)), (EINVAL, dict(feature_stride=16)), (EINVAL, dict(tail_len=16)),
        (ESTATE, dict(frontend_digest=int(state["frontend_digest"]) ^ 1)),
    ]
    for want, over in cases:
        assert _import_rc(b, [0, 2, 5], state, **over) == want, over
    assert _import_rc(b, [0, 2, 20], state) == EINVAL                           # out of range
    assert _import_rc(b, [0, 2, 0], state) == EINVAL                            # listed twice
    assert _import_rc(b, [0, 2, 5], state, feats=False) == EINVAL               # null arrays with n > 0
    assert _import_rc(b, [0, 2, 5], state, tails=False) == EINVAL
    assert _import_rc(b, [0, 2, 5], state, seen=torch.tensor([9000, -2, 0])) == EINVAL
    assert _import_rc(b, [0, 2, 5], state, ws_bytes=0) == ESTATE                # workspace too small
    with pytest.raises(ValueError):
        b.restore([0, 2], state)                                                # three rows for two patients
    assert _import_rc(b, [], {**state, "features": state["features"][:0], "tail": state["tail"][:0],
                              "seen": state["seen"][:0]}) == capi.OK            # k = 0: a no-op
    assert _same(b.features(), f0) and torch.equal(b.samples_seen, s0)
    empty = a.export([])
    assert empty["features"].shape == (0, m.arch.l_out) and empty["seen"].shape == (0,)
    b.restore([], empty)
    for t in range(4):
        seg = _seg(P, 3, S, BF, 110 + t).to(DEV)
        ob, ot = b.push(seg, ages), twin.push(seg, ages)
        assert _same(ob, ot), t                                                 # no NaN mask: the lifecycle stayed off
    assert _import_rc(b, [0, 2, 5], state) == capi.OK


def test_stale_scorer_refuses_both():
    ref, m = _tc_model("mycnn5", 3, 7504, seed=15)
    sc = tskd_b200.SlidingScorer(m, 8, 1876)
    for t in range(5):
        sc.push(_seg(8, 3, 1876, BF, 120 + t).to(DEV))
    state = sc.export([0, 1])
    m.load_state_dict(_head_only(dict(ref.state_dict()), 16))
    with pytest.raises(RuntimeError, match="b2cnn error 5"):
        sc.export([0])
    with pytest.raises(RuntimeError, match="b2cnn error 5"):
        sc.restore([0, 1], state)
    sc.reset()
    sc.restore([0, 1], state)


def test_move_between_two_gpus():
    if torch.cuda.device_count() < 2:
        pytest.skip("needs two GPUs")
    ref, m0 = _tc_model("mycnn5", 3, 7504, seed=17)
    m1 = tskd_b200.B200MyCNN(m0.arch, has_out12=ref.arch.has_out12).to("cuda:1")
    m1.load_state_dict(ref.state_dict())
    P, S = 16, 1876
    a = tskd_b200.SlidingScorer(m0, P, S)
    b = tskd_b200.SlidingScorer(m1, P, S)
    assert b.device == torch.device("cuda", 1)
    for t in range(5):
        a.push(_seg(P, 3, S, BF, 130 + t).to(DEV))
    idx = [2, 9, 5]
    b.restore([0, 1, 2], a.export(idx))
    for t in range(3):
        seg = _seg(P, 3, S, BF, 140 + t)
        oa = a.push(seg.to(DEV))
        ob = b.push(seg[[2, 9, 5, 3, 4, 6, 7, 8, 0, 1, 10, 11, 12, 13, 14, 15]].to("cuda:1"))
        assert _same(oa[torch.tensor(idx, device=DEV)].cpu(), ob[:3].cpu()), t


