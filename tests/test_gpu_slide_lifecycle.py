"""GPU: the per-patient lifecycle of the sliding-window scorer (SlidingScorer.admit / discharge / samples_seen,
b2cnn_slide_admit / _discharge / _samples_seen, csrc/b2cnn_slide.cu).

Every patient's stream is simulated on the host: after a push, a patient with samples_seen >= W is scored on the last W
samples of (its history | the pushes since its admission), judged element by element against the float64 reference of
oracle/infer_ref.py with the grants of tests/test_gpu_infer_elem.py (BETA for the scorer's logits, TC_FEATURES_BETA for
its features); every other patient must be NaN, and the push returns None exactly when no patient is valid."""
import ctypes
import os
from dataclasses import replace

import numpy as np
import pytest
import torch

import tskd_b200
from oracle import mycnn_torch as O
from oracle.infer_ref import TC_FEATURES_BETA, infer_reference
from oracle.train_ref import BETA, check_elems
from tskd_b200 import capi

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
BF, F32 = torch.bfloat16, torch.float32
BETA_SLIDE_LOGITS = BETA
BETA_SLIDE_FEATURES = TC_FEATURES_BETA


def _model(kind, W, seed):
    ref = O.make_ref(O.stretched(O.ARCHS[kind], 3, W), seed=seed)
    arch = replace(tskd_b200.ARCH_PRESETS[kind].with_shape(3, W), age_coef=ref.arch.age_coef)
    m = tskd_b200.B200MyCNN(arch, has_out12=ref.arch.has_out12).to(DEV)
    m.load_state_dict(ref.state_dict())
    return ref, m


def _R(kind):
    return 24 if kind == "mycnn5" else 16


class Ward:
    """A scorer and the host-side truth of its P streams: own[p] holds the last W samples of p's stream (CPU)."""

    def __init__(self, ref, m, P, S, dtype, seed):
        self.ref, self.m, self.P, self.S, self.dtype = ref, m, P, S, dtype
        self.W = m.arch.window
        self.sc = tskd_b200.SlidingScorer(m, P, S, dtype)
        self.own = [torch.empty(3, 0, dtype=dtype) for _ in range(P)]
        self.seen = np.zeros(P, dtype=np.int64)
        self.age = tskd_b200.synth.make_ages(P, seed=seed)
        self.age_dev = self.age.to(DEV)
        self.n = 0

    def admit(self, idx, hist=None):
        """hist: CPU [k, 3, H] or None"""
        self.sc.admit(idx, hist.to(DEV) if hist is not None else None)
        for j, p in enumerate(idx):
            self.own[p] = hist[j].clone() if hist is not None else torch.empty(3, 0, dtype=self.dtype)
            self.seen[p] = hist.shape[2] if hist is not None else 0

    def discharge(self, idx):
        self.sc.discharge(idx)
        self.seen[list(idx)] = -1

    def push(self, seg):
        """seg: [P, 3, S] on the device; returns (out or None, valid mask)"""
        out = self.sc.push(seg, self.age_dev)
        self.n += 1
        segc = seg.cpu()
        for p in range(self.P):
            if self.seen[p] >= 0:
                self.own[p] = torch.cat([self.own[p], segc[p]], dim=1)[:, -self.W:]
                self.seen[p] += self.S
        valid = self.seen >= self.W
        if not valid.any():
            assert out is None, self.n
        else:
            assert out is not None, self.n
            assert torch.isnan(out[torch.from_numpy(~valid).to(DEV)]).all(), self.n
            # a valid patient is NaN exactly when its window holds a NaN sample (inf gives a finite logit)
            vi = np.flatnonzero(valid)
            want_nan = torch.tensor([bool(torch.isnan(self.own[p]).any()) for p in vi])
            assert torch.equal(torch.isnan(out[torch.from_numpy(vi).to(DEV)]).cpu(), want_nan), self.n
            assert self.sc.window_index == self.n - (-(-self.W // self.S))
        assert np.array_equal(self.sc.samples_seen.cpu().numpy(), self.seen), self.n
        return out, valid

    def judge(self, out, rows, tag, features=False):
        """(name, got, truth, ref32, beta) pairs for the given valid patients"""
        rows = sorted(rows)
        win = torch.stack([self.own[p] for p in rows])
        assert win.shape[2] == self.W
        age = self.age[rows]
        truth, ref32 = infer_reference(self.ref, win, age), infer_reference(self.ref, win, age, dtype=torch.float32)
        pairs = [(f"z[{tag}]", out[rows].clone(), truth["z"], ref32["z"], BETA_SLIDE_LOGITS)]
        if features:
            f = self.sc.features()
            pairs.append((f"features[{tag}]", f[rows].clone(), truth["features"], ref32["features"], BETA_SLIDE_FEATURES))
            bad = torch.from_numpy(self.seen < self.W).to(DEV)
            assert torch.isnan(f[bad]).all() and not torch.isnan(f[~bad]).all(dim=1).any()
        return pairs, truth["z"]


def _same(a, b):
    """bit-identical, NaN for NaN (None for None)"""
    if a is None or b is None:
        return a is None and b is None
    na, nb = torch.isnan(a), torch.isnan(b)
    return torch.equal(na, nb) and torch.equal(a[~na], b[~nb])


def _check(pairs):
    check_elems(pairs, os.environ.get("PYTEST_CURRENT_TEST", "").split(" ")[0])


def _hist(k, H, dtype, seed):
    return tskd_b200.synth.make_windows(k, 3, H, "normal", seed=seed, dtype=dtype)


def _bad(h, R):
    """NaN at the first sample, +inf mid-history, -inf and NaN in the last R samples, in the first four rows"""
    H = h.shape[2]
    h[0, 0, 0] = float("nan")
    h[1, 1, H // 2] = float("inf")
    h[2, 2, H - R // 2] = float("-inf")
    h[3, 0, H - 3] = float("nan")


def _stream(P, n_push, S, dtype, seed):
    return tskd_b200.synth.make_windows(P, 3, n_push * S, "normal", seed=seed, dtype=dtype).to(DEV)


# ------------------------------------------------------------------ untouched patients
def test_untouched_patients_bit_identical():
    """one scorer admits, backfills and discharges an unsorted, non-contiguous subset; every other patient's logits
    are bit-identical to a scorer that never used the lifecycle, at every push"""
    W, S, P, n_push = 7504, 1876, 300, 9
    ref, m = _model("mycnn5", W, 1)
    stream = _stream(P, n_push, S, BF, 1)
    ctl = tskd_b200.SlidingScorer(m, P, S)
    sc = tskd_b200.SlidingScorer(m, P, S)
    age = tskd_b200.synth.make_ages(P, seed=1).to(DEV)
    g = torch.Generator().manual_seed(1)
    perm = torch.randperm(P, generator=g).tolist()
    a0, a2, d3, a5 = perm[:140], perm[140:150], perm[150:160], perm[160:170]
    touched = set(perm[:170])
    keep = torch.tensor([p for p in range(P) if p not in touched], device=DEV)
    plan = {0: [("admit", a0, W)], 2: [("admit", a2, 0)], 3: [("discharge", d3)], 5: [("admit", a5, W - S)]}
    for n in range(n_push):
        for act in plan.get(n, []):
            if act[0] == "admit":
                sc.admit(act[1], _hist(len(act[1]), act[2], BF, 100 + n).to(DEV) if act[2] else None)
            else:
                sc.discharge(act[1])
        seg = stream[:, :, n * S:(n + 1) * S]
        want, got = ctl.push(seg, age), sc.push(seg, age)
        assert got is not None                                   # the patients admitted with W samples score at once
        if want is None:
            assert torch.isnan(got[keep]).all()
        else:
            assert torch.equal(got[keep], want[keep]), n
    assert torch.equal(ctl.samples_seen, torch.full((P,), n_push * S, device=DEV))


# ------------------------------------------------------------------ backfilled and staggered admissions
GEOMS = [("mycnn5", BF, 7504, 1876), ("mycnn5", F32, 7502, 1876), ("mycnn3", BF, 7502, 1876), ("mycnn3", F32, 7504, 1876)]


@pytest.mark.parametrize("kind,dtype,W,S", GEOMS, ids=[f"{k}-{'bf16' if d == BF else 'f32'}-w{w}" for k, d, w, _ in GEOMS])
def test_backfilled_and_staggered_admissions(kind, dtype, W, S):
    """P = 300.  Before any push: 130 patients with W samples (tensor cores across a 128-window tile, NaN/inf in four
    histories), 6 with R - 1 (tail only), 8 with 100 (exact kernel only).  Before push 2 (the first global window
    is at push 4): W - S and S + R.  Before push 6: W - 3 (phase psi = 1), S + R, and none (staggered).  Every patient
    scores from exactly the push at which samples_seen reaches W, on its own stream."""
    P, R = 300, _R(kind)
    n_push = 11
    ref, m = _model(kind, W, 7)
    wd = Ward(ref, m, P, S, dtype, 7)
    stream = _stream(P, n_push, S, dtype, 7)
    perm = torch.randperm(P, generator=torch.Generator().manual_seed(7)).tolist()
    groups, at = {}, 0

    def take(k):
        nonlocal at
        at += k
        return perm[at - k:at]

    plan = {0: [("A", 130, W), ("B", 6, R - 1), ("C", 8, 100)],
            1: [("D", 10, W - S), ("E", 4, S + R)],
            5: [("F", 130, W - 3), ("G", 4, S + R), ("H", 6, 0)]}      # 298 of the 300 patients
    pairs, inf_rows, last = [], [], None
    for n in range(n_push):
        for name, k, H in plan.get(n, []):
            idx = groups[name] = take(k)
            h = _hist(k, H, dtype, 1000 + at) if H else None
            if name in ("A", "F"):
                _bad(h, R)
                inf_rows += [idx[1], idx[2]]
            wd.admit(idx, h)
        out, valid = wd.push(stream[:, :, n * S:(n + 1) * S])
        if out is None:
            continue
        last = out
        # judge: the first 8 of each valid group, scratch columns 126-129 of the 130-patient groups, the untouched two
        rows = {p for g_, idx in groups.items() for p in idx[:8] + (idx[126:130] if len(idx) > 128 else []) if valid[p]}
        rows |= {p for p in perm[at:at + 8] if valid[p]}
        if rows:
            feats = n in (0, 4, 9)
            ps, z = wd.judge(out, rows, n, features=feats)
            pairs += ps
    # +-inf samples in a history give finite logits (the NaN pattern itself is judged against the reference above)
    assert not torch.isnan(last[inf_rows]).any()
    assert all(wd.seen[groups[g_]].min() >= W for g_ in groups)     # every group reached its first score in this run
    _check(pairs)


# ------------------------------------------------------------------ history views
@pytest.mark.parametrize("H", [7504, 7501])
def test_aligned_and_unaligned_history_views(H):
    """row-padded and one-sample-offset views of the histories give exactly the contiguous history's scores"""
    W, S, P, k = 7504, 1876, 200, 150
    _, m = _model("mycnn5", W, 3)
    stream = _stream(P, 3, S, BF, 3)
    hist = _hist(k, H, BF, 3).to(DEV)
    idx = torch.randperm(P, generator=torch.Generator().manual_seed(3))[:k].tolist()
    views = {"contiguous": hist}
    padded = torch.empty(k, 3, H + 13, dtype=BF, device=DEV)
    padded[:, :, :H] = hist
    views["padded"] = padded[:, :, :H]
    off = torch.empty(k, 3, H + 8, dtype=BF, device=DEV)
    off[:, :, 1:H + 1] = hist
    views["offset"] = off[:, :, 1:H + 1]
    outs = {}
    for name, v in views.items():
        sc = tskd_b200.SlidingScorer(m, P, S)
        sc.push(stream[:, :, :S])
        sc.admit(idx, v)
        outs[name] = [sc.push(stream[:, :, n * S:(n + 1) * S]) for n in (1, 2)]
        sc.close()
    assert views["padded"].stride(1) == H + 13 and not views["offset"].is_contiguous()
    for name in ("padded", "offset"):
        assert all(_same(a, b) for a, b in zip(outs[name], outs["contiguous"])), name
    assert not torch.isnan(outs["contiguous"][0][idx]).any()     # H + S >= W: scored at the first push after admission


# ------------------------------------------------------------------ full size
def test_full_size_backfilled_admission():
    """W = 75000, S = 7500, P = 300: 200 patients admitted with full histories before push 4 score at push 4"""
    W, S, P, k = 75000, 7500, 300, 200
    ref, m = _model("mycnn5", W, 5)
    wd = Ward(ref, m, P, S, BF, 5)
    stream = _stream(P, 4, S, BF, 5)
    idx = torch.randperm(P, generator=torch.Generator().manual_seed(5))[:k].tolist()
    for n in range(3):
        out, _ = wd.push(stream[:, :, n * S:(n + 1) * S])
        assert out is None
    wd.admit(idx, _hist(k, W, BF, 55))
    out, valid = wd.push(stream[:, :, 3 * S:4 * S])
    assert valid.sum() == k and out is not None
    rows = [idx[i] for i in (0, 1, 2, 126, 127, 128, 129, 199)]
    pairs, _ = wd.judge(out, rows, 4, features=True)
    _check(pairs)


# ------------------------------------------------------------------ features() before the next push
def _features_now(wd, rows, tag):
    """features() as they stand (no push since the last admission): NaN rows for patients without a complete window,
    the listed valid rows judged against their windows"""
    f = wd.sc.features()
    bad = torch.from_numpy(wd.seen < wd.W).to(DEV)
    assert torch.isnan(f[bad]).all(), tag
    rows = sorted(rows)
    win = torch.stack([wd.own[p] for p in rows])
    assert win.shape[2] == wd.W
    truth, ref32 = infer_reference(wd.ref, win, wd.age[rows]), infer_reference(wd.ref, win, wd.age[rows], dtype=torch.float32)
    return [(f"features[{tag}]", f[rows].clone(), truth["features"], ref32["features"], BETA_SLIDE_FEATURES)]


@pytest.mark.parametrize("kind,dtype,W,S", [("mycnn5", BF, 7504, 1876), ("mycnn3", F32, 7502, 1876)])
def test_features_right_after_full_history_admission(kind, dtype, W, S):
    """A patient admitted with W samples has a complete window at once: features() before the next push returns the
    history's window, including the current window's first S / 4 features, which no later window holds.  Before any
    push (133 patients, across a 128-window tile, on a fresh ring), and after five pushes over ring columns that held
    other streams (8 patients, judged next to valid patients that were not readmitted)."""
    P = 140
    ref, m = _model(kind, W, 13)
    wd = Ward(ref, m, P, S, dtype, 13)
    stream = _stream(P, 5, S, dtype, 13)
    perm = torch.randperm(P, generator=torch.Generator().manual_seed(13)).tolist()
    first = perm[:133]
    wd.admit(first, _hist(133, W, dtype, 130))
    pairs = _features_now(wd, [first[i] for i in (0, 1, 126, 127, 128, 129, 132)], "admitted before any push")
    for n in range(5):
        wd.push(stream[:, :, n * S:(n + 1) * S])
    again = perm[100:105] + perm[135:138]             # 5 over earlier admissions, 3 over untouched streams
    wd.admit(again, _hist(len(again), W, dtype, 131))
    pairs += _features_now(wd, again + [perm[0], perm[138]], "readmitted after five pushes")
    _check(pairs)


# ------------------------------------------------------------------ lifecycle order
def test_discharge_readmit_reset_and_replay():
    W, S, P = 7504, 1876, 40
    ref, m = _model("mycnn3", W, 9)
    stream = _stream(P, 8, S, BF, 9)
    hist = _hist(6, W, BF, 9)

    def scenario():
        wd = Ward(ref, m, P, S, BF, 9)
        outs, pairs = [], []
        for n in range(8):
            if n == 1:
                wd.discharge([3, 17, 30])
            if n == 2:
                wd.admit([17, 4, 30, 9, 22, 0], hist)            # 17 and 30 readmitted, 4 and 9 restarted
            out, valid = wd.push(stream[:, :, n * S:(n + 1) * S])
            outs.append(None if out is None else out.clone())
            if out is not None:
                pairs += wd.judge(out, [p for p in (0, 4, 9, 17, 22, 30, 1) if valid[p]], n)[0]
            assert valid[3] == False                              # noqa: E712  (discharged for good)
        return wd, outs, pairs

    wd, first, pairs = scenario()
    _check(pairs)
    assert first[2] is not None and not torch.isnan(first[2][[17, 4, 30]]).any() and torch.isnan(first[2][1])
    # reset: every patient admitted with an empty stream, the masking off again (as a fresh scorer)
    wd.sc.reset()
    assert torch.equal(wd.sc.samples_seen, torch.zeros(P, dtype=torch.int64, device=DEV))
    fresh = tskd_b200.SlidingScorer(m, P, S)
    for n in range(8):
        a, b = wd.sc.push(stream[:, :, n * S:(n + 1) * S], wd.age_dev), fresh.push(stream[:, :, n * S:(n + 1) * S], wd.age_dev)
        assert _same(a, b), n
    _, again, _ = scenario()
    assert all(_same(x, y) for x, y in zip(first, again))


# ------------------------------------------------------------------ errors
def test_lifecycle_errors():
    W, S, P = 7504, 1876, 8
    _, m = _model("mycnn5", W, 2)
    sc = tskd_b200.SlidingScorer(m, P, S)
    lib, s = sc._lib, sc._s
    st = torch.cuda.current_stream().cuda_stream

    def admit(idx, H, dtype=capi.DTYPE_BF16, hist=True, pitch=None):
        arr = (ctypes.c_int32 * len(idx))(*idx)
        n = lib.b2cnn_slide_admit_workspace_bytes(s, len(idx), max(H, 0))
        ws = torch.empty(max(n, 1) + (1 << 20), dtype=torch.uint8, device=DEV)
        h = torch.zeros(len(idx), 3, max(H, 1) + 8, dtype=BF, device=DEV)
        return lib.b2cnn_slide_admit(s, arr, len(idx), h.data_ptr() if hist else None, H, h.shape[2] if pitch is None else pitch,
                                     dtype, ws.data_ptr(), ws.numel(), st)

    assert admit([0, 1], 100) == capi.OK
    assert admit([0, 8], 100) == capi.EINVAL            # out of range
    assert admit([-1], 100) == capi.EINVAL
    assert admit([2, 5, 2], 100) == capi.EINVAL         # duplicate
    assert admit([2], W + 4) == capi.EINVAL             # H > W
    assert admit([2], -4) == capi.EINVAL
    assert admit([2], 100, hist=False) == capi.EINVAL   # null history with H > 0
    assert admit([2], 100, dtype=capi.DTYPE_F32) == capi.EINVAL
    assert admit([2], 100, pitch=50) == capi.EINVAL     # pitch < H
    assert lib.b2cnn_slide_admit_workspace_bytes(s, 2, W + 4) < 0
    arr = (ctypes.c_int32 * 2)(3, 3)
    assert lib.b2cnn_slide_discharge(s, arr, 2, st) == capi.EINVAL
    with pytest.raises(ValueError):
        sc.admit([1, 1])
    with pytest.raises(ValueError):
        sc.admit([1], torch.zeros(1, 3, W + 4, dtype=BF, device=DEV))
    ref2 = O.make_ref(O.stretched(O.ARCHS["mycnn5"], 3, W), seed=4)
    m.load_state_dict(ref2.state_dict())
    m._ensure_handle()
    assert admit([0], 100) == capi.ESTATE               # new weights without a reset
    with pytest.raises(RuntimeError, match="error 5"):
        sc.admit([0], torch.zeros(1, 3, 100, dtype=BF, device=DEV))
    sc.reset()
    assert admit([0], 100) == capi.OK
    # no patient with a complete window: features() refuses, push returns None
    sc.discharge(list(range(P)))
    assert sc.push(torch.zeros(P, 3, S, dtype=BF, device=DEV)) is None
    with pytest.raises(RuntimeError, match="error 5"):
        sc.features()
