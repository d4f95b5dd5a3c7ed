"""GPU: the tensor-core SlidingScorer element by element against the float64 reference of the explicit windows, at the
edges of its index arithmetic (the case tables and the Python mirror of tests/slide_lattice.py; which edge each table
reaches is shown on the CPU by tests/test_slide_lattice_host.py):

- every window phase phi = (-W) mod 4 in both geometries and dtypes, with +-inf / NaN at a seam sample, among a
  segment's first phi samples and among the last (W - R) % 4 samples of a window, which no feature covers;
- pushes of Q = 31, 32 and 33 features at every phase (the exact / tensor-core split), a flagged recompute at Q = 32;
- long runs at W = 1533, S = 164 that reach every split point of the projection's ring wrap, at the default position
  ranges and at B2CNN_TC_TILES = 7;
- the smallest windows (L = 32);
- admissions at odd phase on both sides of the split, with staging shifts and an unaligned history view;
- extra heads at odd phase, each row judged against its own model, and an export / restore into another P;
- pushes staged for their pointer or pitch alone, bit-identical to contiguous ones.

Every emitted push is judged with oracle/train_ref.py::check_elems at the grants of tests/test_gpu_infer_elem.py: BETA
for the logits, TC_FEATURES_BETA for features(); NaN exactly where the truth has NaN."""
import os
from dataclasses import replace

import numpy as np
import pytest
import torch

import slide_lattice as M
import tskd_b200
from oracle import mycnn_torch as O
from oracle.infer_ref import TC_FEATURES_BETA, infer_reference
from oracle.train_ref import BETA, check_elems
from test_gpu_infer_elem import _model
from test_gpu_slide_heads import _head_sd
from test_gpu_slide_lifecycle import Ward

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
DT = {"bf16": torch.bfloat16, "f32": torch.float32}


def _check(pairs):
    check_elems(pairs, os.environ.get("PYTEST_CURRENT_TEST", "").split(" ")[0])


def _pair(c, seed):
    ref = O.make_ref(O.stretched(O.ARCHS[c.kind], c.C, c.W), seed=seed)
    return ref, _model(ref)


def _stream(c, n_push, seed):
    return tskd_b200.synth.make_windows(c.P, c.C, n_push * c.S, "normal", seed=seed, dtype=DT[c.dtype])


def _scorer(m, c, P=None):
    sc = tskd_b200.SlidingScorer(m, P or c.P, c.S, DT[c.dtype])
    assert sc.path == "tensorcore"
    return sc


def _judge(tag, got, refs, win, age, feats=None):
    """row i of got ([P] or [1 + K, P]) against refs[i] on the windows; features against refs[0]"""
    rows = got if got.dim() == 2 else got.unsqueeze(0)
    assert rows.shape[0] == len(refs)
    pairs = []
    for i, r in enumerate(refs):
        t, t32 = infer_reference(r, win, age), infer_reference(r, win, age, dtype=torch.float32)
        pairs.append((f"z{i}[{tag}]", rows[i].clone(), t["z"], t32["z"], BETA))
        if i == 0 and feats is not None:
            pairs.append((f"features[{tag}]", feats, t["features"], t32["features"], TC_FEATURES_BETA))
    return pairs


def _replay(sc, refs, stream, age, S, pushes, first=1, skipped=0, heads=False, seg_of=None):
    """push stream segments `first` .. `pushes` (stream push n is the scorer's push n - skipped); every emitted push
    judged.  Returns the (name, got, truth, ref32, beta) pairs and the emitted outputs by stream push."""
    W = refs[0].arch.window
    n0 = M.n0_of(W, S)
    sd, ad = stream.to(DEV), age.to(DEV)
    pairs, outs = [], {}
    for n in range(first, pushes + 1):
        seg = seg_of(n) if seg_of else sd[:, :, (n - 1) * S:n * S]
        got = sc.push(seg, ad, heads=heads)
        if n * S < W:
            assert got is None, n
            continue
        assert got is not None and sc.window_index == n - skipped - n0, (n, sc.window_index)
        outs[n] = got.clone()
        pairs += _judge(n, got, refs, stream[:, :, n * S - W:n * S], age, sc.features())
    return pairs, outs


# ------------------------------------------------------------------ phase x geometry x dtype
@pytest.mark.parametrize("name", sorted(M.PHASE_CASES))
def test_every_phase(name):
    c = M.PHASE_CASES[name]
    seed = 200 + sorted(M.PHASE_CASES).index(name)
    n0 = M.n0_of(c.W, c.S)
    n_push = n0 + 3
    ref, m = _pair(c, seed)
    stream = _stream(c, n_push, seed)
    for p, ch, t, v, _ in M.inject_sites(c):
        stream[p, ch, t] = v
    age = tskd_b200.synth.make_ages(c.P, seed=seed)
    sc = _scorer(m, c)
    pairs, outs = _replay(sc, [ref], stream, age, c.S, n_push)
    assert sorted(outs) == list(range(n0, n_push + 1))
    p = M.inject_sites(c)[0][0]
    # the +-inf samples leave window n0 finite; the NaN is covered from window n0 + 2 on
    assert not torch.isnan(outs[n0][p]) and torch.isnan(outs[n0 + 2][p])
    assert bool(torch.isnan(outs[n0 + 1][p])) == (M.phi_of(c.W) == 0)
    sc.close()
    _check(pairs)


# ------------------------------------------------------------------ the exact / tensor-core split
@pytest.mark.parametrize("name", sorted(M.Q_CASES))
def test_q_split(name):
    c = M.Q_CASES[name]
    seed = 300 + sorted(M.Q_CASES).index(name)
    n0 = M.n0_of(c.W, c.S)
    n_push = n0 + 2
    ref, m = _pair(c, seed)
    stream = _stream(c, n_push, seed)
    q = M.push_Q(c.kind, c.W, c.S)
    if q == 32:                                       # main features of pushes n0 and n0 + 1: flagged, recomputed
        stream[5, 0, (n0 - 1) * c.S + c.S // 2] = float("nan")
        stream[6, c.C - 1, n0 * c.S + c.S // 2] = float("inf")
    age = tskd_b200.synth.make_ages(c.P, seed=seed)
    sc = _scorer(m, c)
    pairs, outs = _replay(sc, [ref], stream, age, c.S, n_push)
    assert len(outs) == 3
    if q == 32:
        assert torch.isnan(outs[n0][5]) and not torch.isnan(outs[n_push][6])
    sc.close()
    _check(pairs)


# ------------------------------------------------------------------ long runs over every projection wrap
@pytest.mark.parametrize("name", sorted(M.LONG_CASES))
def test_long_run(monkeypatch, name):
    c, tiles = M.LONG_CASES[name]
    if tiles is not None:
        monkeypatch.setenv("B2CNN_TC_TILES", str(tiles))   # read by tc_prepare when the weights are set
    seed = 400 + sorted(M.LONG_CASES).index(name)
    n_push = M.long_pushes()
    ref, m = _pair(c, seed)
    stream = _stream(c, n_push, seed)
    age = tskd_b200.synth.make_ages(c.P, seed=seed)
    sc = _scorer(m, c)
    pairs, outs = _replay(sc, [ref], stream, age, c.S, n_push)
    assert len(outs) == n_push - M.n0_of(c.W, c.S) + 1
    sc.close()
    _check(pairs)


# ------------------------------------------------------------------ the smallest window
@pytest.mark.parametrize("name", sorted(M.SMALL_CASES))
def test_smallest_window(name):
    c = M.SMALL_CASES[name]
    seed = 500 + sorted(M.SMALL_CASES).index(name)
    n_push = M.n0_of(c.W, c.S) + 3
    ref, m = _pair(c, seed)
    stream = _stream(c, n_push, seed)
    age = tskd_b200.synth.make_ages(c.P, seed=seed)
    sc = _scorer(m, c)
    pairs, outs = _replay(sc, [ref], stream, age, c.S, n_push)
    assert len(outs) == 4
    sc.close()
    _check(pairs)


# ------------------------------------------------------------------ admissions at odd phase
def _admit(wd, idx, hist, unaligned):
    """hist: CPU [k, C, H] or None; unaligned: admitted through a view one element past an aligned pointer"""
    if not unaligned:
        wd.admit(idx, hist)
        return
    k, C, H = hist.shape
    buf = torch.zeros(k, C, H + 8, dtype=hist.dtype, device=DEV)
    buf[:, :, 1:H + 1] = hist.to(DEV)
    view = buf[:, :, 1:H + 1]
    assert view.data_ptr() % 16 != 0 and not view.is_contiguous()
    wd.sc.admit(idx, view)
    for j, p in enumerate(idx):
        wd.own[p] = hist[j].clone()
        wd.seen[p] = H


@pytest.mark.parametrize("name", sorted(M.ADMIT_CASES))
def test_admissions_at_odd_phase(name):
    """every history length of the table admitted before push 1 and before push 4, 4 patients each; every valid
    patient judged at every push"""
    c = M.ADMIT_CASES[name]
    seed = 600 + sorted(M.ADMIT_CASES).index(name)
    dtype = DT[c.dtype]
    ref, m = _pair(c, seed)
    wd = Ward(ref, m, c.P, c.S, dtype, seed)
    assert wd.sc.path == "tensorcore"
    stream = _stream(c, M.ADMIT_PUSHES, seed).to(DEV)
    perm = torch.randperm(c.P, generator=torch.Generator().manual_seed(seed)).tolist()
    hs = M.admit_histories(c)
    groups, at, pairs = {}, 0, []
    for n in range(M.ADMIT_PUSHES):
        if n in M.ADMIT_AT:
            for gname, H, unaligned in hs:
                idx = perm[at:at + 4]
                at += 4
                groups[(n, gname)] = idx
                h = tskd_b200.synth.make_windows(4, c.C, H, "normal", seed=seed * 100 + at, dtype=dtype) if H else None
                if gname == "W":
                    h[0, 1, H // 2] = float("inf")          # flagged by the tensor cores, recomputed exactly
                if gname == "W-3":
                    h[1, 0, H // 3] = float("nan")          # in the first windows only
                _admit(wd, idx, h, unaligned)
        out, valid = wd.push(stream[:, :, n * c.S:(n + 1) * c.S])
        if out is None:
            continue
        rows = np.flatnonzero(valid).tolist()
        ps, _ = wd.judge(out, rows, n, features=True)
        pairs += ps
    assert all(wd.seen[idx].min() >= c.W for idx in groups.values())       # every group was scored
    _check(pairs)


# ------------------------------------------------------------------ heads and state at odd phase
@pytest.mark.parametrize("K", [2, 3])
def test_heads_export_restore_at_odd_phase(K):
    """K = 2 (one head pair) and 3 (a padded pair); each row judged against its own model.  Exported after a push whose
    projection wraps, restored into a scorer of another P (with the heads), both scorers pushed on and judged."""
    c = M.HEADS_CASE
    seed = 700 + K
    ref, m = _pair(c, seed)
    sd = dict(ref.state_dict())
    refs, heads = [ref], []
    for i in range(K):
        h = O.RefMyCNN(replace(ref.arch, age_coef=1e-3 * (i + 1)))
        h.load_state_dict(_head_sd(sd, seed * 10 + i))
        h.eval()
        refs.append(h)
        heads.append(_model(h))
    stream = _stream(c, M.HEADS_PUSHES, seed)
    age = tskd_b200.synth.make_ages(c.P, seed=seed)
    sc = _scorer(m, c)
    sc.set_heads(heads)
    pairs, _ = _replay(sc, refs, stream, age, c.S, M.EXPORT_AT, heads=True)
    idx = torch.randperm(c.P, generator=torch.Generator().manual_seed(seed))[:M.RESTORE_P]
    state = sc.export(idx)
    sc2 = _scorer(m, c, M.RESTORE_P)
    sc2.set_heads(heads)
    sc2.restore(range(M.RESTORE_P), state)
    ps, _ = _replay(sc, refs, stream, age, c.S, M.HEADS_PUSHES, first=M.EXPORT_AT + 1, heads=True)
    pairs += ps
    # the restored scorer's window_index counts its own pushes, from 1 at stream push EXPORT_AT + 1
    ps, outs = _replay(sc2, refs, stream[idx], age[idx], c.S, M.HEADS_PUSHES, first=M.EXPORT_AT + 1, skipped=M.EXPORT_AT,
                       heads=True)
    assert len(outs) == M.HEADS_PUSHES - M.EXPORT_AT and all(o.shape == (K + 1, M.RESTORE_P) for o in outs.values())
    pairs += [(f"restored {n}", *rest) for n, *rest in ps]
    sc.close()
    sc2.close()
    _check(pairs)


# ------------------------------------------------------------------ push staging
@pytest.mark.parametrize("name", sorted(M.STAGING_CASES))
def test_push_staging(name):
    """each segment pushed three ways: a view 4 (fp32) or 2 (bf16) bytes past a 16-byte boundary with a 16-byte pitch,
    a view of [P, C, S + 2] rows, and contiguous (not staged at phase 0); the three bit-identical, and judged"""
    c = M.STAGING_CASES[name]
    seed = 800 + sorted(M.STAGING_CASES).index(name)
    dtype = DT[c.dtype]
    n_push = M.n0_of(c.W, c.S) + 2
    ref, m = _pair(c, seed)
    stream = _stream(c, n_push, seed)
    sd = stream.to(DEV)
    age = tskd_b200.synth.make_ages(c.P, seed=seed)

    def offset(n):
        buf = torch.zeros(c.P, c.C, c.S + 8, dtype=dtype, device=DEV)
        buf[:, :, 1:c.S + 1] = sd[:, :, (n - 1) * c.S:n * c.S]
        v = buf[:, :, 1:c.S + 1]
        assert v.data_ptr() % 16 == v.element_size() and v.stride(1) * v.element_size() % 16 == 0
        return v

    def pitched(n):
        buf = torch.zeros(c.P, c.C, c.S + 2, dtype=dtype, device=DEV)
        buf[:, :, :c.S] = sd[:, :, (n - 1) * c.S:n * c.S]
        v = buf[:, :, :c.S]
        assert v.stride(1) * v.element_size() % 16 != 0
        return v

    def contiguous(n):
        v = sd[:, :, (n - 1) * c.S:n * c.S].contiguous()
        assert v.data_ptr() % 16 == 0 and c.S * v.element_size() % 16 == 0
        return v

    outs, pairs = {}, []
    for way, fn in (("contiguous", contiguous), ("offset", offset), ("pitched", pitched)):
        sc = _scorer(m, c)
        ps, outs[way] = _replay(sc, [ref], stream, age, c.S, n_push, seg_of=fn)
        outs[way + " features"] = sc.features()
        if way == "contiguous":
            pairs = ps
        sc.close()
    for way in ("offset", "pitched"):
        assert outs[way].keys() == outs["contiguous"].keys()
        assert all(torch.equal(outs[way][n], outs["contiguous"][n]) for n in outs[way]), way
        assert torch.equal(outs[way + " features"], outs["contiguous features"]), way
    _check(pairs)
