"""GPU: whole-recording scoring (predict_record, b2cnn_score_record[_ex]) where its branches differ from what the other
record tests run, and the probability epilogue of every tensor-core entry point.

Each case asserts through tests/record_plan.py (the plan of csrc/b2cnn_record.cu restated) that it reaches the branch
it is named for, and that the library's workspace size is the plan's.

- production scale: [4096, 3, 142500] bf16 at W = 75000, S = 45000 -- 110592 staged row-channels, so the staging grid
  strides and recording 2427 straddles row-channel 65535; 36864 folded rows, 8192 windows -- in both modes, logits and
  probabilities, judged against float64 at the stride boundary, the ends and 48 random recordings; bit identity of
  single recordings and of the clean recordings around NaN samples.  The generic path at its benchmark size
  ([1024, 10, 7200], the MyCNN5 golden, S = 12: 73728 folded rows) bit for bit against predict();
- views on the tensor-core path (row-padded at pitch N + 8 and N + 3, a one-sample offset, recording slices, a
  direct C call with pitch > N): torch.equal to the contiguous recordings in both modes;
- fold geometry: N = W, N = W + S - 1, L_N = 4096, 4097 and 8 * 4096 + 1, and S = 4 with the fold seam inside every
  window, in both tensor-core geometries and dtypes and both modes, every window judged against float64;
- return_prob on predict() (fused bf16 and the fp32 stream front end, both modes), the tensor-core SlidingScorer with
  patients admitted and discharged, every row of push(heads=True) with a shorter-window head, and predict_record in
  both modes: judged against sigmoid(float64 truth), NaN rows NaN.

Grants: BETA (predict_record independent mode, the scorer), BETA_TC_SEQ (predict_record sequence mode),
BETA_TC_LOGITS / BETA_STREAM_LOGITS (predict() on the fused / stream front ends)."""
import os

import pytest
import torch

import tskd_b200
from oracle.infer_ref import infer_reference
from oracle.train_ref import BETA, check_elems
from record_plan import N_for_L_N, record_plan, row_channel, row_samples, stage_block, windows_of_sample
from test_gpu_infer_elem import BETA_STREAM_LOGITS, BETA_TC_LOGITS
from test_gpu_record import _records, _tc_pair, _wins
from test_gpu_record_sequence import BETA_TC_SEQ, _truth
from test_gpu_slide_generic import _golden, _same
from test_gpu_slide_horizons import _tc_family
from tskd_b200 import capi

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
BF, F32 = torch.bfloat16, torch.float32
MODES = ("independent", "sequence")


def _check(pairs):
    check_elems(pairs, os.environ.get("PYTEST_CURRENT_TEST", "").split(" ")[0])


def _dt(dtype):
    return "bf16" if dtype == BF else "f32"


def _plan(m, kind, N, S, B, dtype, mode="independent", path="tensorcore"):
    a = m.arch
    return record_plan(kind, a.window, N, S, B, a.in_channels, _dt(dtype), mode, path)


def _assert_workspace(m, kind, B, N, S, dtype, pitch=None):
    """the library's workspace bytes (tensor-core path) are the plan's, in both modes"""
    lib, h = m._ensure_handle()
    for mode, cm in zip(MODES, (capi.MODE_INDEPENDENT, capi.MODE_SEQUENCE)):
        got = int(lib.b2cnn_record_workspace_bytes_ex(h, B, N, pitch or N, S, capi.DTYPE_BF16 if dtype == BF else capi.DTYPE_F32,
                                                      capi.PATH_TENSORCORE, cm))
        assert got == _plan(m, kind, N, S, B, dtype, mode).ws, (mode, got)


def _independent_truth(ref, x, S, age):
    """(float64, float32) logits [B, n_w] of every window of x [B, C, N] (CPU), each from the zero state"""
    B = x.shape[0]
    W = ref.arch.window
    win = _wins(x, W, S)
    n_w = win.shape[0] // B
    ages = age.reshape(-1).cpu()
    ages = ages.expand(B) if ages.numel() == 1 else ages
    ages = ages.repeat_interleave(n_w)
    t, t32 = infer_reference(ref, win, ages)["z"], infer_reference(ref, win, ages, dtype=torch.float32)["z"]
    return t.reshape(B, n_w), t32.reshape(B, n_w)


def _record_pairs(tag, ref, m, x, S, age, path="tensorcore", prob=(False,)):
    """both modes of predict_record on x (device), each judged against float64: the (name, got, truth, ref32, beta)"""
    xc = x.cpu()
    pairs = []
    for mode in MODES:
        t, t32 = _independent_truth(ref, xc, S, age) if mode == "independent" else _truth(ref, xc, S, age)
        beta = BETA if mode == "independent" else BETA_TC_SEQ
        for p in prob:
            out = m.predict_record(x, S, age, return_prob=p, path=path, mode=mode)
            assert m.last_path == path
            pairs.append((f"{tag}-{mode}{'-prob' if p else ''}", out, torch.sigmoid(t) if p else t, torch.sigmoid(t32) if p else t32,
                          beta))
    return pairs


# ------------------------------------------------------------------ 1. production scale
PROD_W, PROD_S, PROD_B, PROD_N = 75000, 45000, 4096, 142500
STRIDE_REC = 2427                                                  # its row 2, channel 0 is row-channel 65535


@torch.no_grad()
def test_production_scale_tensorcore():
    ref, m = _tc_pair("mycnn5", 3, PROD_W, 101)
    p = _plan(m, "mycnn5", PROD_N, PROD_S, PROD_B, BF)
    assert (p.L_N, p.nr, p.K, p.rows, p.n_w, p.M) == (35620, 9, 3960, 36864, 2, 8192)
    assert p.row_channels == 110592 and p.stage_strides and p.grid_y == 65535
    assert stage_block(row_channel(p, 3, STRIDE_REC, 2, 0)) == (0, 1)                 # the first row-channel of the second pass
    assert stage_block(row_channel(p, 3, STRIDE_REC, 1, 2)) == (65534, 0)
    print(f"production: row-channels {p.row_channels}, nr {p.nr}, K {p.K}, rows {p.rows}, windows {p.M}")
    _assert_workspace(m, "mycnn5", PROD_B, PROD_N, PROD_S, BF)
    x = tskd_b200.synth.make_windows(PROD_B, 3, PROD_N, "normal", seed=101, dtype=BF, device=DEV)
    age = tskd_b200.synth.make_ages(PROD_B, seed=101, device=DEV)
    out = {}
    for mode in MODES:
        for prob in (False, True):
            out[mode, prob] = m.predict_record(x, PROD_S, age, return_prob=prob, mode=mode)
            assert m.last_path == "tensorcore" and out[mode, prob].shape == (PROD_B, 2)

    # float64 at the stride boundary, the ends and 48 random recordings
    g = torch.Generator().manual_seed(101)
    fixed = [0, 1, STRIDE_REC - 1, STRIDE_REC, STRIDE_REC + 1, PROD_B - 2, PROD_B - 1]
    rand = [i for i in torch.randperm(PROD_B, generator=g).tolist() if i not in fixed][:48]
    sel = torch.tensor(sorted(fixed + rand))
    xs, ags = x[sel.to(DEV)].cpu(), age[sel.to(DEV)].cpu()
    pairs = []
    for mode in MODES:
        t, t32 = _independent_truth(ref, xs, PROD_S, ags) if mode == "independent" else _truth(ref, xs, PROD_S, ags)
        beta = BETA if mode == "independent" else BETA_TC_SEQ
        pairs.append((f"z-{mode}", out[mode, False][sel.to(DEV)], t, t32, beta))
        pairs.append((f"prob-{mode}", out[mode, True][sel.to(DEV)], torch.sigmoid(t), torch.sigmoid(t32), beta))
    _check(pairs)

    # a recording scored alone is its row of the full call
    for b in (STRIDE_REC, PROD_B - 1):
        for mode in MODES:
            alone = m.predict_record(x[b:b + 1], PROD_S, age[b:b + 1], mode=mode)
            assert torch.equal(alone[0], out[mode, False][b]), (b, mode)

    # NaN in recording 2427's row 2 (window 0 only) and in recording 4095's row 7 (window 1) and last row (no window)
    r2 = row_samples(p, 2)
    sites = [(STRIDE_REC, 0, 40000), (PROD_B - 1, 1, 115000), (PROD_B - 1, 2, 140000)]
    assert row_samples(p, 1)[1] < 40000 < row_samples(p, 3)[0] and r2[0] <= 40000 <= r2[1]
    assert row_samples(p, 7)[0] <= 115000 < row_samples(p, 8)[0] <= 140000
    assert windows_of_sample(p, PROD_S, 40000) == [0] and windows_of_sample(p, PROD_S, 115000) == [1]
    assert windows_of_sample(p, PROD_S, 140000) == []
    saved = [x[b, c, s].clone() for b, c, s in sites]
    for b, c, s in sites:
        x[b, c, s] = float("nan")
    nan_w = {STRIDE_REC: {0}, PROD_B - 1: {1}}
    dirty = torch.zeros(PROD_B, dtype=torch.bool, device=DEV)
    dirty[list(nan_w)] = True
    try:
        for mode in MODES:
            got = m.predict_record(x, PROD_S, age, mode=mode)
            assert m.last_path == "tensorcore"
            assert torch.equal(got[~dirty], out[mode, False][~dirty]), mode
            for b, ws in nan_w.items():
                first = min(ws)
                want = {w for w in range(2) if (w in ws if mode == "independent" else w >= first)}
                assert {w for w in range(2) if torch.isnan(got[b, w])} == want, (mode, b)
            xs = x[list(nan_w)].cpu()
            ags = age[list(nan_w)].cpu()
            t, t32 = _independent_truth(ref, xs, PROD_S, ags) if mode == "independent" else _truth(ref, xs, PROD_S, ags)
            _check([(f"nan-{mode}", got[list(nan_w)], t, t32, BETA if mode == "independent" else BETA_TC_SEQ)])
    finally:
        for (b, c, s), v in zip(sites, saved):
            x[b, c, s] = v


@torch.no_grad()
def test_production_scale_generic():
    """the generic path at its benchmark size, bit for bit against predict() on the materialised windows"""
    ref, m = _golden(5)
    B, C, N, S = 1024, 10, 7200, 12
    p = _plan(m, "mycnn5", N, S, B, F32, path="generic")
    assert (p.L, p.L_N, p.nr, p.K, p.rows, p.n_w) == (25, 1795, 72, 25, 73728, 591)
    assert p.stage_strides
    print(f"generic production: row-channels {p.row_channels}, nr {p.nr}, rows {p.rows}, windows {p.M}")
    x = tskd_b200.synth.make_windows(B, C, N, "normal", seed=102, device=DEV)
    age = tskd_b200.synth.make_ages(B, seed=102, device=DEV)
    out = m.predict_record(x, S, age, path="generic")
    assert m.last_path == "generic" and out.shape == (B, p.n_w)
    for b0 in range(0, B, 64):
        want = m.predict(_wins(x[b0:b0 + 64], 120, S), age[b0:b0 + 64].repeat_interleave(p.n_w))
        assert m.last_path == "generic"
        assert _same(out[b0:b0 + 64].reshape(-1), want), b0


# ------------------------------------------------------------------ 2. views on the tensor-core path
VIEW_MODELS = {"m5-bf16": ("mycnn5", 3, BF, 7504), "m3-bf16": ("mycnn3", 2, BF, 7502), "m3-f32": ("mycnn3", 1, F32, 7502)}


def _in_place(v, C):
    """predict_record reads v where it lies, without a contiguous copy: contiguous from an offset pointer, or rows at a
    pitch > N"""
    return v.is_contiguous() or (v.stride(2) == 1 and v.stride(1) > v.shape[2] and (v.shape[0] == 1 or v.stride(0) == C * v.stride(1)))


@pytest.mark.parametrize("name", sorted(VIEW_MODELS))
def test_views_tensorcore(name):
    kind, C, dtype, W = VIEW_MODELS[name]
    S, B = 752, 3
    N = W + 12 * S + 5
    seed = 110 + sorted(VIEW_MODELS).index(name)
    ref, m = _tc_pair(kind, C, W, seed)
    p = _plan(m, kind, N, S, B, dtype)
    assert p.nr >= 2
    age = tskd_b200.synth.make_ages(B, seed=seed).to(DEV)
    pad8 = _records(B, C, N + 8, dtype, seed).to(DEV)
    pad3 = _records(B, C, N + 3, dtype, seed + 1).to(DEV)
    views = {"pitch-n+8": (pad8[:, :, :N], age), "pitch-n+3": (pad3[:, :, :N], age), "offset-1": (pad8[:, :, 1:N + 1], age),
             "slice-1": (pad8[1:2, :, 3:N + 3], age[1:2]), "slice-1:3": (pad3[1:3, :, 2:N + 2], age[1:3])}
    if dtype == BF:
        assert pad8[:, :, 1:].data_ptr() % 4 == 2                    # bf16 rows at 2-byte alignment
    for vname, (v, a) in views.items():
        assert _in_place(v, C), vname
        for mode in MODES:
            got = m.predict_record(v, S, a, mode=mode)
            assert m.last_path == "tensorcore"
            assert torch.equal(got, m.predict_record(v.contiguous(), S, a, mode=mode)), (vname, mode)
    # the C ABI with pitch > N on the padded buffer itself
    lib, h = m._ensure_handle()
    st = torch.cuda.current_stream().cuda_stream
    dt = capi.DTYPE_BF16 if dtype == BF else capi.DTYPE_F32
    _assert_workspace(m, kind, B, N, S, dtype, pitch=N + 8)
    for mode, cm in zip(MODES, (capi.MODE_INDEPENDENT, capi.MODE_SEQUENCE)):
        need = int(lib.b2cnn_record_workspace_bytes_ex(h, B, N, N + 8, S, dt, capi.PATH_TENSORCORE, cm))
        ws = torch.empty(need, dtype=torch.uint8, device=DEV)
        out = torch.full((B, p.n_w), 7.0, device=DEV)
        rc = lib.b2cnn_score_record_ex(h, pad8.data_ptr(), dt, B, N, N + 8, S, capi.PATH_TENSORCORE, cm, age.data_ptr(), B, 0,
                                       out.data_ptr(), ws.data_ptr(), need, st)
        assert rc == 0, capi.last_error()
        assert m.last_path == "tensorcore"
        assert torch.equal(out, m.predict_record(pad8[:, :, :N].contiguous(), S, age, mode=mode)), mode
    _check(_record_pairs(f"{name}-offset-1", ref, m, views["offset-1"][0], S, age))


# ------------------------------------------------------------------ 3. fold geometry
GEOMETRY = {"m5": ("mycnn5", 3, 7504), "m3": ("mycnn3", 2, 7502)}
FOLDS = ("n-eq-w", "n-eq-w+s-1", "ln-4096", "ln-4097", "ln-8x4096+1", "s4-seam")
FOLD_CASES = [(g, d, f) for g in GEOMETRY for d in ("bf16", "f32") for f in FOLDS]


def _fold_case(kind, W, fold):
    """(W, S, B, N) of a fold case"""
    S, B = 752, 3
    if fold == "n-eq-w":
        return W, S, B, W
    if fold == "n-eq-w+s-1":
        return W, S, B, W + S - 1
    if fold == "s4-seam":                                         # a long window: fewer windows, each holds the seam
        return W + 8496, 4, 2, N_for_L_N(kind, 4097) + 400
    L_N = {"ln-4096": 4096, "ln-4097": 4097, "ln-8x4096+1": 8 * 4096 + 1}[fold]
    return W, S, B, N_for_L_N(kind, L_N)


@pytest.mark.parametrize("geo,dt,fold", FOLD_CASES, ids=[f"{g}-{d}-{f}" for g, d, f in FOLD_CASES])
def test_fold_geometry(geo, dt, fold):
    kind, C, W0 = GEOMETRY[geo]
    dtype = BF if dt == "bf16" else F32
    W, S, B, N = _fold_case(kind, W0, fold)
    seed = 200 + FOLD_CASES.index((geo, dt, fold))
    ref, m = _tc_pair(kind, C, W, seed)
    p = _plan(m, kind, N, S, B, dtype)
    if fold in ("n-eq-w", "n-eq-w+s-1"):
        assert p.n_w == 1 and p.nr == 1 and (N - W == 0 if fold == "n-eq-w" else N - W == S - 1)
    elif fold == "ln-4096":
        assert (p.L_N, p.nr, p.K, p.pad) == (4096, 1, 4096, 0)
    elif fold == "ln-4097":
        assert (p.L_N, p.nr, p.K, p.pad) == (4097, 2, 2056, 15)      # the last row's last 15 features read the zero fill
    elif fold == "ln-8x4096+1":
        assert p.L_N == 8 * 4096 + 1 and p.nr == 9 and p.pad > 0
    else:
        assert p.nr == 2 and p.n_w > 100
        assert all(w * p.step <= p.K - 1 and p.K <= w * p.step + p.L - 1 for w in range(p.n_w))   # both sides of the seam
    print(f"{geo}-{dt}-{fold}: N {N}, L_N {p.L_N}, nr {p.nr}, K {p.K}, pad {p.pad}, windows {p.n_w}, row-channels {p.row_channels}")
    _assert_workspace(m, kind, B, N, S, dtype)
    x = _records(B, C, N, dtype, seed).to(DEV)
    age = torch.tensor([48.0], device=DEV) if fold == "ln-4097" else tskd_b200.synth.make_ages(B, seed=seed).to(DEV)
    _check(_record_pairs(f"{geo}-{dt}-{fold}", ref, m, x, S, age))


# ------------------------------------------------------------------ 4. the probability epilogue
@pytest.mark.parametrize("dtype", [BF, F32], ids=["fused-bf16", "stream-f32"])
def test_predict_prob(dtype):
    """predict(return_prob=True) on the fused bf16 and fp32 stream front ends, both modes, NaN windows included"""
    B, W = 129, 7504
    ref, m = _tc_pair("mycnn5", 3, W, 120)
    x = tskd_b200.synth.make_windows(B, 3, W, "normal", seed=120, dtype=dtype)
    x[5, 0, 100] = float("nan")                                   # independent: window 5; sequence: windows 5 onwards
    x[B - 2, 2, W - 1] = float("inf")
    age = tskd_b200.synth.make_ages(B, seed=120)
    want_path = "tensorcore" if dtype == BF else "stream"
    beta = BETA_TC_LOGITS if dtype == BF else BETA_STREAM_LOGITS
    pairs = []
    for mode in MODES:
        t, t32 = infer_reference(ref, x, age, mode)["z"], infer_reference(ref, x, age, mode, dtype=torch.float32)["z"]
        got = m.predict(x.to(DEV), age.to(DEV), mode=mode, return_prob=True)
        assert m.last_path == want_path
        assert torch.isnan(got[5]) and (mode == "independent") == bool(torch.isfinite(got[6]))
        pairs.append((f"prob-{mode}", got, torch.sigmoid(t), torch.sigmoid(t32), beta))
    _check(pairs)


@torch.no_grad()
def test_scorer_prob_with_lifecycle_and_heads():
    """SlidingScorer.push(return_prob=True) on the tensor-core path with patients admitted and discharged, and every
    row of push(heads=True, return_prob=True) with a head of half the window"""
    P, W, S = 130, 7504, 1876
    Wk = W // 2
    rows = _tc_family("mycnn5", 3, W, (Wk,), 130)
    m0 = rows[0].model
    n0 = -(-W // S)
    n_push = n0 + 2
    stream = tskd_b200.synth.make_windows(P, 3, n_push * S, "normal", seed=130, dtype=BF)
    stream[11, 0, (n0 + 1) * S - 10] = float("nan")              # a NaN window for a patient that stays scored
    age = tskd_b200.synth.make_ages(P, seed=130)
    sd, ad = stream.to(DEV), age.to(DEV)
    plain = tskd_b200.SlidingScorer(m0, P, S, BF)
    heads = tskd_b200.SlidingScorer(m0, P, S, BF)
    heads.set_heads([rows[1].model], shorter_windows=True)
    assert plain.path == heads.path == "tensorcore"
    admitted, discharged = [3, 70], [9, 129]
    seen = torch.zeros(P, dtype=torch.int64)
    pairs = []
    for n in range(1, n_push + 1):
        if n == n0 + 1:
            for sc in (plain, heads):
                sc.admit(admitted)
                sc.discharge(discharged)
            seen[admitted] = 0
        seg = sd[:, :, (n - 1) * S:n * S]
        got = plain.push(seg, ad, return_prob=True)
        goth = heads.push(seg, ad, return_prob=True, heads=True)
        seen += S
        if n > n0:
            seen[discharged] = -1
        if n * S < Wk:
            assert got is None and goth is None
            continue
        if n < n0:                                                # the head's window is complete, the scorer's not
            assert got is None and torch.isnan(goth[0]).all()
        else:
            assert _same(goth[0], got), n
        for i, (row, g) in enumerate(zip(rows, (got, goth[1]))):
            if g is None:
                continue
            win = stream[:, :, n * S - row.W:n * S]
            t, t32 = infer_reference(row.ref, win, age)["z"], infer_reference(row.ref, win, age, dtype=torch.float32)["z"]
            off = seen < row.W
            t[off], t32[off] = float("nan"), float("nan")
            assert torch.isnan(g.cpu()[off]).all(), (n, i)
            pairs.append((f"prob[{n}] row {i}", g.clone(), torch.sigmoid(t), torch.sigmoid(t32), BETA))
    plain.close()
    heads.close()
    _check(pairs)


def test_record_prob():
    """predict_record(return_prob=True), both modes, a NaN sample in one recording"""
    W, S, B = 7504, 752, 3
    N = W + 12 * S + 5
    ref, m = _tc_pair("mycnn5", 3, W, 140)
    assert _plan(m, "mycnn5", N, S, B, BF).nr >= 2
    x = _records(B, 3, N, BF, seed=140)
    x[1, 2, 5 * S + 100] = float("nan")
    age = tskd_b200.synth.make_ages(B, seed=140).to(DEV)
    pairs = _record_pairs("record", ref, m, x.to(DEV), S, age, prob=(False, True))
    for name, got, *_ in pairs:
        assert torch.isnan(got[1]).any() and torch.isfinite(got[0]).all() and torch.isfinite(got[2]).all(), name
    _check(pairs)
