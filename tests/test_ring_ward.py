"""The per-patient window rings (csrc/b2cnn_prep.cu b2cnn_ring_*, stream.PatientRing) judged patient by patient.

Every patient of a ring has its own record, selection, gains and baselines, so a kernel that read another patient's
column map, gains, signal count or fill carry would show.  Each emitted window is checked against
  - the whole-record device pass (b2cnn_prep_windows) of that patient's own record: bit for bit wherever a stream can
    know what the whole record knows, and
  - the float64 restatement (oracle/stream_np.py, pinned to pandas) in its causal form everywhere: within one f32 ulp.
One push emits at most one window; pushes that would leave a completed window behind are refused (the grid ring holds
256 points, and a backlog of windows would be read back from overwritten slots).
"""
import functools

import numpy as np
import pytest
import torch

import tskd_b200
from tskd_b200 import stream as S
from conftest import load_golden
from oracle import stream_np as N

STEP = S.STRIDE_S // S.GRID_S                  # 12 grid points per window stride
WARD_FS, WARD_N, WARD_SIG = 1.0, 2400, 9       # 40 min at 1 Hz: 480 grid points, 31 windows
# (seed, missing rate, leading gap [samples] on the first selected signal, dead column, selection in model-channel order)
WARD = [(101, 0.0, 0, None, [0, 1, 2, 3, 4, 5, 6]),
        (102, 0.2, 0, None, [5, 2, 7, 0]),
        (103, 0.5, 900, None, [3]),
        (104, 0.3, 0, 2, [8, 2, 4, 6]),
        (105, 0.9, 0, None, [1, 0, 3, 2, 6, 5, 4]),
        (106, 0.1, 0, None, []),
        (107, 0.2, 1300, None, [4, 8, 0, 1]),
        (108, 0.0, 0, 7, [7]),
        (109, 0.4, 700, None, [6, 1, 8, 3, 0, 2, 5]),
        (110, 0.2, 0, 3, [3, 5, 7, 1]),
        (111, 0.05, 2000, None, [2]),
        (112, 0.3, 0, None, [])]
# ring schedules that outrun the 60 s stride: (rate, samples per push, first push whose window the old rule read from
# overwritten grid slots).  9 samples per push at 1/7 Hz is round(60 * fs), the fixed cut replay_stream used to make.
BACKLOG = [(1 / 60, 2, 17), (1.0, 61, 685), (0.2, 13, 137), (1 / 7, 9, 229)]


def _record(seed, n, fs, p_missing=0.2, lead=0, lead_col=0, dead=None, names=None):
    rng = np.random.default_rng(seed)
    raw = rng.integers(-500, 3000, size=(n, WARD_SIG)).astype(np.int16)
    raw[rng.random(raw.shape) < p_missing] = -32768
    if lead:
        raw[:lead, lead_col] = -32768
    if dead is not None:
        raw[:, dead] = -32768
    gains = rng.choice([0.5, 1.0, 3.0, 10.0, 12.5], size=WARD_SIG)
    bases = rng.integers(-50, 50, size=WARD_SIG).astype(np.float64)
    return S.NumericsRecord(tuple(names or [f"s{j}" for j in range(WARD_SIG)]), gains, bases, fs, raw)


def _view(rec, sel):
    """The record as the whole-record pass sees the selection: selected columns in model-channel order."""
    return S.NumericsRecord(S.CHANNEL_NAMES[:len(sel)], rec.gains[sel], rec.baselines[sel], rec.fs, rec.raw[:, sel])


def _ward_records():
    return [_record(seed, WARD_N, WARD_FS, pm, lead, sel[0] if sel else 0, dead) for seed, pm, lead, dead, sel in WARD]


@functools.lru_cache(maxsize=None)
def _oracle():
    """Per patient: unfilled grid of the selection (as far as any push can finalise), the whole-record float64 windows,
    and the filled grids of all columns (the grid-point payload)."""
    period = N.sample_period_ns(WARD_FS)
    k_max = WARD_N * period // (S.GRID_S * N.NS)
    out = []
    for rec, (_, _, _, _, sel) in zip(_ward_records(), WARD):
        phys = rec.physical
        unf = np.stack([N.smooth_to_grid(phys[:, s], WARD_FS, fill=False, n_grid=k_max) for s in sel]) if sel else np.zeros((0, k_max))
        whole, _ = N.assemble_windows(_view(rec, sel), list(range(len(sel))))
        filled = np.stack([N.smooth_to_grid(phys[:, j], WARD_FS) for j in range(WARD_SIG)])
        out.append((unf, whole, filled))
    return out


def _expected_causal(p, k_ends):
    unf, _, _ = _oracle()[p]
    return N.causal_windows(unf, k_ends) if unf.shape[0] else np.zeros((len(k_ends), S.N_CHANNELS, S.WINDOW_POINTS))


# ------------------------------------------------------------------------------------------------------------ CPU
def test_causal_fill_is_the_whole_record_fill_of_the_final_points():
    """causal_windows(unfilled, k_ends)[w] == the whole-record form run on grid points 0 .. k_ends[w]-1 only, and equals
    the whole-record form outright for every patient whose signals appear within the first window."""
    for p, (seed, pm, lead, dead, sel) in enumerate(WARD):
        unf, whole, _ = _oracle()[p]
        if not sel:
            assert whole.shape[0] == 0
            continue
        n_win = whole.shape[0]
        assert n_win == 31
        for extra in (0, 7, 11):
            k_ends = [min(unf.shape[1], STEP * w + S.WINDOW_POINTS + extra) for w in range(n_win)]
            got = N.causal_windows(unf, k_ends)
            for w in (0, 5, 9, 10, 17, 20, 21, 30):
                pref, _ = N.windows_from_grids(np.stack([N.fill_grid(g[:k_ends[w]]) for g in unf]))
                assert np.array_equal(got[w], pref[w]), (p, w, extra)
            if lead == 0:
                assert np.array_equal(got, whole), p
            else:
                first = int(np.nonzero(~np.isnan(unf[0]))[0][0])
                assert first >= S.WINDOW_POINTS                            # the gap is longer than one window
                before = [w for w in range(n_win) if k_ends[w] <= first]
                assert before and all((got[w, 0] == 0).all() for w in before)
                assert not np.array_equal(got[before[0]], whole[before[0]])   # the whole record back-fills from the future
                after = [w for w in range(n_win) if k_ends[w] > first]
                assert np.array_equal(got[after], whole[after]) and np.array_equal(got[before, 1:], whole[before, 1:])
    with pytest.raises(ValueError):
        N.causal_windows(_oracle()[0][0], [120, 132, 144, STEP * 3 + S.WINDOW_POINTS - 1])   # window 3 is not complete yet


def test_stride_cut_triggers_emit_exactly_one_window_each_at_any_rate():
    """trigger_cuts (replay_stream's triggers) never trips the one-window rule and never lags: trigger n >= 10 emits
    window n - 10, at rates on and off the 5-second lattice."""
    for fs in (1 / 60, 1 / 59, 1 / 7, 0.2, 1 / 3, 0.5, 1.0, 2.0, 3.7, 25.0):
        period = N.sample_period_ns(fs)
        n = -(-300 * S.STRIDE_S * N.NS // period)                       # 300 strides of samples
        cuts = S.trigger_cuts(n, fs)
        sizes = np.diff(cuts)
        assert cuts[0] == 0 and cuts[-1] == n and (sizes >= 1).all()
        assert (sizes * period <= S.STRIDE_S * N.NS + period).all()          # the per-push size limit
        for t, c in enumerate(cuts[1:-1], start=1):
            assert (c - 1) * period < t * S.STRIDE_S * N.NS <= c * period, (fs, t)
        sched = N.ring_schedule(fs, sizes)
        assert not any(r for _, _, r in sched), fs
        assert [w for _, w, _ in sched] == [-1] * 9 + list(range(len(sizes) - 9)), fs


def test_backlog_schedules_are_refused_before_any_window_is_overwritten():
    """The schedules of BACKLOG under the old size-only rule build a backlog until a window is read from grid slots that
    newer points overwrote; under the one-window rule their first refusal comes long before that."""
    for fs, per, first_bad in BACKLOG:
        period, grid = N.sample_period_ns(fs), S.GRID_S * N.NS
        assert per * period <= S.STRIDE_S * N.NS + period                  # passed the old check
        n_in, w, bad = 0, 0, None
        for push in range(1, first_bad + 1):                               # the old rule: no refusal, one window per push
            n_in += per
            k_end = n_in * period // grid
            if STEP * w + S.WINDOW_POINTS <= k_end:
                if k_end > STEP * w + 256:                                 # slot (12 w + j) % 256 rewritten by a newer point
                    bad = push
                    break
                w += 1
        assert bad == first_bad, (fs, per)
        sched = N.ring_schedule(fs, [per] * first_bad)
        refused = [i + 1 for i, (_, _, r) in enumerate(sched) if r]
        assert refused and refused[0] < first_bad


# ------------------------------------------------------------------------------------------------------------ GPU
def _set_signals(ring, p, rec, sel, physical=False):
    if physical:
        ring.set_signals(p, sel)
    else:
        ring.set_signals(p, sel, rec.gains, rec.baselines)


def _whole_dev(rec, sel):
    return S.assemble_windows_gpu(_view(rec, sel), "cuda:0")[0]


@pytest.mark.gpu
@pytest.mark.parametrize("fs,per,first_bad", BACKLOG)
def test_ring_refuses_pushes_that_would_leave_a_window_behind(fs, per, first_bad):
    """Push the BACKLOG schedules.  A push after which two windows would be complete is refused (and then delivered in
    halves); every push emits the newest complete window, with the right index and start time, equal bit for bit to the
    whole-record window of that index for each of three different patients."""
    n = per * (first_bad + 15)
    pats = [(21, 0.2, [0, 1, 2, 3]), (22, 0.5, [6, 3, 1]), (23, 0.0, [2])]
    recs = [_record(seed, n, fs, pm) for seed, pm, _ in pats]
    whole = [_whole_dev(r, sel) for r, (_, _, sel) in zip(recs, pats)]
    ring = S.PatientRing(3, WARD_SIG, fs, device="cuda:0")
    for p, (r, (_, _, sel)) in enumerate(zip(recs, pats)):
        _set_signals(ring, p, r, sel)
    src = torch.from_numpy(np.stack([r.raw for r in recs])).cuda()
    period, grid = N.sample_period_ns(fs), S.GRID_S * N.NS
    st = {"w": 0, "refused": 0}

    def push(i0, i1):
        k_end = i1 * period // grid
        if STEP * (st["w"] + 1) + S.WINDOW_POINTS <= k_end:               # would complete two windows
            with pytest.raises(RuntimeError, match="two windows"):
                ring.push(src[:, i0:i1])
            st["refused"] += 1
            mid = (i0 + i1) // 2
            push(i0, mid)
            push(mid, i1)
            return
        out = ring.push(src[:, i0:i1])
        assert (out is not None) == (STEP * st["w"] + S.WINDOW_POINTS <= k_end), (i0, i1)
        if out is not None:
            x, widx, t0 = out
            assert widx == st["w"] and t0 == S.STRIDE_S * float(widx)
            for p in range(3):
                if widx < len(whole[p]):
                    assert torch.equal(x[p], whole[p][widx]), (p, widx, i1)
            st["w"] += 1
        assert st["w"] == max(0, (k_end - S.WINDOW_POINTS) // STEP + 1)   # nothing complete is left behind

    for i0 in range(0, n, per):
        push(i0, min(n, i0 + per))
    ring.close()
    assert st["refused"] > 0 and st["w"] >= len(whole[0]) - 1


@pytest.mark.gpu
def test_refused_push_leaves_later_output_bit_identical():
    """Ring A is offered pushes it must refuse (two 1/60 Hz samples that would complete two windows; three samples, more
    than one stride); ring B never
    sees them.  Both then get the same one-sample triggers: every later output, index and start time is identical, and
    a refusal does not touch A's output tensor."""
    fs, n = 1 / 60, 400
    recs = [_record(s, n, fs, 0.3) for s in (31, 32)]
    sels = [[0, 4, 2], [5, 1, 8, 3]]
    a, b = S.PatientRing(2, WARD_SIG, fs, device="cuda:0"), S.PatientRing(2, WARD_SIG, fs, device="cuda:0")
    for p in range(2):
        _set_signals(a, p, recs[p], sels[p])
        _set_signals(b, p, recs[p], sels[p])
    src = torch.from_numpy(np.stack([r.raw for r in recs])).cuda()
    n_out = 0
    for t in range(n - 3):
        if t in (130, 131, 250):
            before = a.x.clone()
            with pytest.raises(RuntimeError, match="two windows"):
                a.push(src[:, t:t + 2])
            with pytest.raises(RuntimeError, match="at most stride_s"):
                a.push(src[:, t:t + 3])
            assert torch.equal(a.x, before)
        oa, ob = a.push(src[:, t:t + 1]), b.push(src[:, t:t + 1])
        assert (oa is None) == (ob is None)
        if oa is not None:
            assert oa[1:] == ob[1:] == (n_out, S.STRIDE_S * float(n_out))
            assert torch.equal(oa[0], ob[0]), t
            n_out += 1
    assert n_out == n - 3 - 9
    a.close(); b.close()
    with pytest.raises(RuntimeError):
        S.PatientRing(1, 4, 1 / 61, device="cuda:0")                      # one sample would complete two windows


@pytest.mark.gpu
def test_replay_stream_at_one_seventh_hz_equals_whole_record_replay():
    """replay_stream cuts triggers at stride boundaries (9, 9, 8, ... samples at 1/7 Hz): three different patients scored
    trigger by trigger give, row for row, the whole-record replay of each one's own record."""
    _, sd = load_golden("mycnn5_xtestinput.npz")
    model = tskd_b200.B200MyCNN.from_reference(sd).to("cuda:0")
    names = ["HR", "junk", "RESP", "SpO2", "x", "PULSE", "CVP", "y", "NBP Mean"]
    recs = [_record(s, 2600, 1 / 7, pm, names=names) for s, pm in ((41, 0.1), (42, 0.4), (43, 0.0))]
    ids = [7, 8, 9]
    rows = S.replay_stream(model, recs, ids)
    for rec, sid in zip(recs, ids):
        mine = [r for r in rows if r[0] == sid]
        whole = S.replay(model, rec, subject_id=sid, micro_batch=3)
        assert len(whole) == 294 and len(mine) in (len(whole), len(whole) + 1)
        assert [r[1] for r in mine[:len(whole)]] == [r[1] for r in whole]
        assert np.array_equal(np.array([r[2] for r in mine[:len(whole)]]), np.array([r[2] for r in whole])), sid


def _run_ward(rings, src, sizes, grid_points):
    """Pushes `sizes` rows of src [P, n, n_sig] into every ring in lockstep.  Returns (k_end of each emitting push,
    [n_emit, P, 10, 120] f32 outputs of rings[0]); the bf16 ring must equal the f32 ring cast to bf16."""
    sched = N.ring_schedule(WARD_FS, sizes, grid_points=grid_points)
    k_ends, xs, i0 = [], [], 0
    for s, (k_end, w, refused) in zip(sizes, sched):
        assert not refused
        outs = [r.push(src[:, i0:i0 + s], grid_points=grid_points) for r in rings]
        i0 += s
        assert all((o is None) == (w < 0) for o in outs), i0
        if w < 0:
            continue
        for o in outs:
            assert o[1] == w and o[2] == S.STRIDE_S * float(w)
        x32 = outs[0][0]
        for r, o in zip(rings[1:], outs[1:]):
            assert torch.equal(o[0], x32.to(r.dtype)), (w, r.dtype)
        k_ends.append(k_end)
        xs.append(x32.cpu().numpy())
    return k_ends, np.stack(xs)


def _check_ward(k_ends, xs, whole_dev):
    """Patient p of every emitted window: within one f32 ulp of the causal float64 oracle; bit for bit the whole-record
    device window wherever the oracle's causal and whole-record forms agree; zeros beyond the patient's selection."""
    n_same = 0
    for p, (_, _, _, _, sel) in enumerate(WARD):
        got = xs[:, p].astype(np.float64)
        want = _expected_causal(p, k_ends)
        ulp = np.spacing(np.abs(want).astype(np.float32)).astype(np.float64)
        assert (np.abs(got - want) <= ulp).all(), (p, np.argwhere(np.abs(got - want) > ulp)[:5])
        assert (xs[:, p, len(sel):] == 0).all()
        whole_np = _oracle()[p][1] if sel else np.zeros((whole_dev[p].shape[0], S.N_CHANNELS, S.WINDOW_POINTS))
        m = min(len(got), len(whole_np))
        for w in range(m):
            if np.array_equal(want[w], whole_np[w]):
                n_same += 1
                assert np.array_equal(xs[w, p], whole_dev[p][w]), (p, w)
    return n_same


@functools.lru_cache(maxsize=None)
def _whole_ward():
    return [_whole_dev(r, sel).cpu().numpy() for r, (_, _, _, _, sel) in zip(_ward_records(), WARD)]


def _ward_rings(kind, P=len(WARD), dtypes=(torch.float32, torch.bfloat16), slot=None):
    recs = _ward_records()
    slot = np.arange(P) % len(WARD) if slot is None else slot
    rings = [S.PatientRing(P, WARD_SIG, WARD_FS, device="cuda:0", dtype=dt) for dt in dtypes]
    for r in rings:
        for q in range(P):
            p = int(slot[q])
            _set_signals(r, q, recs[p], WARD[p][4], physical=kind != "adc16")
    if kind == "adc16":
        src = np.stack([rec.raw for rec in recs])
    elif kind == "f64":
        src = np.stack([rec.physical for rec in recs])
    else:
        src = np.stack([o[2].T for o in _oracle()])                      # [P, n_grid, n_sig] filled grid points
    return rings, torch.from_numpy(np.ascontiguousarray(src[slot])).cuda()


def _sizes(total, per):
    return [min(per, total - i) for i in range(0, total, per)]


@pytest.mark.gpu
@pytest.mark.parametrize("kind,per", [("adc16", 1), ("adc16", 7), ("adc16", 37), ("adc16", 60),
                                      ("f64", 1), ("f64", 7), ("f64", 37), ("f64", 60),
                                      ("grid", 1), ("grid", 7), ("grid", 12)])
def test_heterogeneous_ward_each_patient_against_its_own_record(kind, per):
    """Twelve patients with their own records, selections (0, 1, 4 or 7 signals in shuffled column order), gains,
    baselines, missing rates, leading gaps longer than a window and dead signals, in f32 and bf16."""
    rings, src = _ward_rings(kind)
    k_ends, xs = _run_ward(rings, src, _sizes(src.shape[1], per), grid_points=kind == "grid")
    for r in rings:
        r.close()
    assert len(k_ends) >= 31
    if kind == "grid":                                                     # points appended as they are: exact f32 casts
        for p, (_, _, _, _, sel) in enumerate(WARD):
            filled = _oracle()[p][2]
            want = np.zeros((len(k_ends), S.N_CHANNELS, S.WINDOW_POINTS), dtype=np.float32)
            for w in range(len(k_ends)):
                want[w, :len(sel)] = filled[sel, STEP * w:STEP * w + S.WINDOW_POINTS]
            assert np.array_equal(xs[:, p], want), p
        return
    n_same = _check_ward(k_ends, xs, _whole_ward())
    assert n_same >= 300                       # of 31 x 12: only windows inside a leading gap are judged by the oracle alone


@pytest.mark.gpu
def test_ward_of_4096_patients_and_a_reset():
    """4096 slots holding a fixed permutation of the twelve records: every slot equals, bit for bit, the twelve-patient
    ring's row of its record (itself checked against the oracle); then reset() and a replay with other push sizes."""
    slot = np.random.default_rng(5).permutation(np.arange(4096) % len(WARD))
    big, src_big = _ward_rings("adc16", P=4096, dtypes=(torch.float32,), slot=slot)
    small, src = _ward_rings("adc16", dtypes=(torch.float32,))
    big, small = big[0], small[0]
    slot_t = torch.from_numpy(slot).cuda()
    for per in (37, 60):                                                   # the second pass follows a reset()
        k_ends, xs, i0 = [], [], 0
        for s in _sizes(WARD_N, per):
            o_big, o_small = big.push(src_big[:, i0:i0 + s]), small.push(src[:, i0:i0 + s])
            i0 += s
            assert (o_big is None) == (o_small is None)
            if o_big is None:
                continue
            assert o_big[1:] == o_small[1:] == (len(xs), S.STRIDE_S * float(len(xs)))
            assert torch.equal(o_big[0], o_small[0][slot_t]), len(xs)
            k_ends.append(i0 * N.sample_period_ns(WARD_FS) // (S.GRID_S * N.NS))
            xs.append(o_small[0].cpu().numpy())
        assert len(xs) >= 31
        _check_ward(k_ends, np.stack(xs), _whole_ward())
        big.reset(); small.reset()
    big.close(); small.close()
