"""Row f3 of SURVEY.md section 8: the reference's wire formats.  Messages are generated the way the reference's own code
emits them (oracle/wire_ref.py restates bin/sendStream.py:59-64 and bin/processStream.py:126-131); the expected values
are what ``json.loads`` returns for those strings.  CPU tests run the parser compiled for the host (the same source as
the device kernel); GPU tests decode whole triggers on the device and feed the ring buffers."""
import ctypes
import json
import math
import random
import struct

import numpy as np
import pytest
import torch

import tskd_b200
from tskd_b200 import capi
from tskd_b200 import stream as S
from conftest import load_golden
from oracle import stream_np as N
from oracle import wire_ref as R


def _record():
    g, _ = load_golden("p000194_replay.npz")
    return g, S.NumericsRecord(tuple(str(n) for n in g["names"]), g["gains"], g["baselines"], float(g["fs"]), g["raw"])


def _parse(s: bytes):
    st = ctypes.c_int32(0)
    return capi.load_library().b2cnn_parse_decimal(s, len(s), ctypes.byref(st)), st.value


def _same_bits(a: float, b: float) -> bool:
    return struct.pack("<d", a) == struct.pack("<d", b)


def test_host_parser_equals_json_loads_on_the_reference_messages_of_p000194():
    """Every [i, val] message sendStream.py would publish for the shipped record: val parsed == json.loads bit for bit."""
    g, rec = _record()
    sel = S.selected_signals(rec)
    names = [rec.names[i].replace(" ", "_") for i in sel]
    msgs = R.sample_messages(rec.physical[:, sel], names, "p000194-2112-05-23-14-34n")
    assert len(msgs) == 1625 * 4 and msgs[0][1] == b"p000194" and msgs[0][0] == "HR"
    n_nan = 0
    for topic, key, value in msgs:
        i, want = json.loads(value)
        body = value[value.index(b",") + 1:value.rindex(b"]")].strip()
        got, st = _parse(body)
        assert st == 0, value
        if isinstance(want, float) and math.isnan(want):
            assert math.isnan(got); n_nan += 1
        else:
            assert _same_bits(got, float(want)), value
    assert n_nan == int(np.isnan(rec.physical[:, sel]).sum())
    # a record with missing samples: json.dumps writes the bare token NaN (bin/sendStream.py does not filter it)
    rng = np.random.default_rng(3)
    p_signal = np.round(rng.normal(80, 20, size=(300, 5)), 1)
    p_signal[rng.random(p_signal.shape) < 0.3] = np.nan
    for topic, key, value in R.sample_messages(p_signal, list("abcde"), "p004980-x"):
        i, want = json.loads(value)
        got, st = _parse(value[value.index(b",") + 1:value.rindex(b"]")].strip())
        assert st == 0 and (math.isnan(got) if math.isnan(want) else _same_bits(got, want)), value


# exact halfway cases, 17 - 19 digits, both exponent spellings, the edges of the supported exponent range
EDGE_NUMBERS = ["0.30000000000000004", "9007199254740993", "9007199254740992", "4503599627370497.5", "4503599627370496.5",
                "1e22", "1e23", "8.5e-10", "123456789012345678", "1234567890123456789", "0.1", "1.0E-5", "1e-05", "-0.0",
                "2.5e+16", "0.000001", "1e27", "1E-27", "00012.50"]
OUT_OF_RANGE = ["1e28", "1e-300", "5e-324", "1.7976931348623157e308", "12345678901234567891"]
MALFORMED = ["abc", "1e", "--1", "", "1 ", "1,2", "0x10"]
# json.dumps writes bare NaN / Infinity, Spark's to_json quotes them (sign inside the quotes); null is a missing value
NON_FINITE = [("NaN", math.nan), ('"NaN"', math.nan), ("null", math.nan), ("Infinity", math.inf), ("-Infinity", -math.inf),
              ('"Infinity"', math.inf), ('"-Infinity"', -math.inf)]


def _corpus():
    """Shortest-repr strings (Python repr, Java Double.toString) of 36 000 values from 1e-6 to 1e15, both spellings."""
    rng = random.Random(7)
    vals = [rng.uniform(0, 300) for _ in range(20000)] + [round(rng.uniform(0, 250), 1) for _ in range(5000)]
    vals += [rng.uniform(-1e-6, 1e-6) for _ in range(3000)] + [rng.uniform(-1e15, 1e15) for _ in range(3000)]
    vals += [rng.randint(0, 10 ** 17) / rng.choice([3, 7, 10, 1000]) for _ in range(5000)]
    return [s for v in vals for s in (repr(v), R.java_double_to_string(v))]


def test_host_parser_is_correctly_rounded():
    """Shortest-repr strings (Python repr, Java Double.toString), 17-digit cases, exact halfway cases, both exponent
    spellings -- against float(); out-of-range exponents and malformed text are flagged, never mis-parsed."""
    for s in _corpus() + EDGE_NUMBERS:
        got, st = _parse(s.encode())
        assert st == 0 and _same_bits(got, float(s)), s
    for s, want in NON_FINITE:
        got, st = _parse(s.encode())
        assert st == 0 and (math.isnan(got) if math.isnan(want) else got == want)
    for s in MALFORMED:
        assert _parse(s.encode())[1] == 1, s
    for s in OUT_OF_RANGE:
        got, st = _parse(s.encode())
        assert st == 2 and math.isnan(got), s            # outside the supported range: flagged


def test_java_double_formatting_round_trips():
    for v in [81.0, 80.4, 1e-5, 1.5e-4, 0.001, 9999999.0, 1e7, 12345678.9, 100.0, 0.30000000000000004, 123456789012.0]:
        assert float(R.java_double_to_string(v)) == v
    assert R.java_double_to_string(1e-5) == "1.0E-5" and R.java_double_to_string(1e7) == "1.0E7"
    assert R.array_message("p000194", 3, [81.0, 80.4]) == (b"p000194_3", b"[81.0,80.4]")


def test_binary_frame_round_trip_and_validation():
    rng = np.random.default_rng(0)
    adc = rng.integers(-500, 3000, size=(3, 2, 7)).astype(np.int16)
    f = S.pack_frame([194, 195, 196], adc, first_index=120)
    assert len(f) == 32 + 12 + 4 + adc.nbytes
    ids, smp, first, grid = S.unpack_frame(f)
    assert list(ids) == [194, 195, 196] and np.array_equal(smp, adc) and first == 120 and not grid
    pts = rng.normal(80, 5, size=(2, 12, 10))
    ids, smp, first, grid = S.unpack_frame(S.pack_frame([1, 2], pts, first_index=7, grid_points=True))
    assert np.array_equal(smp, pts) and grid and first == 7
    with pytest.raises(RuntimeError):
        S.unpack_frame(f[:-2])                           # truncated
    with pytest.raises(RuntimeError):
        S.unpack_frame(b"XXXX" + f[4:])                  # bad magic
    with pytest.raises(ValueError):
        S.pack_frame([1], adc)


def test_binary_frame_header_counts_cannot_wrap_the_size_check():
    """An untrusted header whose counts multiply to 2^64 bytes (2^24 patients x 2^31 samples x 64 signals x 8 bytes)
    must not pass the length check of a 64 MB frame: the size is formed in 128-bit arithmetic."""
    lib = capi.load_library()
    n_pat, n_new, n_sig = 1 << 24, 1 << 31, 64
    head = struct.pack("<IHHIIIIQ", capi.FRAME_MAGIC, 1, capi.SAMPLES_F64, n_pat, n_new, n_sig, 0, 0)
    assert (8 * n_pat * n_new * n_sig) % (1 << 64) == 0
    frame = head + bytes(4 * n_pat)                       # header + ids: exactly the size a wrapped product describes
    buf = ctypes.create_string_buffer(frame, len(frame))
    hd, a, b = capi.FrameHeader(), ctypes.c_int64(0), ctypes.c_int64(0)
    rc = lib.b2cnn_frame_check(ctypes.addressof(buf), len(frame), ctypes.byref(hd), ctypes.byref(a), ctypes.byref(b))
    assert rc == capi.EINVAL and "header describes" in capi.last_error()


# ------------------------------------------------------------------------------------------------------ GPU
@pytest.mark.gpu
def test_gpu_decoder_rebuilds_the_physical_record_from_sendstream_messages():
    """All 6500 messages of p000194 in arrival order -> one device call -> the [1625, 4] fp64 frame == record.physical."""
    g, rec = _record()
    sel = S.selected_signals(rec)
    phys = rec.physical[:, sel]
    msgs = R.sample_messages(phys, [rec.names[i] for i in sel], "p000194-2112-05-23-14-34n")
    rows = np.repeat(np.arange(1625), 4)                 # message t belongs to sample t // 4 (arrival order)
    frame, bad = S.decode_sample_messages([m[2] for m in msgs], rows, 1625, 4, "cuda:0")
    got = frame.cpu().numpy()
    assert bad == 0 and np.array_equal(np.isnan(got), np.isnan(phys))
    assert np.array_equal(got[~np.isnan(phys)].view(np.int64), phys[~np.isnan(phys)].view(np.int64))     # bit for bit
    # malformed and out-of-range messages are counted, not mis-parsed; a signal without a message stays NaN
    frame, bad = S.decode_sample_messages([b"[0, 81.0]", b"[1, oops]", b"[2 81.0]", b"[3, 1e99]", b"[9, 5.0]"], [0, 0, 0, 0, 0], 1, 4, "cuda:0")
    assert bad == 3 and frame.cpu().numpy()[0, 0] == 81.0 and np.isnan(frame.cpu().numpy()[0, 1:]).all()
    # a row outside the frame (caller error) is dropped, not written: the frame is the tail of a larger buffer here
    frame, bad = S.decode_sample_messages([b"[0, 1.0]", b"[1, 2.0]", b"[2, 3.0]"], [0, 1, -1], 1, 4, "cuda:0")
    assert bad == 0 and frame.cpu().numpy()[0, 0] == 1.0 and np.isnan(frame.cpu().numpy()[0, 1:]).all()


@pytest.mark.gpu
def test_messages_to_ring_equals_whole_record_windows():
    """sendStream messages -> device decoder -> ring buffers (one trigger = one sample at 1/60 Hz) == b2cnn_prep_windows."""
    g, rec = _record()
    sel = S.selected_signals(rec)
    msgs = R.sample_messages(rec.physical[:, sel], [rec.names[i] for i in sel], "p000194-2112-05-23-14-34n")
    whole, _ = S.assemble_windows_gpu(rec, "cuda:0")
    ring = S.PatientRing(1, 4, rec.fs, device="cuda:0")
    ring.set_signals(0, [0, 1, 2, 3])
    out = []
    for i in range(400):                                 # 400 triggers: 391 windows
        frame, bad = S.decode_sample_messages([m[2] for m in msgs[4 * i:4 * i + 4]], [0, 0, 0, 0], 1, 4, "cuda:0")
        assert bad == 0
        r = ring.push(frame.view(1, 1, 4))
        if r is not None:
            out.append(r[0][0].clone())
    assert len(out) == 391 and torch.equal(torch.stack(out), whole[:391])


@pytest.mark.gpu
def test_call_stream_array_messages_to_ring():
    """processStream's call-stream payload (12 grid points per channel and trigger as a JSON array printed by the JVM)
    -> device decoder -> ring (grid points appended as they are) == the windows cut from the pandas-built grids."""
    g, rec = _record()
    grids = g["grids"]                                   # [4][19489] from pandas (make_golden.py)
    want, _ = N.windows_from_grids(grids)
    ring = S.PatientRing(2, 10, rec.fs, device="cuda:0")
    for p in range(2):
        ring.set_signals(p, [0, 1, 2, 3])
    out = []
    for trig in range(60):
        msgs = [R.array_message("p000194", c, grids[c, 12 * trig:12 * trig + 12]) for c in range(4)]
        vals, counts, bad = S.decode_array_messages([m[1] for m in msgs], 12, "cuda:0")
        assert bad == 0 and (counts == 12).all()
        assert np.array_equal(vals.cpu().numpy(), grids[:, 12 * trig:12 * trig + 12])           # exact doubles
        pts = torch.full((2, 12, 10), float("nan"), dtype=torch.float64, device="cuda:0")
        pts[:, :, :4] = vals.t().unsqueeze(0)            # channel index from the message key "<pid>_<chan>"
        r = ring.push(pts, grid_points=True)
        if r is not None:
            out.append(r[0][0].clone())
    assert len(out) == 51
    assert torch.equal(torch.stack(out).cpu(), torch.from_numpy(want[:51].astype(np.float32)))
    vals, counts, bad = S.decode_array_messages([b"[]", b"[1.0,2.0", b'["NaN",3.5]', b"[1.0,2.0,3.0]"], 2, "cuda:0")
    c = counts.cpu().numpy()
    assert c[0] == 0 and c[1] == -1 and c[2] == 2 and c[3] == 3 and bad == 2
    assert np.isnan(vals.cpu().numpy()[2, 0]) and vals.cpu().numpy()[2, 1] == 3.5


@pytest.mark.gpu
def test_binary_frames_feed_the_ring_without_decoding():
    g, rec = _record()
    whole, _ = S.assemble_windows_gpu(rec, "cuda:0")
    ring = S.PatientRing(2, 7, rec.fs, device="cuda:0")
    for p in range(2):
        ring.set_record_signals(p, rec)
    out = []
    for i in range(200):
        frame = S.pack_frame([194, 195], np.repeat(rec.raw[None, i:i + 1], 2, axis=0), first_index=i)
        ids, smp, first, grid = S.unpack_frame(frame)
        assert first == i and list(ids) == [194, 195]
        r = ring.push(smp)
        if r is not None:
            out.append(r[0].clone())
    assert len(out) == 191 and torch.equal(torch.stack([o[1] for o in out]), whole[:191])


def _decode_pairs_raw(msgs, rows=None, frame=None, frame_rows=0, n_sig=0):
    """b2cnn_decode_sample_messages with idx_out / val_out (and optionally a caller-owned frame): (idx, val, n_bad)."""
    lib = capi.load_library()
    b, offs, n = S._message_buffer(msgs, "cuda:0")
    idx = torch.full((n,), -7, dtype=torch.int32, device="cuda:0")
    val = torch.empty((n,), dtype=torch.float64, device="cuda:0")
    bad = torch.zeros(1, dtype=torch.int32, device="cuda:0")
    rows_t = None if rows is None else torch.as_tensor(np.asarray(rows, dtype=np.int64)).to("cuda:0")
    capi.check(lib.b2cnn_decode_sample_messages(b.data_ptr(), offs.data_ptr(), n, idx.data_ptr(), val.data_ptr(),
                                                None if rows_t is None else rows_t.data_ptr(), frame, frame_rows, n_sig,
                                                bad.data_ptr(), torch.cuda.current_stream().cuda_stream), "decode")
    torch.cuda.synchronize()
    return idx.cpu().numpy(), val.cpu().numpy(), int(bad.item())


def _float(s: str) -> float:
    """float() of a message value; Spark's quoted non-finite doubles unquoted, null = missing."""
    return math.nan if s == "null" else float(s.strip('"'))


def _same_values(got: np.ndarray, want: np.ndarray) -> bool:
    nan = np.isnan(want)
    return bool(np.array_equal(np.isnan(got), nan) and np.array_equal(got[~nan].view(np.int64), want[~nan].view(np.int64)))


@pytest.mark.gpu
def test_gpu_decoders_equal_float_on_the_whole_parser_corpus():
    """The nvcc build of the parser (128-bit division, __clzll, device ldexp) on every string the host build is checked
    with: each of 72 000 shortest-repr strings plus the edge, non-finite, out-of-range and malformed cases, once through
    each device kernel in one call.  Values match float() bit for bit; a message is flagged exactly when the host build
    flags the string, and the flagged count is n_bad."""
    strings = _corpus() + EDGE_NUMBERS + [s for s, _ in NON_FINITE] + OUT_OF_RANGE + ["abc", "1e", "--1", "0x10", "+-1", ".", "e5"]
    host = [_parse(s.encode()) for s in strings]
    ok = np.array([st == 0 for _, st in host])
    assert ok.sum() == len(strings) - len(OUT_OF_RANGE) - 7
    want = np.array([_float(s) if o else math.nan for s, o in zip(strings, ok)])
    assert _same_values(np.array([v for v, _ in host])[ok], want[ok])
    # [i, val] messages, the index cycling through 0 .. 9
    idx, val, bad = _decode_pairs_raw([f"[{t % 10}, {s}]".encode() for t, s in enumerate(strings)])
    assert bad == (~ok).sum()
    assert np.array_equal(idx, np.where(ok, np.arange(len(strings)) % 10, -1))
    assert _same_values(val, want)
    # one-element arrays
    vals, counts, bad = S.decode_array_messages([f"[{s}]".encode() for s in strings], 1, "cuda:0")
    assert bad == (~ok).sum()
    assert np.array_equal(counts.cpu().numpy(), np.where(ok, 1, -1))
    assert _same_values(vals.cpu().numpy()[:, 0], want)
    # and call-stream messages of twelve Double.toString values each (bin/processStream.py:128)
    js = [R.java_double_to_string(float(v)) for v in want[ok][:12 * 3000]]
    msgs = ["[" + ",".join(js[12 * m:12 * m + 12]) + "]" for m in range(len(js) // 12)]
    vals, counts, bad = S.decode_array_messages([m.encode() for m in msgs], 12, "cuda:0")
    assert bad == 0 and (counts.cpu().numpy() == 12).all()
    assert _same_values(vals.cpu().numpy().ravel(), np.array([_float(s) for s in js]))


@pytest.mark.gpu
def test_gpu_pair_decoder_flags_indices_that_do_not_fit():
    """The signal index is read in full: one that an int32 cannot hold is malformed (counted, idx -1, NaN), never
    truncated to its leading digits."""
    msgs = [b"[1234567, 5.0]", b"[2147483647, 1.0]", b"[2147483648, 1.0]", b"[99999999999999999999, 2.0]", b"[100000, 3.0]",
            b"[0000000000003, 4.0]"]
    idx, val, bad = _decode_pairs_raw(msgs)
    assert list(idx) == [1234567, 2147483647, -1, -1, 100000, 3] and bad == 2
    assert list(val[[0, 1, 4, 5]]) == [5.0, 1.0, 3.0, 4.0] and np.isnan(val[[2, 3]]).all()


@pytest.mark.gpu
def test_gpu_decoders_on_empty_messages_whitespace_and_truncation():
    """What json.loads accepts -- whitespace between tokens, quoted non-finite values -- decodes; an empty message, a
    missing value or bracket, or anything after the closing bracket is malformed; arrays longer than max_vals keep
    their first max_vals values, report the full count and are counted in n_bad."""
    nan, inf = math.nan, math.inf
    pairs = [(b"", None), (b"[]", None), (b"[0]", None), (b"[0,]", None), (b"[, 1.0]", None), (b"[0, 1.0", None),
             (b" [ 1 , 2.5 ] ", (1, 2.5)), (b"\t[2,\t-3.25\t]\n", (2, -3.25)), (b"[3,\r\n1e2]", (3, 100.0)),
             (b'[4, "NaN"]', (4, nan)), (b'[5, "Infinity"]', (5, inf)), (b'[6, "-Infinity"]', (6, -inf)), (b"[7, null]", (7, nan)),
             (b"[8, -Infinity]", (8, -inf)), (b"[0, 1.0] x", None), (b"[0, 1.0]]", None), (b"[-1, 1.0]", None), (b"[1.5, 2.0]", None)]
    idx, val, bad = _decode_pairs_raw([m for m, _ in pairs])
    assert bad == sum(w is None for _, w in pairs)
    for t, (m, w) in enumerate(pairs):
        wi, wv = w if w is not None else (-1, nan)
        assert idx[t] == wi and _same_values(val[t:t + 1], np.array([wv])), m
    arrays = [(b"", -1, []), (b"[]", 0, []), (b" [ ] ", 0, []), (b"[\t1.0 ,\n2.0\r]", 2, [1.0, 2.0]),
              (b'["NaN","Infinity","-Infinity"]', 3, [nan, inf, -inf]), (b"[1.0,2.0,3.0,4.0,5.0]", 5, [1.0, 2.0, 3.0]),
              (b"[1.0,,2.0]", -1, []), (b"[1.0] 7", -1, []), (b"[1.0", -1, []), (b"1.0", -1, []), (b"[1.0,2.0,3.0]", 3, [1.0, 2.0, 3.0]),
              (b"[1e28]", -1, []), (b"[0.5, null]", 2, [0.5, nan])]
    vals, counts, bad = S.decode_array_messages([m for m, _, _ in arrays], 3, "cuda:0")
    vals, counts = vals.cpu().numpy(), counts.cpu().numpy()
    assert bad == sum(c < 0 or c > 3 for _, c, _ in arrays)
    for t, (m, c, v) in enumerate(arrays):
        assert counts[t] == c, m
        assert _same_values(vals[t], np.array(v + [nan] * (3 - len(v)))), m
    vals, counts, bad = S.decode_array_messages([], 3, "cuda:0")
    assert vals.shape == (0, 3) and bad == 0


@pytest.mark.gpu
def test_gpu_frame_scatter_stays_inside_the_frame():
    """The frame is rows 1 .. 3 of a larger buffer: messages with rows or signal indices outside it write nothing, the
    frame is NaN where no message landed, and the rows around it keep their contents."""
    buf = torch.full((6, 4), 7.0, dtype=torch.float64, device="cuda:0")
    msgs = [(b"[0, 1.0]", 0), (b"[3, 2.0]", 2), (b"[4, 3.0]", 0), (b"[0, 4.0]", 3), (b"[0, 5.0]", -1), (b"[1, 6.0]", 1),
            (b"[99999999999, 7.0]", 1), (b"[2, oops]", 1), (b"[2147483647, 8.0]", 0), (b"[1, 9.0]", 1 << 40), (b"[2, -0.0]", 0)]
    idx, val, bad = _decode_pairs_raw([m for m, _ in msgs], rows=[r for _, r in msgs], frame=buf[1].data_ptr(), frame_rows=3, n_sig=4)
    assert bad == 2 and list(idx) == [0, 3, 4, 0, 0, 1, -1, -1, 2147483647, 1, 2]
    want = np.full((3, 4), np.nan)
    want[0, 0], want[2, 3], want[1, 1], want[0, 2] = 1.0, 2.0, 6.0, -0.0
    got = buf.cpu().numpy()
    assert _same_values(got[1:4].ravel(), want.ravel())
    assert (got[0] == 7.0).all() and (got[4:] == 7.0).all()
