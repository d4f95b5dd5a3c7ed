"""CPU: training on whole recordings without a GPU -- the Python refusals, the bound _record symbols and their refusals
before any CUDA call, the record workspace layout computed by hand, the index-overflow refusal, and the oracle helper
against a per-window loop of the reference module."""
import ctypes
import math

import pytest
import torch

import tskd_b200
from tskd_b200 import capi
from tskd_b200.autograd import check_record_batch, cut_record_windows
from oracle import mycnn_torch as O
from oracle.train_ref import MaskDropout
from oracle.train_record_ref import train_reference_record

ARCH = tskd_b200.ARCH_PRESETS["mycnn5"]          # [., 10, 120], feature stride 4


def _arr(v):
    return (ctypes.c_int64 * len(v))(*v)


@pytest.mark.parametrize("kw,msg", [
    (dict(records=torch.zeros(2, 9, 400)), r"expected records \[B, 10, N\]"),
    (dict(records=torch.zeros(2, 400)), r"expected records \[B, 10, N\]"),
    (dict(records=torch.zeros(2, 10, 400, dtype=torch.float64)), "float32 or bfloat16"),
    (dict(records=torch.zeros(0, 10, 400)), "at least one recording"),
    (dict(stride=70), "positive multiple of the feature stride 4"),
    (dict(stride=0), "positive multiple"),
    (dict(stride=72.0), "stride must be an integer"),
    (dict(stride=True), "got bool"),
    (dict(age=torch.ones(3)), "one per recording"),
    (dict(window_counts=[4]), "1 entries, the batch has 2"),
    (dict(window_counts=[5, 0]), r"window_counts\[0\] = 5"),       # n_w = (400 - 120) // 72 + 1 = 4
    (dict(window_counts=[-1, 2]), r"window_counts\[0\] = -1"),
    (dict(window_counts=[0, 0]), "hold no window"),
    (dict(window_counts=[2.0, 1]), "must be an integer, got float"),
    (dict(window_counts=torch.tensor([1.0, 1.0])), "integer tensor"),
    (dict(window_counts="41"), "list, tuple or integer tensor"),
    (dict(records=torch.zeros(2, 10, 100), window_counts=None), "hold no window"),   # N < W
    (dict(records=torch.zeros(2, 10, 191), window_counts=[2, 1]), r"window_counts\[0\] = 2"),   # N too short for 2
])
def test_bad_record_arguments_are_refused_with_a_clear_message(kw, msg):
    args = dict(records=torch.zeros(2, 10, 400), stride=72, age=torch.ones(2), window_counts=[4, 2])
    args.update(kw)
    with pytest.raises(ValueError, match=msg):
        check_record_batch(ARCH, args["records"], args["stride"], args["age"], args["window_counts"])


def test_good_record_arguments():
    stride, age, counts, M, rarch = check_record_batch(ARCH, torch.zeros(3, 10, 400, dtype=torch.bfloat16), 72, 50.0, None)
    assert stride == 72 and age.numel() == 1 and list(counts) == [4, 4, 4] and M == 12
    assert (rarch.window, rarch.p1, rarch.l_out) == (400, ARCH.with_shape(10, 400).p1, 95)
    _, _, counts, M, _ = check_record_batch(ARCH, torch.zeros(3, 10, 400), 8, torch.ones(3), torch.tensor([0, 36, 1]))
    assert list(counts) == [0, 36, 1] and M == 37


def test_record_symbols_are_bound_and_declared():
    lib = capi.load_library()
    for name in ("b2cnn_train_workspace_bytes_record", "b2cnn_train_step_record", "b2cnn_train_forward_record",
                 "b2cnn_train_backward_record"):
        assert name in capi.SYMBOLS
        assert getattr(lib, name).restype is not None


def _dims(C, W, K1, K2, PK, PS):
    L1 = W - K1 + 1
    P1 = (L1 - PK) // PS + 1
    L2 = P1 - K2 + 1
    return P1, (L2 - PK) // PS + 1


def _layout_bytes(arch, B, N, counts, sequence):
    """The record workspace of b2cnn_train.cu's train_plan, by hand: every region rounded up to 64 floats."""
    C, K1, K2, PK, PS = arch.in_channels, arch.k1, arch.k2, arch.pool_k, arch.pool_s
    _, L = _dims(C, arch.window, K1, K2, PK, PS)
    _, LN = _dims(C, N, K1, K2, PK, PS)
    M = sum(counts)
    n_seq = sum(1 for c in counts if c > 0) if sequence else 0
    r = lambda n: (n + 63) // 64 * 64
    tiles = -(-LN // 128)
    win = min(8, max(1, -(-B * tiles // 1024)))
    groups = -(-B // win)
    n_conv = 4 * C * K1 + 4 + 4 * K2 + 1
    slices = -(-L // 1024)
    chunk = -(-M // 16)
    chunks = -(-M // chunk)
    head_row = 64 * 16 * 3 + 64 * 4 + 16 + 1 + 1
    seq_per = -(-n_seq // 256) if n_seq > 256 else 1
    seq_ctas = -(-n_seq // seq_per) if n_seq else 1
    part = max(slices * M * 64, chunks * 64 * L, tiles * groups * n_conv, seq_ctas * head_row if seq_ctas > 1 else 0)
    floats = (r(B * LN) + r(M * 64) + r(M * 128) + 2 * r(M * 32) + 2 * r(M) + r(M * 64) + r(B * LN) + r(part)
              + (r(2 * (n_seq + 1)) if n_seq else 0) + r(M * L) + r(2 * (B + 1)))
    return 4 * floats


@pytest.mark.parametrize("arch,B,N,S,counts,mode", [
    (ARCH, 3, 120 + 72 * 4 + 30, 72, [5, 2, 0], capi.MODE_SEQUENCE),
    (ARCH.with_shape(3, 7504), 2, 7504 + 3752 * 3, 3752, [4, 1], capi.MODE_INDEPENDENT),
])
def test_record_workspace_layout_by_hand(arch, B, N, S, counts, mode):
    lib, cfg = capi.load_library(), capi.make_config(arch)
    got = lib.b2cnn_train_workspace_bytes_record(ctypes.byref(cfg), B, N, S, _arr(counts), mode)
    assert got == _layout_bytes(arch, B, N, counts, mode == capi.MODE_SEQUENCE)


def test_train_record_calls_refuse_bad_arguments_before_any_cuda_call():
    # fake, never dereferenced device pointers: an EINVAL here proves the arguments are checked before the first CUDA call
    lib, cfg = capi.load_library(), capi.make_config(ARCH)
    p = ctypes.c_void_p(16)
    opt = capi.Adam(1e-3, 0.9, 0.999, 1e-8)
    B, N = 2, 400
    bad = [  # (N, stride, counts, mode, the message)
        (N, 70, _arr([1, 1]), 1, "stride"),
        (N, 0, _arr([1, 1]), 1, "stride"),
        (N, 72, _arr([5, 1]), 1, "window count"),
        (N, 72, _arr([-1, 1]), 1, "window count"),
        (N, 72, _arr([0, 0]), 1, "add up to 0"),
        (100, 72, _arr([1, 0]), 1, "window count"),          # N < W: no window fits
        (N, 72, None, 1, "window_counts"),
        (N, 72, _arr([1, 1]), 2, "mode"),
        (2 ** 31, 72, _arr([1, 1]), 1, "2^31 - 1"),          # samples indexed with int in the kernels
    ]
    for n, s, counts, mode, msg in bad:
        assert lib.b2cnn_train_workspace_bytes_record(ctypes.byref(cfg), B, n, s, counts, mode) == -1
        rc = lib.b2cnn_train_step_record(ctypes.byref(cfg), p, p, p, p, 1, ctypes.byref(opt), 1, p, B, n, s, counts, mode, p, p, None,
                                         None, None, p, p, 1 << 40, None)
        assert rc == capi.EINVAL and msg in capi.last_error(), (n, s, mode, capi.last_error())
        assert lib.b2cnn_train_forward_record(ctypes.byref(cfg), p, p, B, n, s, counts, mode, p, None, None, p, p, 1 << 40,
                                              None) == capi.EINVAL
        assert lib.b2cnn_train_backward_record(ctypes.byref(cfg), p, p, B, n, s, counts, mode, p, None, None, p, p, None, None, 0, p,
                                               1 << 40, None) == capi.EINVAL
    good = _arr([4, 2])
    # NULL records / age, a bad flag, frozen conv with d_records, a bad pos_weight: still before CUDA
    assert lib.b2cnn_train_forward_record(ctypes.byref(cfg), p, None, B, N, 72, good, 1, p, None, None, p, p, 1 << 40, None) == capi.EINVAL
    assert lib.b2cnn_train_backward_record(ctypes.byref(cfg), p, p, B, N, 72, good, 1, p, None, None, p, p, None, None, 4, p, 1 << 40,
                                           None) == capi.EINVAL
    assert lib.b2cnn_train_backward_record(ctypes.byref(cfg), p, p, B, N, 72, good, 1, p, None, None, p, p, p, None, capi.TRAIN_FROZEN_CONV,
                                           p, 1 << 40, None) == capi.EINVAL
    pw = ctypes.c_float(-1.0)
    assert lib.b2cnn_train_step_record(ctypes.byref(cfg), p, p, p, p, 1, ctypes.byref(opt), 1, p, B, N, 72, good, 1, p, p, ctypes.byref(pw),
                                       None, None, p, p, 1 << 40, None) == capi.EINVAL
    # a workspace sized by another query: B2CNN_ESTATE, still before CUDA
    need = lib.b2cnn_train_workspace_bytes_record(ctypes.byref(cfg), B, N, 72, good, 1)
    assert need > 0
    assert lib.b2cnn_train_forward_record(ctypes.byref(cfg), p, p, B, N, 72, good, 1, p, None, None, p, p, need - 1, None) == capi.ESTATE
    assert "b2cnn_train_workspace_bytes_record" in capi.last_error()
    small = lib.b2cnn_train_workspace_bytes_seq(ctypes.byref(cfg), 6, _arr([4, 2]), 2)
    assert small < need
    assert lib.b2cnn_train_forward_record(ctypes.byref(cfg), p, p, B, N, 72, good, 1, p, None, None, p, p, small, None) == capi.ESTATE


def test_index_overflow_is_refused():
    # 2^21 recordings of 4e6 samples: more conv tiles than a grid of int32 CTAs holds
    lib, cfg = capi.load_library(), capi.make_config(ARCH)
    B, N = 1 << 21, 4_000_000
    counts = (ctypes.c_int64 * B)()
    counts[0] = 1
    p = ctypes.c_void_p(16)
    assert lib.b2cnn_train_workspace_bytes_record(ctypes.byref(cfg), B, N, 72, counts, 1) == -1
    assert lib.b2cnn_train_forward_record(ctypes.byref(cfg), p, p, B, N, 72, counts, 1, p, None, None, p, p, 1 << 60, None) == capi.EINVAL
    assert "batch too large" in capi.last_error()
    assert lib.b2cnn_train_workspace_bytes_record(ctypes.byref(cfg), 1, N, 72, counts, 1) > 0          # one recording fits


@pytest.mark.parametrize("mode", ["sequence", "independent"])
def test_oracle_helper_matches_a_per_window_loop(mode):
    oarch = O.stretched(O.ARCHS["mycnn5"], 10, 120)
    ref = O.make_ref(oarch, seed=3)
    ref.dropout = MaskDropout()
    ref.train()
    g = torch.Generator().manual_seed(4)
    S, counts = 72, [3, 0, 2]
    N = 120 + 3 * S + 10
    rec = torch.randn(3, 10, N, generator=g)
    age = torch.tensor([40.0, 50.0, 70.0])
    ra = ARCH.with_shape(10, N)
    m1 = torch.bernoulli(torch.full((3, 4, ra.p1), 0.9), generator=g) / 0.9
    m2 = torch.bernoulli(torch.full((3, ra.l_out), 0.9), generator=g) / 0.9
    r = torch.randn(5, generator=g)
    out = train_reference_record(ref, rec, S, age, counts, mode, m1, m2, dz=r, dtype=torch.float32)
    # the loop: one reference call per recording (sequence) or per window (independent), windows cut by slicing
    zs = []
    for b, n in enumerate(counts):
        ws = [(rec[b:b + 1, :, w * S:w * S + 120], m1[b:b + 1, :, w * S // 2:w * S // 2 + oarch.p1],
               m2[b:b + 1, w * S // 4:w * S // 4 + oarch.l_out]) for w in range(n)]
        if not ws:
            continue
        groups = [ws] if mode == "sequence" else [[w] for w in ws]
        for grp in groups:
            ref.dropout.set(torch.cat([w[1] for w in grp]), torch.cat([w[2] for w in grp]))
            zs.append(ref(torch.cat([w[0] for w in grp]), age[b].expand(len(grp))).reshape(-1))
    want = torch.cat(zs).detach()
    assert torch.allclose(out["z"], want, rtol=1e-5, atol=1e-6)
    # d records folds the windows' dx: samples no window reads get 0, and the total equals the windows' total
    d = out["dz"]["drecords"]
    assert d.shape == rec.shape and float(d[1].abs().max()) == 0.0 and float(d[0, :, 120 + 2 * S:].abs().max()) == 0.0
    assert math.isclose(float(d.sum()), float(out["dz"]["dx"].sum()), rel_tol=1e-4, abs_tol=1e-6)
    x, c1, c2 = cut_record_windows(rec, 120, S, counts, 2, m1, m2)
    assert torch.equal(x, out["windows"]) and torch.equal(c1, out["mask1"]) and torch.equal(c2, out["mask2"])
