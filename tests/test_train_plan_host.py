"""CPU: the grids and the workspace of a training shape (csrc/b2cnn_train.cu: train_plan).  b2cnn_train_workspace_bytes is
one layout for every L_out (f, pre0, the scan's records, da0, d f and one region of partial sums); the conv backward
runs up to 8 windows per CTA, fewer where B x tiles would leave it under 1024 CTAs; and a geometry whose conv tile does
not fit shared memory is refused before any launch."""
import ctypes

import pytest

import tskd_b200
from tskd_b200 import capi
from tskd_b200.arch import ArchConfig

T, WIN, BWD_CTAS, SLICE, CHUNKS = 128, 8, 1024, 1024, 16
SMEM_MAX = 227 * 1024


def _r64(n):
    return (n + 63) // 64 * 64


def _win(B, tiles):
    """windows per CTA of the conv backward"""
    return min(max(-(-B * tiles // BWD_CTAS), 1), WIN)


def _floats(a: ArchConfig, B):
    L = a.l_out
    tiles, slices = -(-L // T), -(-L // SLICE)
    chunk = -(-B // CHUNKS)
    chunks, groups = -(-B // chunk), -(-B // _win(B, tiles))
    n_conv = 4 * a.in_channels * a.k1 + 4 + 4 * a.k2 + 1
    part = max(slices * B * 64, chunks * 64 * L, tiles * groups * n_conv)
    return sum(_r64(n) for n in [B * L, B * 64, B * 128, B * 32, B * 32, B, B, B * 64, B * L, part])


def _smem_bwd(a: ArchConfig):
    """bytes of the conv backward's tile: min(128, L_out) features and their receptive span"""
    r4 = lambda n: (n + 3) // 4 * 4
    C, K1, K2, PK, PS, t = a.in_channels, a.k1, a.k2, a.pool_k, a.pool_s, min(T, a.l_out)
    n2 = PS * (t - 1) + PK + PS - 1
    np1 = n2 + K2 - 1
    n1 = PS * (np1 - 1) + PK + PS - 1
    nx = n1 + K1 - 1
    fwd = r4(4 * C * K1) + 4 + r4(4 * K2) + 4 + C * r4(nx) + r4(4 * n1) + 4 * r4(np1) + r4(n2)
    return 4 * (fwd + r4(t) + r4(n2) + 4 * r4(np1) + r4(4 * n1) + r4(4 * C * K1 + 4 + 4 * K2 + 1))


def _bytes(a, B):
    cfg = capi.make_config(a)
    return int(capi.load_library().b2cnn_train_workspace_bytes(ctypes.byref(cfg), B))


@pytest.mark.parametrize("kind,C,W", [("mycnn5", 10, 120), ("mycnn2", 7, 120), ("mycnn5", 3, 1528), ("mycnn3", 3, 1500),
                                      ("mycnn5", 3, 7504), ("mycnn5", 3, 75000)])
@pytest.mark.parametrize("B", [1, 12, 2048])
def test_one_workspace_layout_for_every_window(kind, C, W, B):
    a = tskd_b200.ARCH_PRESETS[kind].with_shape(C, W)
    assert _bytes(a, B) == 4 * _floats(a, B)


def test_windows_per_cta():
    assert [_win(B, 1) for B in (1, 32, 256, 1024, 1025, 2048, 8192, 100000)] == [1, 1, 1, 1, 2, 2, 8, 8]
    assert _win(256, 147) == _win(4096, 147) == WIN                       # [B,3,75000]: 147 tiles, B x tiles >= 37 632
    assert _win(3, 147) == 1 and _win(10, 15) == 1


def test_short_workspace_by_hand():
    a = tskd_b200.ARCH_PRESETS["mycnn5"]
    assert (a.l_out, 4 * 10 * 10 + 4 + 4 * 5 + 1) == (25, 425)
    # [32,10,120]: one window per CTA, so 32 partial rows of 425; f and d f 800 each, pre0 2048, acts 4096, cs / hs 1024,
    # lin / z 64, da0 2048, and max(1 slice x 32 x 64, 16 chunks x 64 x 25, 32 x 425) = 25600
    assert _bytes(a, 32) == 4 * (832 + 2048 + 4096 + 1024 + 1024 + 64 + 64 + 2048 + 832 + 25600) == 4 * _floats(a, 32)
    # [2048,10,120]: two windows per CTA, 1024 partial rows
    assert _bytes(a, 2048) == 4 * (2 * 51200 + 2 * 131072 + 262144 + 2 * 65536 + 2 * 2048 + 1024 * 425) == 4 * _floats(a, 2048)


def test_long_workspace_by_hand():
    a = tskd_b200.ARCH_PRESETS["mycnn5"].with_shape(3, 7504)
    assert a.l_out == 1871
    # B = 10: f and d f 18752 each, pre0 640, acts 1280, cs 320, hs 320, lin 64, z 64, da0 640, and the partial sums:
    # max(2 slices x 10 x 64, 10 chunks x 64 x 1871, 15 tiles x 10 groups of one window x 145) = 1197440
    assert _bytes(a, 10) == 4 * 1238272 == 4 * _floats(a, 10)
    big = tskd_b200.ARCH_PRESETS["mycnn5"].with_shape(3, 75000)
    assert big.l_out == 18745
    # [4096, 3, 75000]: 2 x 76779520 (f, d f) + 19194880 (16 chunks x 64 x 18745) + 1318912 for everything per window
    assert _bytes(big, 4096) == 4 * 174072832 == 4 * _floats(big, 4096)


def test_across_the_old_plan_boundary():
    """L_out = 1023 and 1024 once had different layouts; now both follow one formula"""
    p = tskd_b200.ARCH_PRESETS["mycnn5"]
    below, at = p.with_shape(3, 4112), p.with_shape(3, 4116)
    assert (below.l_out, at.l_out) == (1023, 1024)
    for B in (1, 7, 64, 4096, 100000):
        assert _bytes(below, B) == 4 * _floats(below, B)
        assert _bytes(at, B) == 4 * _floats(at, B)
    # B = 64: 8 tiles, one window per CTA; f, d f 65472 / 65536, partial sums max(64 x 64, 16 x 64 x L, 512 x 145)
    assert _bytes(below, 64) == 4 * (2 * 65472 + 4096 + 8192 + 2048 + 2048 + 64 + 64 + 4096 + 1047552)
    assert _bytes(at, 64) == 4 * (2 * 65536 + 4096 + 8192 + 2048 + 2048 + 64 + 64 + 4096 + 1048576)
    assert _bytes(at, 0) == -1


def _forward_rc(a, ws):
    """b2cnn_train_forward's argument checks; with a workspace below the shape's size nothing is launched"""
    lib = capi.load_library()
    cfg = capi.make_config(a)
    p = ctypes.c_void_p(1)
    return lib.b2cnn_train_forward(ctypes.byref(cfg), p, p, 4, p, capi.MODE_SEQUENCE, None, None, p, p, ws, None)


@pytest.mark.parametrize("W,first_refused", [(120, 278), (1528, 83)])
def test_channels_beyond_a_conv_tile_are_refused(W, first_refused):
    p = tskd_b200.ARCH_PRESETS["mycnn5"]
    ok, refused = p.with_shape(first_refused - 1, W), p.with_shape(first_refused, W)
    assert _smem_bwd(ok) <= SMEM_MAX < _smem_bwd(refused)
    assert _smem_bwd(p.with_shape(3, 75000)) == 35488 and _smem_bwd(p) == 14352
    # a workspace one byte short: the shape that fits stops there, the other one before
    assert _forward_rc(ok, _bytes(ok, 4) - 1) == capi.ESTATE and "workspace" in capi.last_error()
    assert _forward_rc(refused, _bytes(refused, 4) - 1) == capi.EINVAL and "shared memory" in capi.last_error()


def test_backward_ex_is_exported_and_checks_its_flags():
    lib = capi.load_library()
    assert "b2cnn_train_backward_ex" in capi.SYMBOLS and capi.TRAIN_FROZEN_CONV == 1
    cfg = capi.make_config(tskd_b200.ARCH_PRESETS["mycnn5"])
    p = ctypes.c_void_p(1)

    def bwd(flags, dx=None, ws=1 << 30):
        return lib.b2cnn_train_backward_ex(ctypes.byref(cfg), p, p, 4, p, capi.MODE_SEQUENCE, None, None, p, p, dx, None, flags, p, ws, None)
    assert bwd(2) == capi.EINVAL and "flag" in capi.last_error()
    assert bwd(capi.TRAIN_FROZEN_CONV, dx=p) == capi.EINVAL and "dx" in capi.last_error()
    need = _bytes(tskd_b200.ARCH_PRESETS["mycnn5"], 4)
    assert bwd(capi.TRAIN_FROZEN_CONV, ws=need - 1) == capi.ESTATE and "workspace" in capi.last_error()
