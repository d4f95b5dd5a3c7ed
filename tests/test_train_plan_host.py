"""CPU: which training kernels a shape runs is decided from L_out alone (csrc/b2cnn_train.cu: train_plan), and
b2cnn_train_workspace_bytes is that plan's size: the one-CTA-per-window layout below L_out = 1024, the tiled layout
(f, pre0, the scan's records, da0, d f and one region of partial sums) from there on."""
import ctypes

import pytest

import tskd_b200
from tskd_b200 import capi
from tskd_b200.arch import ArchConfig

LONG_MIN_L, T, WIN, SLICE, CHUNKS = 1024, 128, 8, 1024, 16


def _r64(n):
    return (n + 63) // 64 * 64


def _short_floats(a: ArchConfig, B):
    """the workspace of the per-window kernels: c1, p1, c2, f, acts, cs, hs, lin, z, da0, dfeat, dc2, dd1, dc1"""
    parts = [B * 4 * a.l1, B * 4 * a.p1, B * a.l2, B * a.l_out, B * 128, B * 32, B * 32, B, B, B * 64,
             B * a.l_out, B * a.l2, B * 4 * a.p1, B * 4 * a.l1]
    return sum(_r64(n) for n in parts)


def _long_floats(a: ArchConfig, B):
    L = a.l_out
    tiles, slices = -(-L // T), -(-L // SLICE)
    chunk = -(-B // CHUNKS)
    chunks, groups = -(-B // chunk), -(-B // WIN)
    n_conv = 4 * a.in_channels * a.k1 + 4 + 4 * a.k2 + 1
    part = max(slices * B * 64, chunks * 64 * L, tiles * groups * n_conv)
    return sum(_r64(n) for n in [B * L, B * 64, B * 128, B * 32, B * 32, B, B, B * 64, B * L, part])


def _bytes(a, B):
    cfg = capi.make_config(a)
    return int(capi.load_library().b2cnn_train_workspace_bytes(ctypes.byref(cfg), B))


@pytest.mark.parametrize("kind,C,W", [("mycnn5", 10, 120), ("mycnn2", 7, 120), ("mycnn5", 3, 1528), ("mycnn3", 3, 1500)])
@pytest.mark.parametrize("B", [1, 12, 2048])
def test_short_windows_keep_their_workspace(kind, C, W, B):
    a = tskd_b200.ARCH_PRESETS[kind].with_shape(C, W)
    assert a.l_out < LONG_MIN_L
    assert _bytes(a, B) == 4 * _short_floats(a, B)


def test_long_workspace_by_hand():
    a = tskd_b200.ARCH_PRESETS["mycnn5"].with_shape(3, 7504)
    assert a.l_out == 1871
    # B = 10: f and d f 18752 each, pre0 640, acts 1280, cs 320, hs 320, lin 64, z 64, da0 640, and the partial sums:
    # max(2 slices x 10 x 64, 10 chunks x 64 x 1871, 15 tiles x 2 groups x 145) = 1197440
    assert _bytes(a, 10) == 4 * 1238272 == 4 * _long_floats(a, 10)
    big = tskd_b200.ARCH_PRESETS["mycnn5"].with_shape(3, 75000)
    assert big.l_out == 18745
    # [4096, 3, 75000]: 2 x 76779520 (f, d f) + 19194880 (16 chunks x 64 x 18745) + 1318912 for everything per window
    assert _bytes(big, 4096) == 4 * 174072832 == 4 * _long_floats(big, 4096)
    assert 4 * _short_floats(big, 4096) > 16e9                      # what the per-window kernels would have asked for


def test_the_plan_depends_on_l_out_only():
    p = tskd_b200.ARCH_PRESETS["mycnn5"]
    below, at = p.with_shape(3, 4112), p.with_shape(3, 4116)
    assert (below.l_out, at.l_out) == (LONG_MIN_L - 1, LONG_MIN_L)
    for B in (1, 7, 64, 4096, 100000):
        assert _bytes(below, B) == 4 * _short_floats(below, B)
        assert _bytes(at, B) == 4 * _long_floats(at, B)
    assert _bytes(at, 0) == -1


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
