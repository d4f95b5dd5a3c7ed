"""CPU: B200HeadTrainer without a GPU -- its refusals, raised before any library call; the C symbols declared, listed
in capi and bound with their argument types; and the workspace size of b2cnn_train_heads_workspace_bytes worked out by
hand from the layout DESIGN.md §8 states (f once, K copies of every per-row region, one partial-sum region)."""
import copy
import ctypes
import math
import os
import re
from dataclasses import replace

import pytest
import torch

import tskd_b200
from conftest import ROOT
from tskd_b200 import capi

NEW = ("b2cnn_train_heads_workspace_bytes", "b2cnn_train_heads_step", "b2cnn_train_heads_workspace_bytes_record",
       "b2cnn_train_heads_step_record")
ARCH = tskd_b200.ARCH_PRESETS["mycnn5"]


@pytest.fixture
def no_library(monkeypatch):
    """every check below must fire before the library is loaded"""
    def refuse():
        raise AssertionError("the library was reached")
    monkeypatch.setattr(capi, "load_library", refuse)


def _heads(n, seed=0):
    torch.manual_seed(seed)
    m = tskd_b200.B200MyCNN(ARCH)
    hs = []
    for i in range(n):
        h = copy.deepcopy(m)
        with torch.no_grad():
            h.lstm.weight_hh_l0.add_(0.01 * (i + 1))
        hs.append(h)
    return m, hs


def test_symbols_declared_listed_and_bound():
    header = open(os.path.join(ROOT, "include", "b2cnn.h")).read()
    for name in NEW:
        assert name in capi.SYMBOLS
        assert re.search(rf"\b{name}\s*\(", header), name
    if not os.path.exists(capi.lib_path()):
        pytest.skip("libb2cnn.so not built")
    lib = capi.load_library()
    c_i64, c_int, c_i32, c_vp = ctypes.c_int64, ctypes.c_int, ctypes.c_int32, ctypes.c_void_p
    cfgp, adamp = ctypes.POINTER(capi.Config), ctypes.POINTER(capi.Adam)
    assert lib.b2cnn_train_heads_workspace_bytes.argtypes == [cfgp, c_i32, c_i64, c_vp, c_i64]
    assert lib.b2cnn_train_heads_workspace_bytes.restype == c_i64
    assert lib.b2cnn_train_heads_step.argtypes == [cfgp, c_vp, c_i32, c_vp, c_vp, c_vp, c_vp, c_vp, c_i64, adamp, c_int, c_vp, c_i64,
                                                   c_vp, c_vp, c_vp, c_int, c_vp, c_i64, c_vp, c_vp, c_vp, c_vp, c_i64, c_vp]
    assert lib.b2cnn_train_heads_step.restype == c_int
    assert lib.b2cnn_train_heads_workspace_bytes_record.argtypes == [cfgp, c_i32, c_i64, c_i64, c_i64, c_vp, c_int]
    assert lib.b2cnn_train_heads_workspace_bytes_record.restype == c_i64
    assert lib.b2cnn_train_heads_step_record.argtypes == [cfgp, c_vp, c_i32, c_vp, c_vp, c_vp, c_vp, c_vp, c_i64, adamp, c_int, c_vp,
                                                          c_i64, c_i64, c_i64, c_vp, c_int, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp,
                                                          c_i64, c_vp]
    assert lib.b2cnn_train_heads_step_record.restype == c_int


def test_refusals_before_the_library(no_library):
    m, hs = _heads(9)
    with pytest.raises(TypeError, match="B200MyCNN"):
        tskd_b200.B200HeadTrainer(object(), hs[:1])
    with pytest.raises(TypeError, match="list of B200MyCNN"):
        tskd_b200.B200HeadTrainer(m, hs[0])
    with pytest.raises(ValueError, match="at least one head"):
        tskd_b200.B200HeadTrainer(m, [])
    with pytest.raises(ValueError, match="at most 8 heads"):
        tskd_b200.B200HeadTrainer(m, hs)
    with pytest.raises(TypeError, match=r"heads\[1\]"):
        tskd_b200.B200HeadTrainer(m, [hs[0], "head"])
    with pytest.raises(ValueError, match="distinct"):
        tskd_b200.B200HeadTrainer(m, [hs[0], hs[1], hs[0]])
    other = tskd_b200.B200MyCNN(ARCH.with_shape(10, 240))
    with pytest.raises(ValueError, match=r"heads\[1\] differs from the model in"):
        tskd_b200.B200HeadTrainer(m, [hs[0], other])
    bad = copy.deepcopy(hs[2])
    with torch.no_grad():
        bad.conv2.bias.add_(1e-6)
    with pytest.raises(ValueError, match=r"heads\[2\] differs from the model's front end in conv2.bias"):
        tskd_b200.B200HeadTrainer(m, [hs[0], hs[1], bad])
    with pytest.raises(ValueError, match="one float or 3 floats"):
        tskd_b200.B200HeadTrainer(m, hs[:3], lr=[1e-3, 1e-4])
    with pytest.raises(ValueError, match="lr"):
        tskd_b200.B200HeadTrainer(m, hs[:2], lr=[1e-3, math.nan])
    with pytest.raises(ValueError, match="mode"):
        tskd_b200.B200HeadTrainer(m, hs[:2], mode="batch")
    with pytest.raises(ValueError, match="dropout"):
        tskd_b200.B200HeadTrainer(m, hs[:2], dropout=1.0)
    with pytest.raises(ValueError, match="pos_weight"):
        tskd_b200.B200HeadTrainer(m, hs[:2], pos_weight=-1.0)
    affine = tskd_b200.B200MyCNN(replace(ARCH, affine=True))
    with pytest.raises(NotImplementedError):
        tskd_b200.B200HeadTrainer(affine, [affine])
    # everything valid on a CPU model: the device is the last refusal, still before the library
    with pytest.raises(RuntimeError, match="CUDA device"):
        tskd_b200.B200HeadTrainer(m, [m] + hs[:2], lr=[1e-3, 1e-4, 1e-5])


def _r64(n):
    return (n + 63) // 64 * 64


def _by_hand(B, L, K):
    """b2cnn_train_heads_workspace_bytes for B windows of L features and K heads, in a mode (no sequence offsets):
    f [B][L] once; per head pre0 [B][64], acts [B][2][64], cs and hs [B][2][16], lin and z [B], da0 [B][64]; one
    partial-sum region holding the larger of the projection's split-K partials [slices][K][B][64] and dW_ih_l0's batch-
    chunk partials [chunks][K][64][L].  Every region starts on a 64-float boundary."""
    slices = (L + 1023) // 1024
    chunk = (B + 15) // 16
    chunks = (B + chunk - 1) // chunk
    regions = [B * L, K * B * 64, K * B * 128, K * B * 32, K * B * 32, K * B, K * B, K * B * 64,
               max(slices * K * B * 64, chunks * K * 64 * L)]
    return 4 * sum(_r64(n) for n in regions)


@pytest.mark.parametrize("B,C,W,L", [(32, 10, 120, 25), (4096, 3, 75000, 18745)])
@pytest.mark.parametrize("K", [1, 8])
def test_workspace_size_by_hand(B, C, W, L, K):
    if not os.path.exists(capi.lib_path()):
        pytest.skip("libb2cnn.so not built")
    arch = ARCH.with_shape(C, W)
    assert arch.l_out == L
    lib = capi.load_library()
    cfg = capi.make_config(arch)
    got = lib.b2cnn_train_heads_workspace_bytes(ctypes.byref(cfg), K, B, None, 0)
    assert got == _by_hand(B, L, K), (got, _by_hand(B, L, K))
    # the numbers themselves, so a change of the formula shows here too
    want = {(32, 1): 4 * (832 + 2048 + 4096 + 1024 + 1024 + 64 + 64 + 2048 + 25600),
            (32, 8): 4 * (832 + 8 * 2048 + 8 * 4096 + 8 * 1024 + 8 * 1024 + 256 + 256 + 8 * 2048 + 8 * 25600),
            (4096, 1): 4 * (4096 * 18745 + 4096 * 64 + 4096 * 128 + 4096 * 32 * 2 + 4096 * 2 + 4096 * 64 + 16 * 64 * 18745),
            (4096, 8): 4 * (4096 * 18745 + 8 * 4096 * (64 + 128 + 64 + 2 + 64) + 16 * 8 * 64 * 18745)}[(B, K)]
    assert got == want, (got, want)


def test_workspace_refuses_bad_head_counts():
    if not os.path.exists(capi.lib_path()):
        pytest.skip("libb2cnn.so not built")
    lib = capi.load_library()
    cfg = capi.make_config(ARCH)
    for K in (0, -1, 9):
        assert lib.b2cnn_train_heads_workspace_bytes(ctypes.byref(cfg), K, 32, None, 0) == -1
    counts = (ctypes.c_int64 * 2)(1, 0)
    assert lib.b2cnn_train_heads_workspace_bytes_record(ctypes.byref(cfg), 9, 2, 120, 8, counts, capi.MODE_SEQUENCE) == -1
    assert lib.b2cnn_train_heads_workspace_bytes_record(ctypes.byref(cfg), 2, 2, 120, 8, counts, capi.MODE_SEQUENCE) > 0
