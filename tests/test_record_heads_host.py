"""CPU: predict_record(heads=[...]) without a GPU -- the refusals of the candidate heads and of the per-model state,
raised before any library call; the C symbols declared, listed in capi and bound with their argument types."""
import ctypes
import os
import re
from dataclasses import replace

import pytest
import torch

import tskd_b200
from conftest import ROOT
from tskd_b200 import capi
from tskd_b200.model import check_record_state

NEW = ("b2cnn_record_workspace_bytes_heads", "b2cnn_score_record_heads")
ARCH = tskd_b200.ARCH_PRESETS["mycnn5"].with_shape(3, 7504)


def _model(**change):
    return tskd_b200.B200MyCNN(replace(ARCH, **change))


@pytest.fixture
def no_library(monkeypatch):
    """every check below must fire before the library is loaded"""
    def refuse():
        raise AssertionError("the library was reached")
    monkeypatch.setattr(capi, "load_library", refuse)


def test_symbols_declared_listed_and_bound():
    header = open(os.path.join(ROOT, "include", "b2cnn.h")).read()
    for name in NEW:
        assert name in capi.SYMBOLS
        assert re.search(rf"\b{name}\s*\(", header), name
    if not os.path.exists(capi.lib_path()):
        pytest.skip("libb2cnn.so not built")
    lib = capi.load_library()
    c_i64, c_int, c_i32, c_vp = ctypes.c_int64, ctypes.c_int, ctypes.c_int32, ctypes.c_void_p
    assert lib.b2cnn_record_workspace_bytes_heads.argtypes == [c_vp, c_i32, c_i64, c_i64, c_i64, c_i64, c_int, c_int, c_int]
    assert lib.b2cnn_record_workspace_bytes_heads.restype == c_i64
    assert lib.b2cnn_score_record_heads.argtypes == [c_vp, c_vp, c_i32, c_vp, c_int, c_i64, c_i64, c_i64, c_i64, c_int, c_int, c_vp,
                                                     c_i64, c_int, c_vp, c_vp, c_vp, c_vp, c_i64, c_vp]
    assert lib.b2cnn_score_record_heads.restype == c_int


def test_head_refusals_before_the_library(no_library):
    m = _model()
    x = torch.zeros(2, 3, 9000, dtype=torch.bfloat16)
    for bad in (_model(), "heads", torch.zeros(3), 3):
        with pytest.raises(TypeError, match="predict_record takes a list of B200MyCNN models"):
            m.predict_record(x, 8, heads=bad)
    with pytest.raises(TypeError, match=r"heads\[1\] is a Linear"):
        m.predict_record(x, 8, heads=[_model(), torch.nn.Linear(2, 2)])
    with pytest.raises(ValueError, match="at most 8 heads, got 9"):
        m.predict_record(x, 8, heads=[_model() for _ in range(9)])
    for change, field in (({"window": 7508}, "window"), ({"act": "relu"}, "act"), ({"k1": 9}, "k1"), ({"affine": True}, "affine")):
        with pytest.raises(ValueError, match=rf"heads\[0\] differs from the model in .*{field}"):
            m.predict_record(x, 8, heads=[_model(**change)])
    other = _model()
    other.to(torch.device("meta"))
    with pytest.raises(ValueError, match=r"heads\[0\] is on meta, the model on cpu"):
        m.predict_record(x, 8, heads=[other])
    # the record arguments are still checked first
    with pytest.raises(ValueError, match="stride"):
        m.predict_record(x, 6, heads=[_model(age_coef=1e-3)])


def test_state_shape_with_heads(no_library):
    m = _model()
    x = torch.zeros(2, 3, 9000, dtype=torch.bfloat16)
    hs = [_model(age_coef=1e-3), _model(age_coef=2e-3)]
    for bad in (torch.zeros(2, 2, 2, 16), torch.zeros(2, 2, 2, 2, 16), torch.zeros(3, 3, 2, 2, 16), torch.zeros(3, 2, 2, 2, 16, dtype=torch.int32)):
        with pytest.raises(ValueError, match=r"state must be a float tensor \[3, 2, 2, 2, 16\]"):
            m.predict_record(x, 8, mode="sequence", state=bad, heads=hs)
    with pytest.raises(ValueError, match="sequence"):
        m.predict_record(x, 8, state=torch.zeros(3, 2, 2, 2, 16), heads=hs)
    with pytest.raises(ValueError, match="sequence"):
        m.predict_record(x, 8, return_state=True, heads=hs)


def test_check_record_state_rows():
    x = torch.zeros(2, 3, 100)
    check_record_state(x, "sequence", torch.zeros(4, 2, 2, 2, 16), True, 4)
    check_record_state(x, "sequence", torch.zeros(2, 2, 2, 16), True)            # without heads: [B, 2, 2, 16]
    with pytest.raises(ValueError, match=r"\[4, 2, 2, 2, 16\]"):
        check_record_state(x, "sequence", torch.zeros(2, 2, 2, 16), True, 4)


def test_set_heads_messages_unchanged():
    """SlidingScorer.set_heads goes through the same check with its own words"""
    from tskd_b200.model import check_head_models
    m = _model()
    with pytest.raises(TypeError, match="set_heads takes a list of B200MyCNN models"):
        check_head_models(m, m.arch, m._device(), "set_heads", "the scorer's model", "the scorer")
    with pytest.raises(ValueError, match=r"heads\[0\] differs from the scorer's model in window"):
        check_head_models([_model(window=7508)], m.arch, m._device(), "set_heads", "the scorer's model", "the scorer")
