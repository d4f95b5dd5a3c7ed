"""CPU: SlidingScorer.restore rejects malformed states in Python, before any library or device call (the scorer here
has no library behind it: touching it fails the test)."""
import ctypes

import pytest
import torch

import tskd_b200
from tskd_b200 import capi


class _NoLibrary:
    def __getattr__(self, name):
        raise AssertionError(f"library reached: {name}")


class _NoModel:
    def _ensure_handle(self):
        raise AssertionError("library handle requested")


P, C, W, L, T = 6, 3, 7504, 1871, 24
FIELDS = dict(magic=capi.SLIDE_STATE_MAGIC, version=capi.SLIDE_STATE_VERSION, path=capi.PATH_TENSORCORE, dtype=capi.DTYPE_BF16,
              in_channels=C, window=W, lstm_input=L, feature_stride=4, tail_len=T)


def _scorer():
    sc = object.__new__(tskd_b200.SlidingScorer)
    sc.model, sc.n_patients, sc.stride, sc.dtype, sc.channels, sc.window = _NoModel(), P, 1876, torch.bfloat16, C, W
    sc._lib, sc._s, sc._hv, sc.device, sc.window_index = _NoLibrary(), object(), 0, torch.device("cpu"), -1
    sc._state_fields = dict(FIELDS)
    return sc


def _state(k=2):
    s = {"features": torch.zeros(k, L), "tail": torch.zeros(k, C, T), "seen": torch.full((k,), W, dtype=torch.int64)}
    s.update(FIELDS, frontend_digest=0xFEDCBA9876543210)
    return s


def test_header_fields_match_the_c_struct():
    assert tskd_b200.SlidingScorer.STATE_HEADER == tuple(FIELDS) + ("frontend_digest",)
    assert ctypes.sizeof(capi.SlideStateHeader) == 40


def _without(key):
    s = _state()
    del s[key]
    return s


def _with(**kw):
    s = _state()
    s.update(kw)
    return s


BAD = {
    "not-a-dict": [("features", 0)],
    "no-features": _without("features"),
    "no-tail": _without("tail"),
    "no-seen": _without("seen"),
    "no-digest": _without("frontend_digest"),
    "no-magic": _without("magic"),
    "magic": _with(magic=0x12345678),
    "version": _with(version=2),
    "path": _with(path=capi.PATH_GENERIC),
    "dtype": _with(dtype=capi.DTYPE_F32),
    "channels": _with(in_channels=2),
    "window": _with(window=7500),
    "lstm-input": _with(lstm_input=1870),
    "feature-stride": _with(feature_stride=16),
    "tail-len": _with(tail_len=16),
    "digest-not-int": _with(frontend_digest=1.5),
    "digest-negative": _with(frontend_digest=-1),
    "digest-too-big": _with(frontend_digest=1 << 64),
    "features-rows": _with(features=torch.zeros(3, L)),
    "features-length": _with(features=torch.zeros(2, L - 1)),
    "features-dtype": _with(features=torch.zeros(2, L, dtype=torch.float64)),
    "features-list": _with(features=[[0.0] * L] * 2),
    "tail-shape": _with(tail=torch.zeros(2, C, T + 1)),
    "tail-dtype": _with(tail=torch.zeros(2, C, T, dtype=torch.bfloat16)),
    "seen-dtype": _with(seen=torch.zeros(2, dtype=torch.int32)),
    "seen-shape": _with(seen=torch.zeros(2, 1, dtype=torch.int64)),
    "seen-below-minus-one": _with(seen=torch.tensor([0, -2])),
}


@pytest.mark.parametrize("name", list(BAD))
def test_malformed_states_are_rejected_in_python(name):
    with pytest.raises(ValueError):
        _scorer().restore([0, 4], BAD[name])


def test_bad_indices_are_rejected_in_python():
    for idx in ([0, 0], [6, 1], [-1, 2]):
        with pytest.raises(ValueError):
            _scorer().restore(idx, _state())
        with pytest.raises(ValueError):
            _scorer().export(idx)


def test_valid_state_reaches_the_library_only_then():
    """a valid state passes validation and stops at the first library touch"""
    sc = _scorer()
    f, t, s = sc.check_state(_state(), 2)
    assert f.shape == (2, L) and t.shape == (2, C, T) and s.dtype == torch.int64
    assert sc.check_state(_state(0), 0)[0].shape == (0, L)
    with pytest.raises(AssertionError, match="library handle"):
        sc.restore([0, 5], _state())
    with pytest.raises(AssertionError, match="library handle"):
        sc.export([1, 2])
