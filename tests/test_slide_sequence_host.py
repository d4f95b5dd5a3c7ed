"""CPU: SlidingScorer's sequence mode without a GPU -- mode validation before any library call, the C symbols bound in
capi, check_state's "lstm" rule in both modes, and the window arithmetic of the sequence identity (s0, o, j) on
hand-worked cases."""
import pytest
import torch

import tskd_b200
from tskd_b200 import capi
from test_slide_state_host import FIELDS, C, L, T, _scorer, _state


def _seq_state(k=2):
    s = _state(k)
    s["lstm"] = torch.zeros(k, 2, 2, 16)
    return s


def _seq_scorer():
    sc = _scorer()
    sc.mode = "sequence"
    return sc


class _Arch:
    window, in_channels, pool_s = 7504, 3, 2


class _Model:
    arch = _Arch()

    def _ensure_handle(self):
        raise AssertionError("library handle requested")


@pytest.mark.parametrize("mode", ["seq", "Sequence", "", None, 1, capi.MODE_SEQUENCE])
def test_bad_mode_is_refused_before_the_library(mode):
    with pytest.raises(ValueError, match="mode"):
        tskd_b200.SlidingScorer(_Model(), 4, 1876, mode=mode)


def test_modes_and_symbols():
    assert tskd_b200.SlidingScorer.MODES == {"independent": capi.MODE_INDEPENDENT, "sequence": capi.MODE_SEQUENCE}
    assert tskd_b200.SlidingScorer.mode == "independent"                       # the default of every scorer
    for name in ("b2cnn_slide_create_ex", "b2cnn_slide_mode", "b2cnn_slide_export_ex", "b2cnn_slide_import_ex"):
        assert name in capi.SYMBOLS


def test_check_state_lstm_in_both_modes():
    ind, seq = _scorer(), _seq_scorer()
    f, t, s = ind.check_state(_state(), 2)                                    # unchanged for an independent scorer
    assert f.shape == (2, L) and t.shape == (2, C, T)
    f, t, s = seq.check_state(_seq_state(), 2)
    assert s.dtype == torch.int64
    assert seq.check_state(_seq_state(0), 0)[0].shape == (0, L)
    with pytest.raises(ValueError, match="another mode"):
        ind.check_state(_seq_state(), 2)
    with pytest.raises(ValueError, match="another mode"):
        seq.check_state(_state(), 2)
    for bad in (torch.zeros(3, 2, 2, 16), torch.zeros(2, 4, 16), torch.zeros(2, 2, 2, 16, dtype=torch.float64),
                torch.zeros(2, 2, 2, 15), [[0.0]]):
        with pytest.raises(ValueError, match="lstm"):
            seq.check_state(dict(_seq_state(), lstm=bad), 2)
    with pytest.raises(ValueError, match="another mode"):                     # refused before any library call
        seq.restore([0, 1], _state())
    with pytest.raises(AssertionError, match="library handle"):               # a valid state reaches the library only then
        seq.restore([0, 1], _seq_state())


def test_set_heads_is_refused_on_a_sequence_scorer():
    sc = _seq_scorer()
    sc.check_heads = lambda models, shorter_windows=False: tuple(models)
    with pytest.raises(ValueError, match="heads"):
        sc.set_heads([object()])


def s0_o(W, S, H=0):
    """(s0, o): samples_seen at the first push with samples_seen >= W after an admission with H samples, and the
    stream offset of that push's window"""
    s0 = H + max(1, -(-(W - H) // S)) * S
    return s0, s0 - W


def j_of(seen, W, S, H=0):
    """the index j of the push at which samples_seen == seen (None before the first window)"""
    s0, _ = s0_o(W, S, H)
    return None if seen < s0 else (seen - s0) // S


@pytest.mark.parametrize("W,S,H,s0,o", [
    (120, 12, 0, 120, 0),             # W a multiple of S: the 10th push
    (7504, 1876, 0, 7504, 0),
    (7504, 752, 0, 7520, 16),         # ceil(W / S) S: the first window starts 16 samples into the stream
    (75000, 7500, 0, 75000, 0),
    (120, 12, 108, 120, 0),           # H = W - S: the next push completes the window
    (120, 12, 120, 132, 12),          # H = W: the history's own window is not scored; the next push's is
    (7504, 1876, 7504, 9380, 1876),
    (120, 12, 36, 120, 0),            # H = S + R (R = 24 of the generic golden)
    (7504, 1876, 1900, 7528, 24),     # H = S + R on the tensor cores
    (120, 120, 0, 120, 0),
])
def test_window_arithmetic(W, S, H, s0, o):
    assert s0_o(W, S, H) == (s0, o)
    assert j_of(s0 - S, W, S, H) is None
    assert [j_of(s0 + j * S, W, S, H) for j in range(4)] == [0, 1, 2, 3]
    # window j spans stream samples [o + j S, o + j S + W) and ends at samples_seen
    for j in range(4):
        assert o + j * S + W == s0 + j * S
