"""CPU: SlidingScorer.set_heads(models, shorter_windows=True) accepts and rejects head windows in Python, before any
library or device call, and shorter_windows=False keeps the messages of same-window heads (the scorer here has no
library behind it: touching it fails the test)."""
from dataclasses import replace

import pytest
import torch

import tskd_b200

ARCH = tskd_b200.ARCH_PRESETS["mycnn5"].with_shape(3, 7504)
P = 6


class _NoLibrary:
    def __getattr__(self, name):
        raise AssertionError(f"library reached: {name}")


class _NoModel:
    arch = ARCH

    def _ensure_handle(self):
        raise AssertionError("library handle requested")


def _scorer(arch=ARCH):
    sc = object.__new__(tskd_b200.SlidingScorer)
    sc.model, sc.n_patients, sc.stride, sc.dtype, sc.channels, sc.window = _NoModel(), P, 752, torch.bfloat16, 3, arch.window
    sc.model.arch = arch
    sc._lib, sc._s, sc._hv, sc.device, sc.window_index = _NoLibrary(), object(), 0, torch.device("cpu"), -1
    sc._heads = ()
    return sc


def _model(window=7504, **change):
    return tskd_b200.B200MyCNN(replace(ARCH, window=window, **change))


@pytest.mark.parametrize("windows", [(7504,), (3008, 1504, 752, 7504), (24,), (7500, 28), (500,)])
def test_windows_that_end_on_the_lattice_are_accepted(windows):
    sc = _scorer()
    models = [_model(Wk) for Wk in windows]
    assert sc.check_heads(models, shorter_windows=True) == tuple(models)
    with pytest.raises(AssertionError, match="library handle"):
        sc.set_heads(models, shorter_windows=True)
    assert sc.heads == () and sc.head_windows == (7504,)


@pytest.mark.parametrize("Wk,match", [(7508, "longer"), (8000, "longer"), (3006, "multiple"), (7503, "multiple"),
                                      (7501, "multiple")])
def test_other_windows_are_rejected(Wk, match):
    with pytest.raises(ValueError, match=match):
        _scorer().set_heads([_model(3008), _model(Wk)], shorter_windows=True)


@pytest.mark.parametrize("change", [dict(in_channels=2), dict(k1=5, k2=5, pool_k=2), dict(act="relu"), dict(affine=True),
                                    dict(pool_s=3)])
def test_other_front_ends_are_rejected(change):
    with pytest.raises(ValueError, match="differs"):
        _scorer().set_heads([_model(3008, **change)], shorter_windows=True)


def test_an_lstm_input_that_does_not_fit_the_window_is_rejected():
    """lstm_input == L_out(window): a head whose l_out is not the feature count of its window"""
    class OffByOne(type(ARCH)):
        @property
        def l_out(self):
            return super().l_out + 1

    m = object.__new__(tskd_b200.B200MyCNN)
    object.__setattr__(m, "__dict__", {"arch": OffByOne(**{f: getattr(ARCH, f) for f in ARCH.__dataclass_fields__} | {"window": 3008})})
    with pytest.raises(ValueError, match="feature count"):
        _scorer().check_heads([m], shorter_windows=True)


def test_odd_phase_scorer():
    """W = 7501 (phi = 3): heads at 3001 and 1 + 4 k are on its lattice, 3000 is not"""
    sc = _scorer(replace(ARCH, window=7501))
    assert len(sc.check_heads([_model(3001), _model(1501), _model(7501)], shorter_windows=True)) == 3
    with pytest.raises(ValueError, match="multiple"):
        sc.check_heads([_model(3000)], shorter_windows=True)


def test_generic_feature_stride():
    """pool_s = 4: F = 16"""
    arch = tskd_b200.ArchConfig(in_channels=16, k1=3, k2=8, pool_k=4, pool_s=4, window=1470)
    sc = _scorer(arch)
    ok = tskd_b200.B200MyCNN(replace(arch, window=670))
    assert sc.check_heads([ok], shorter_windows=True) == (ok,)
    with pytest.raises(ValueError, match="multiple of the feature stride 16"):
        sc.check_heads([tskd_b200.B200MyCNN(replace(arch, window=674))], shorter_windows=True)


def test_without_the_flag_a_window_is_an_architecture_difference():
    """shorter_windows=False keeps the message of same-window heads"""
    for Wk in (3008, 7508):
        with pytest.raises(ValueError, match=r"heads\[0\] differs from the scorer's model in window, l_out"):
            _scorer().set_heads([_model(Wk)])
    with pytest.raises(ValueError, match=r"heads\[0\] differs from the scorer's model in window, l_out"):
        _scorer().set_heads([_model(3008)], shorter_windows=False)


@pytest.mark.parametrize("bad", [1, "yes", None])
def test_flag_must_be_a_bool(bad):
    with pytest.raises(TypeError, match="shorter_windows"):
        _scorer().set_heads([_model(3008)], shorter_windows=bad)


def test_head_windows_is_read_only_and_follows_the_heads():
    sc = _scorer()
    with pytest.raises(AttributeError):
        sc.head_windows = (1,)
    sc._heads = (_model(3008), _model(752))
    assert sc.head_windows == (7504, 3008, 752)
