"""CPU: SlidingScorer.set_heads and push(heads=...) reject bad arguments in Python, before any library or device call
(the scorer here has no library behind it: touching it fails the test)."""
import pytest
import torch

import tskd_b200
from tskd_b200 import capi

ARCH = tskd_b200.ARCH_PRESETS["mycnn5"].with_shape(3, 7504)
P = 6


class _NoLibrary:
    def __getattr__(self, name):
        raise AssertionError(f"library reached: {name}")


class _NoModel:
    arch = ARCH

    def _ensure_handle(self):
        raise AssertionError("library handle requested")


def _scorer(device="cpu"):
    sc = object.__new__(tskd_b200.SlidingScorer)
    sc.model, sc.n_patients, sc.stride, sc.dtype, sc.channels, sc.window = _NoModel(), P, 1876, torch.bfloat16, 3, 7504
    sc._lib, sc._s, sc._hv, sc.device, sc.window_index = _NoLibrary(), object(), 0, torch.device(device), -1
    sc._heads = ()
    return sc


def _model(arch=ARCH):
    return tskd_b200.B200MyCNN(arch)


@pytest.mark.parametrize("bad", [None, 3, "model", torch.zeros(2)])
def test_non_lists_are_rejected(bad):
    with pytest.raises(TypeError):
        _scorer().set_heads(bad)


def test_a_bare_model_is_not_a_list():
    with pytest.raises(TypeError):
        _scorer().set_heads(_model())


@pytest.mark.parametrize("bad", [None, 1.5, torch.nn.Linear(2, 1), "m"])
def test_non_models_are_rejected(bad):
    with pytest.raises(TypeError):
        _scorer().set_heads([_model(), bad])


@pytest.mark.parametrize("change", [dict(in_channels=2), dict(window=7500), dict(k1=5, k2=5, pool_k=2), dict(act="relu"),
                                    dict(affine=True), dict(pool_s=3)])
def test_other_architectures_are_rejected(change):
    from dataclasses import replace
    with pytest.raises(ValueError, match="differs"):
        _scorer().set_heads([_model(), _model(replace(ARCH, **change))])


def test_too_many_heads_are_rejected():
    with pytest.raises(ValueError, match="at most"):
        _scorer().set_heads([_model() for _ in range(capi.SLIDE_MAX_HEADS + 1)])


def test_heads_on_another_device_are_rejected():
    with pytest.raises(ValueError, match="scorer on cuda"):
        _scorer("cuda:0").set_heads([_model()])


def test_valid_heads_reach_the_library_only_then():
    """another age_coef is allowed; valid heads pass validation and stop at the first library touch"""
    from dataclasses import replace
    sc = _scorer()
    models = [_model() for _ in range(capi.SLIDE_MAX_HEADS)]
    models[1] = _model(replace(ARCH, age_coef=1e-3))
    assert sc.check_heads(models) == tuple(models)
    assert sc.check_heads([]) == ()
    with pytest.raises(AssertionError, match="library handle"):
        sc.set_heads(models)
    assert sc.heads == ()                                          # nothing attached


def test_heads_is_read_only():
    sc = _scorer()
    with pytest.raises(AttributeError):
        sc.heads = (_model(),)


@pytest.mark.parametrize("bad", [1, "yes", None])
def test_push_heads_flag_must_be_a_bool(bad):
    with pytest.raises(TypeError):
        _scorer().push(torch.zeros(P, 3, 1876, dtype=torch.bfloat16), heads=bad)


def test_push_with_heads_validates_samples_first():
    with pytest.raises(RuntimeError, match="expected samples"):
        _scorer().push(torch.zeros(P, 3, 1875, dtype=torch.bfloat16), heads=True)
    with pytest.raises(AssertionError, match="library handle"):
        _scorer().push(torch.zeros(P, 3, 1876, dtype=torch.bfloat16), heads=True)
