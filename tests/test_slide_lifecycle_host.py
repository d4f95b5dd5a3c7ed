"""CPU: SlidingScorer.admit / discharge reject bad patient indices and histories in Python, before any library or
device call (the scorer here has no library behind it: touching it fails the test)."""
import pytest
import torch

import tskd_b200


class _NoLibrary:
    def __getattr__(self, name):
        raise AssertionError(f"library reached: {name}")


class _NoModel:
    def _ensure_handle(self):
        raise AssertionError("library handle requested")


def _scorer(P=6, C=3, W=7504, S=1876, dtype=torch.bfloat16):
    sc = object.__new__(tskd_b200.SlidingScorer)
    sc.model, sc.n_patients, sc.stride, sc.dtype, sc.channels, sc.window = _NoModel(), P, S, dtype, C, W
    sc._lib, sc._s, sc._hv, sc.device, sc.window_index = _NoLibrary(), object(), 0, torch.device("cpu"), -1
    return sc


@pytest.mark.parametrize("patients", [[6], [-1], [0, 3, 0], [1.0], torch.tensor([0.0, 1.0]), torch.tensor([True]),
                                      "01", [2, 2], torch.tensor([5, 6])])
def test_bad_patient_indices(patients):
    sc = _scorer()
    with pytest.raises(ValueError):
        sc.admit(patients)
    with pytest.raises(ValueError):
        sc.discharge(patients)


@pytest.mark.parametrize("shape,dtype", [
    ((2, 3, 7508), torch.bfloat16),      # longer than the window
    ((3, 3, 100), torch.bfloat16),       # one row per listed patient
    ((2, 2, 100), torch.bfloat16),       # channels
    ((2, 3), torch.bfloat16),
    ((2, 3, 100), torch.float32),        # not the scorer's dtype
    ((2, 3, 100), torch.float16),
])
def test_bad_histories(shape, dtype):
    with pytest.raises(ValueError):
        _scorer().admit([0, 4], torch.zeros(shape, dtype=dtype))


def test_history_must_be_a_tensor():
    with pytest.raises(ValueError):
        _scorer().admit([0], [[0.0] * 100] * 3)


def test_valid_arguments_reach_the_library_only_then():
    """a valid call passes validation and stops at the first library touch"""
    sc = _scorer()
    assert sc.check_patients(torch.tensor([4, 0, 2])) == [4, 0, 2]
    assert sc.check_history(torch.zeros(2, 3, 7504, dtype=torch.bfloat16), 2) == 7504
    assert sc.check_history(torch.zeros(2, 3, 0, dtype=torch.bfloat16), 2) == 0
    with pytest.raises(AssertionError, match="library handle"):
        sc.admit([0, 5], torch.zeros(2, 3, 64, dtype=torch.bfloat16))
    with pytest.raises(AssertionError, match="library handle"):
        sc.discharge([])
