"""CPU: SlidingScorer rejects bad arguments before it touches the library or a device."""
import pytest
import torch

import tskd_b200


def _model(W=7504):
    return tskd_b200.B200MyCNN(tskd_b200.ARCH_PRESETS["mycnn5"].with_shape(3, W))


@pytest.mark.parametrize("P,S,dtype", [
    (4, 6, torch.bfloat16),          # not a multiple of the feature stride
    (4, 0, torch.bfloat16),
    (4, 7508, torch.bfloat16),       # longer than the window
    (0, 1876, torch.bfloat16),
    (4, 1876, torch.float16),
])
def test_scorer_rejects_bad_arguments(P, S, dtype):
    with pytest.raises(ValueError):
        tskd_b200.SlidingScorer(_model(), P, S, dtype)


def test_scorer_is_exported_next_to_the_ring():
    assert tskd_b200.SlidingScorer.__module__.endswith("slide")
    assert "SlidingScorer" in tskd_b200.__all__ and "PatientRing" in tskd_b200.__all__
