"""CPU: SlidingScorer's path argument and the stride rule of each path are checked in Python, before the library."""
import pytest
import torch

import tskd_b200


class _NoHandle(tskd_b200.B200MyCNN):
    def _ensure_handle(self):
        raise AssertionError("library handle requested")


def _model(C=3, k1=10, k2=5, pk=3, ps=2, W=7504):
    return _NoHandle(tskd_b200.ArchConfig(in_channels=C, k1=k1, k2=k2, pool_k=pk, pool_s=ps, window=W))


@pytest.mark.parametrize("path", ["tc", "GENERIC", "stream", "", None, 1])
def test_unknown_path(path):
    with pytest.raises(ValueError, match="path"):
        tskd_b200.SlidingScorer(_model(), 4, 1876, path=path)


@pytest.mark.parametrize("path,geo,S", [
    ("generic", (3, 4, 3, 2, 3, 600), 48),     # F = 9
    ("auto", (3, 4, 3, 2, 3, 600), 12),
    ("generic", (16, 3, 8, 4, 4, 1470), 24),   # F = 16
    ("generic", (3, 10, 5, 3, 2, 7504), 6),    # F = 4
    ("tensorcore", (3, 4, 3, 2, 3, 600), 6),   # the tensor-core path's rule: a multiple of 4
    ("generic", (3, 4, 3, 2, 3, 600), 603),    # longer than the window
    ("auto", (3, 4, 3, 2, 3, 600), 0),
])
def test_stride_must_be_a_multiple_of_the_feature_stride(path, geo, S):
    with pytest.raises(ValueError, match="stride"):
        tskd_b200.SlidingScorer(_model(*geo), 4, S, path=path)


@pytest.mark.parametrize("path,geo,S", [
    ("generic", (3, 4, 3, 2, 3, 600), 45),
    ("auto", (16, 3, 8, 4, 4, 1470), 32),
    ("generic", (2, 4, 3, 1, 1, 300), 7),      # F = 1: any stride
    ("tensorcore", (3, 10, 5, 3, 2, 7504), 1876),
])
def test_valid_arguments_reach_the_library(path, geo, S):
    with pytest.raises(AssertionError, match="library handle"):
        tskd_b200.SlidingScorer(_model(*geo), 4, S, path=path)
