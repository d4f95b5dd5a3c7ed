"""CPU: the argument checks of B200MyCNN.predict_record, which run before any library call, and the window set it
scores (create_batch's windows, plus the last full window that range(0, N - W, S) drops)."""
import pytest
import torch

import tskd_b200
from tskd_b200 import capi


def _model(kind="mycnn5", C=3, W=7504):
    return tskd_b200.B200MyCNN(tskd_b200.ARCH_PRESETS[kind].with_shape(C, W))


def _generic_model():
    arch = tskd_b200.ArchConfig(in_channels=3, k1=5, k2=5, pool_k=4, pool_s=4, window=250, age_coef=1e-4)
    return tskd_b200.B200MyCNN(arch, has_out12=False)


def test_shape_and_dtype_checks():
    m = _model()
    x = torch.zeros(2, 3, 9000, dtype=torch.bfloat16)
    for bad in (x[0], x[:, :2], x.unsqueeze(0), x.half(), x.double(), torch.zeros(0, 3, 9000), "x"):
        with pytest.raises(ValueError):
            m.check_record_args(bad, 8)
        with pytest.raises(ValueError):
            m.predict_record(bad, 8)


def test_stride_checks():
    m = _model()
    x = torch.zeros(2, 3, 9000)
    for bad in (0, -4, 2, 6, 7501, 2.5, "8", None, True):
        with pytest.raises(ValueError):
            m.predict_record(x, bad)
    assert m.check_record_args(x, 8)[0] == 8
    assert m.check_record_args(x, torch.tensor(12))[0] == 12
    assert m.check_record_args(x, 90000)[0] == 90000              # strides past the window are allowed
    g = _generic_model()                                           # pool (4, 4): feature stride 16
    xg = torch.zeros(1, 3, 1000)
    for bad in (4, 8, 24):
        with pytest.raises(ValueError):
            g.predict_record(xg, bad, path="generic")
        with pytest.raises(ValueError):
            g.predict_record(xg, bad)
    assert g.check_record_args(xg, 32, path="generic")[0] == 32
    assert g.check_record_args(xg, 4, path="tensorcore")[0] == 4   # the library refuses the path itself (B2CNN_EARCH)


def test_age_and_path_checks():
    m = _model()
    x = torch.zeros(3, 3, 9000)
    for bad in (torch.ones(2), torch.ones(4), [1.0, 2.0], torch.ones(2, 2)):
        with pytest.raises(ValueError):
            m.predict_record(x, 8, bad)
    for bad in ("stream", "tc", None):
        with pytest.raises(ValueError):
            m.predict_record(x, 8, path=bad)
    for ok in (None, 50.0, torch.tensor(50.0), torch.ones(1), torch.arange(3.0), [1.0, 2.0, 3.0]):
        s, age = m.check_record_args(x, 8, ok)
        assert age.dtype == torch.float32 and age.dim() == 1 and age.numel() in (1, 3)
    assert float(m.check_record_args(x, 8)[1][0]) == 65.0


@pytest.mark.parametrize("N,W,S", [(600, 120, 72), (120 + 5 * 72, 120, 72), (119, 120, 12), (120, 120, 12),
                                   (75000 * 3, 75000, 45000), (10_800_000, 75000, 7500), (400, 200, 260)])
def test_window_set_is_create_batch_plus_the_last(N, W, S):
    n_w = (N - W) // S + 1 if N >= W else 0
    starts = list(range(0, N - W, S))                                # bin/utils.py create_batch
    mine = [w * S for w in range(n_w)]
    assert all(s + W <= N for s in mine)
    if n_w and (N - W) % S == 0:
        assert mine[:-1] == starts and mine[-1] == N - W
    else:
        assert mine == starts


def test_symbols_bound():
    assert "b2cnn_score_record" in capi.SYMBOLS and "b2cnn_record_workspace_bytes" in capi.SYMBOLS
