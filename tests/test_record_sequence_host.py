"""CPU: predict_record(mode="sequence") -- its mode check, which runs before any library call, the C symbols it binds, and
the golden of the reference's utils.run_model (tests/golden/run_model_record.npz) against the float64 oracle scanning
each recording's windows w*120 .. w*120 + 119 as one LSTM sequence (which also pins the window set)."""
import os

import numpy as np
import pytest
import torch

import tskd_b200
from conftest import GOLDEN, load_golden
from oracle import mycnn_torch as O
from oracle.infer_ref import infer_reference
from oracle.train_ref import assert_close_elem
from tskd_b200 import capi


def test_mode_checks():
    m = tskd_b200.B200MyCNN(tskd_b200.ARCH_PRESETS["mycnn5"].with_shape(3, 7504))
    x = torch.zeros(2, 3, 9000, dtype=torch.bfloat16)
    for bad in ("seq", "Sequence", "", None, 1, capi.MODE_SEQUENCE, ["sequence"]):
        with pytest.raises(ValueError, match="mode"):
            m.check_record_args(x, 8, mode=bad)
        with pytest.raises(ValueError, match="mode"):
            m.predict_record(x, 8, mode=bad)
    for ok in ("independent", "sequence"):
        assert m.check_record_args(x, 8, mode=ok)[0] == 8


def test_symbols_bound():
    assert "b2cnn_score_record_ex" in capi.SYMBOLS and "b2cnn_record_workspace_bytes_ex" in capi.SYMBOLS


def _windows(frame, W=120, S=120):
    """[n_w, 10, W] float32 windows of a [N, 10] frame, starting at multiples of S"""
    x = torch.from_numpy(frame).T.contiguous()
    return x.unfold(1, W, S).permute(1, 0, 2).contiguous()


@pytest.mark.parametrize("tag", ["a", "b", "nan"])
def test_run_model_golden_against_float64(tag):
    g = np.load(os.path.join(GOLDEN, "run_model_record.npz"))
    _, sd = load_golden("mycnn5_xtestinput.npz")                    # the same MyCNN5.pth checkpoint
    ref = O.RefMyCNN(O.ARCH_MYCNN5)
    ref.load_state_dict(sd)
    ref.eval()
    frame = g[f"frame_{tag}"]
    win = _windows(frame)
    n_gold = g[f"prob_{tag}"].shape[1]
    N = frame.shape[0]
    assert n_gold == len(range(0, N - 120, 120))                     # create_batch's window count
    assert win.shape[0] == n_gold + (1 if (N - 120) % 120 == 0 else 0)
    for i, age in enumerate(g["ages"]):
        a = torch.tensor([float(age)])
        t = torch.sigmoid(infer_reference(ref, win, a, "sequence")["z"])[:n_gold]
        t32 = torch.sigmoid(infer_reference(ref, win, a, "sequence", dtype=torch.float32)["z"])[:n_gold]
        gold = torch.from_numpy(g[f"prob_{tag}"][i])
        assert_close_elem(f"run_model {tag} age {age}", gold, t, t32)
        if tag == "nan":                                               # the NaN at row 6000 is in window 50
            assert torch.isfinite(gold[:50]).all() and torch.isnan(gold[50:]).all()
