"""Generate ``tests/golden/run_model_record.npz`` by running the UNMODIFIED reference's whole-recording scorer.

Needs a checkout of the reference at ``make_golden.REF``; the tests only read the fixture:

    python tests/golden/make_golden_run_model.py

What is executed is ``bin/utils.py``'s ``run_model`` (utils.py:671-692), verbatim, with the stub modules
``make_golden.py`` uses for the absent ``wfdb`` / ``pyspark`` imports, on the shipped ``model/MyCNN5.pth``.
``run_model`` cuts one recording into ``create_batch(df, 120, overlap_pct=0)`` windows and calls ``model(x_arr, a_arr)``
once on all of them, so the LSTM scans the recording's windows in order.  Its age is ``(1, n)``, which broadcasts the
``(n, 1)`` logits to ``(1, n, n)`` with ``[0, i, j]`` = window i at age j; with one age per call every column is the
same, and column 0 is stored.  Frames: 8640 rows ((N - 120) % 120 == 0: create_batch drops the last full window), 8660
rows (it does not), and the first frame again with one NaN at row 6000, each at ages 50 and 72.  Nothing from this
repo's product code is used to produce the expected values.
"""
import os
import sys
import types

import numpy as np
import pandas as pd
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from make_golden import OUT, REF, load_ckpt  # noqa: E402  (also registers the reference class for the pickles)


def _physio_frame(rng, n):
    """n rows x 10 vital-sign-like float32 columns (5-second grid): a per-channel baseline, a slow random walk and noise"""
    base = np.array([80.0, 16.0, 97.0, 2.0, 97.0, 8.0, 0.5, 85.0, 60.0, 120.0])
    walk = np.cumsum(rng.normal(0.0, 0.05, size=(n, 10)), axis=0) * base * 0.02
    noise = rng.normal(0.0, 1.0, size=(n, 10)) * np.maximum(base * 0.02, 0.05)
    return np.clip(base + walk + noise, 0.0, 250.0).astype(np.float32)


def golden_run_model_record():
    for name in ("wfdb", "pyspark", "pyspark.sql"):
        sys.modules.setdefault(name, types.ModuleType(name))
    sys.modules["pyspark.sql"].SparkSession = object
    cwd = os.getcwd(); os.chdir(REF)
    try:
        import utils as ref_utils
    finally:
        os.chdir(cwd)
    m = load_ckpt(5)
    rng = np.random.default_rng(2024)
    frame_a, frame_b = _physio_frame(rng, 8640), _physio_frame(rng, 8660)
    frame_nan = frame_a.copy()
    frame_nan[6000, 3] = np.nan
    ages = np.array([50.0, 72.0])
    out = dict(frame_a=frame_a, frame_b=frame_b, frame_nan=frame_nan, ages=ages)
    for tag, fr in (("a", frame_a), ("b", frame_b), ("nan", frame_nan)):
        probs = []
        for age in ages:
            _, y_prob = ref_utils.run_model(m, torch.device("cpu"), pd.DataFrame(fr), float(age))
            y = np.array(y_prob, dtype=np.float64)
            n = len(range(0, fr.shape[0] - 120, 120))
            assert y.shape == (1, n, n), y.shape
            assert np.array_equal(y[0], np.repeat(y[0][:, :1], n, axis=1), equal_nan=True)    # every column the same
            probs.append(y[0][:, 0])
        out[f"prob_{tag}"] = np.stack(probs)
    p = out["prob_nan"]
    assert np.isfinite(p[:, :50]).all() and np.isnan(p[:, 50:]).all()                        # row 6000 is in window 50
    np.savez_compressed(os.path.join(OUT, "run_model_record.npz"), **out)
    print("run_model_record:", {k: v.shape for k, v in out.items()}, out["prob_a"][:, :3])


if __name__ == "__main__":
    golden_run_model_record()
